"""The training step of `bench.py --workload train` on the three GEMM engines of the training path, in one process.

    python tools/bench_train.py [--rounds 6] [--steps 5] [--warmup 3] [--rays 1200] [--out DIR] [--dry-run]

One step is bench.py's run_train step: config A (KITTI defaults, sphere 1500x452), 1200 pixels of the stride-2 grid x 64
samples in ONE chunk, the same depth + colour + KL + gaussian-mean loss, backward to the 2 x 22 ResnetFC tensors and the
five feature maps.  Engines: matmul="fp32" (float32 SIMT, the strict mode), "tf32" (wgmma tf32) and "fp32tc" (split
3xTF32 wgmma).  After --warmup steps of each, --rounds rounds time --steps steps of every engine with CUDA events, the
engine order rotating from round to round; per engine: median ms per step and its spread over the rounds, the forward /
backward split of one more step per round (events around the two halves), and the launch counts.

Gradients: one more step per engine on the same pixels and explicit, seeded noise; the relative L2 of every tf32 and
fp32tc gradient tensor against the fp32 engine's (worst tensor and all parameters / all maps together), next to a
second fp32 run (its feature-map gradients differ run to run by the order of float atomics: the strict mode's own
noise floor).  Prints one JSON line per engine and a summary line with the card's name, power limit and maximum SM
clock, read in the same run; --out DIR also writes them to DIR/bench_train.json.  --dry-run stops before the device."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (hp_from_cfg, flop_per_ray of the train workload)
from scenerf_b200 import synth  # noqa: E402

ENGINES = ("fp32", "tf32", "fp32tc")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "nvidia-smi unavailable"


def setup(rays):
    """Host side of the workload: config, pixels (bench.py's selection), the seeded noise of the gradient step."""
    cfg = synth.config_A(name="train")
    grid = synth.grid_pixels(cfg.img_W, cfg.img_H, stride=2)
    sel = np.random.default_rng(7).permutation(grid.shape[0])[:rays]
    pix = np.ascontiguousarray(grid[sel])
    rng = np.random.default_rng(11)
    nu = rng.random((rays, cfg.n_pts_uni)).astype(np.float32)
    nn_ = rng.standard_normal((rays, cfg.n_gaussians * cfg.n_pts_per_gaussian)).astype(np.float32)
    return cfg, pix, nu, nn_


def rel_l2(a, b):
    return float(np.linalg.norm(a - b) / max(1e-30, np.linalg.norm(b)))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=6)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rays", type=int, default=1200)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dry-run", action="store_true", help="build the host inputs and print the plan; no device work")
    args = ap.parse_args()
    cfg, pix, nu, nn_ = setup(args.rays)
    flop_fwd = args.rays * bench.flop_per_ray(cfg)
    plan = {"rays": args.rays, "samples_per_ray": cfg.S, "sphere": [cfg.sphere_W, cfg.sphere_H], "pixels": list(pix.shape),
            "noise": [list(nu.shape), list(nn_.shape)], "engines": ENGINES, "rounds": args.rounds, "steps": args.steps,
            "warmup": args.warmup, "algorithmic_flop_per_step": 3.0 * flop_fwd}
    if args.dry_run:
        print(json.dumps({"dry_run": plan}))
        return

    import torch
    from scenerf_b200.autograd import PARAM_KEYS, TrainableRenderer
    if not torch.cuda.is_available():
        raise SystemExit("bench_train.py measures on a CUDA device; none is available (use --dry-run for the host path)")
    dev = torch.device("cuda", 0)
    pm, pg = synth.make_model_params(cfg)
    mk = lambda d: {k: torch.from_numpy(d[k]).to(dev).requires_grad_(True) for k in PARAM_KEYS}
    tm, tg = mk(pm), mk(pg)
    x_rgb = {k: torch.from_numpy(v).to(dev).requires_grad_(True) for k, v in synth.make_pyramid(5, cfg.sphere_W, cfg.sphere_H).items()}
    leaves = list(tm.values()) + list(tg.values()) + list(x_rgb.values())
    hp = bench.hp_from_cfg(cfg)
    tr = {e: TrainableRenderer(hp, tm, tg, device=dev, rng="philox", matmul=e) for e in ENGINES}
    K, T = torch.from_numpy(cfg.K).to(dev), torch.from_numpy(cfg.T).to(dev)
    pix_host = torch.from_numpy(pix).pin_memory()
    R = args.rays
    target = torch.rand(R, 3, device=dev, generator=torch.Generator(device=dev).manual_seed(3))

    def forward(e, noise=None):
        for p_ in leaves:
            p_.grad = None
        out = tr[e].render_rays_batch(K, T, x_rgb, sampled_pixels=pix_host.to(dev, non_blocking=True), ray_batch_size=R, noise=noise)
        return (out["color"] - target).abs().mean() + 0.01 * out["depth"].mean() + out["loss_kl"].mean() \
            + 0.01 * (out["gaussian_means"] - out["depth"].detach().unsqueeze(-1)).abs().min(dim=1)[0].mean()

    for e in ENGINES:
        for _ in range(args.warmup):
            forward(e).backward()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    step_ms = {e: [] for e in ENGINES}
    fwd_ms = {e: [] for e in ENGINES}
    bwd_ms = {e: [] for e in ENGINES}
    for r in range(args.rounds):
        for i in range(len(ENGINES)):
            e = ENGINES[(r + i) % len(ENGINES)]
            ev[0].record()
            for _ in range(args.steps):
                loss = forward(e)
                loss.backward()
            float(loss.detach().cpu())                     # D2H read of the step's result, as bench.py
            ev[1].record()
            ev[2].record()                                 # forward / backward split of one more step
            loss = forward(e)
            ev[3].record()
            loss.backward()
            ev[4].record()
            torch.cuda.synchronize()
            step_ms[e].append(ev[0].elapsed_time(ev[1]) / args.steps)
            fwd_ms[e].append(ev[2].elapsed_time(ev[3]))
            bwd_ms[e].append(ev[3].elapsed_time(ev[4]))

    noise = (torch.from_numpy(nu), torch.from_numpy(nn_))
    grads, losses = {}, {}
    for e in ENGINES + ("fp32",):
        loss = forward(e, noise)
        loss.backward()
        key = e if e not in grads else "fp32_rerun"
        losses[key] = float(loss.detach().cpu())
        grads[key] = ({"main." + k: tm[k].grad.double().cpu().numpy() for k in PARAM_KEYS} |
                      {"gauss." + k: tg[k].grad.double().cpu().numpy() for k in PARAM_KEYS},
                      {k: v.grad.double().cpu().numpy() for k, v in x_rgb.items()})

    def deviation(e):
        res = {}
        for what, i in (("params", 0), ("maps", 1)):
            a, b = grads[e][i], grads["fp32"][i]
            per = {k: rel_l2(a[k], b[k]) for k in b if np.abs(b[k]).max() > 0}
            res[what] = {"worst_tensor": max(per, key=per.get), "worst_rel_l2": max(per.values()),
                         "all_rel_l2": rel_l2(np.concatenate([a[k].ravel() for k in b]), np.concatenate([b[k].ravel() for k in b]))}
        res["loss_rel"] = abs(losses[e] - losses["fp32"]) / abs(losses["fp32"])
        return res

    gpu = card()
    rows = []
    for e in ENGINES:
        ms = np.array(step_ms[e])
        t = tr[e].renderer
        row = {"engine": e, "ms_per_step_median": float(np.median(ms)), "ms_per_step_min": float(ms.min()),
               "ms_per_step_max": float(ms.max()), "rounds": args.rounds, "steps_per_round": args.steps,
               "forward_ms_median": float(np.median(fwd_ms[e])), "backward_ms_median": float(np.median(bwd_ms[e])),
               "launches_forward": int(t.last_launches), "launches_backward": int(t.last_backward_launches),
               "rays_per_sec": R / (float(np.median(ms)) * 1e-3),
               "algorithmic_tflops": 3.0 * flop_fwd / (float(np.median(ms)) * 1e-3) / 1e12}
        row["grad_vs_fp32"] = deviation("fp32_rerun" if e == "fp32" else e)
        rows.append(row)
        print(json.dumps(row))
    base = float(np.median(step_ms["fp32"]))
    summary = {"device": torch.cuda.get_device_name(dev), "nvidia_smi": gpu, "workload": plan,
               "speedup_vs_fp32": {e: base / float(np.median(step_ms[e])) for e in ENGINES}}
    print(json.dumps(summary))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_train.json"), "w") as f:
            json.dump({"rows": rows, "summary": summary}, f, indent=1)


if __name__ == "__main__":
    main()
