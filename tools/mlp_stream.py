#!/usr/bin/env python
"""Weight-stream rate of the main point-MLP pass (point_mlp_tc_kernel) on config B's points, fp32tc and fp16.

    python tools/mlp_stream.py [--steps 5] [--warmup 2] [--cluster 1] [--precisions fp32tc,fp16]

Renders config B (453 620 rays x 128 samples, dense, no latent table) with device-side timing of the main pass
(set_profiling / last_mlp_ms) and prints one JSON line per precision mode:
  * kernel_ms: median main-pass time over --steps renders after --warmup;
  * tiles: main-pass points / 64 points per tile (both modes);
  * l2_weight_bytes: the bytes of weight images read from L2 per pass.  Every tile streams the whole image region of
    the blob once, so the count is tiles * image bytes (divided by --cluster for a kernel in which a cluster of CTAs
    shares one L2 read of each image);
  * l2_weight_gbs: l2_weight_bytes / kernel time;
  * tensor_tflops: executed wgmma FLOP (m64n128k16 for the 512-wide layers, m64n16k16 for lin_out; in fp32tc four
    products per image pair: both A parts against the hi and the lo image) / kernel time;
  * the GPU's name, power limit and median SM clock, sampled by nvidia-smi during the timed renders.
--cluster is the number of CTAs that share one L2 read of each image in the library measured (1: the kernel here,
where every CTA streams its own copy)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HEADER_BYTES = 8 * 512 * 4            # bias header of a weight blob (csrc/mlp_tc.cu kHeaderBytes)
BLOB_SLACK = 256                      # tail of a blob (tc_weights_bytes)
IMG_BYTES = 128 * 128                 # one 128 x 64 fp16 weight image
OUT_IMG_BYTES = 16 * 128              # one 16 x 64 lin_out image
OUT_CHUNKS = 8


def gpu_info():
    q = subprocess.run(["nvidia-smi", "-i", str(_dev_index()), "--query-gpu=name,power.limit,clocks.max.sm",
                        "--format=csv,noheader,nounits"], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    f = [x.strip() for x in q.stdout.strip().split(",")] if q.returncode == 0 else []
    return {"gpu": f[0] if f else None, "power_limit_w": float(f[1]) if len(f) > 1 else None,
            "sm_max_mhz": float(f[2]) if len(f) > 2 else None}


def _dev_index():
    import torch
    return torch.cuda.current_device()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cluster", type=int, default=1)
    ap.add_argument("--precisions", default="fp32tc,fp16")
    args = ap.parse_args()

    import torch
    from bench import ClockSampler, hp_from_cfg, workload
    from scenerf_b200 import synth
    from scenerf_b200.renderer import B200Renderer
    if not torch.cuda.is_available():
        sys.exit("mlp_stream.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg, pix_np, _ = workload("B")
    pm, pg = synth.make_model_params(cfg)
    to_t = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
    gen = torch.Generator(device=dev)
    gen.manual_seed(5)
    x_rgb = {k: torch.randn((c, h, w), generator=gen, device=dev) * 0.5
             for k, (c, h, w) in zip(synth.SCALE_KEYS, synth.pyramid_shapes(cfg.sphere_W, cfg.sphere_H))}
    K, T = torch.from_numpy(cfg.K), torch.from_numpy(cfg.T)
    pix = torch.from_numpy(pix_np).to(dev)
    n_points = pix_np.shape[0] * cfg.S
    info = gpu_info()
    for prec in args.precisions.split(","):
        r = B200Renderer(hp_from_cfg(cfg), to_t(pm), to_t(pg), device=dev, precision=prec, rng="philox")
        split = prec == "fp32tc"
        blob = r.mlp.packed_split if split else r.mlp.packed
        parts = 2 if split else 1
        images = blob.numel() - HEADER_BYTES - BLOB_SLACK
        wide_chunks = (images // parts - OUT_CHUNKS * OUT_IMG_BYTES) // (4 * IMG_BYTES)   # K-chunks of the 512-wide layers
        tiles = -(-n_points // 64)
        products = 4 if split else 1                       # (A_hi, A_lo) x (W_hi, W_lo) in fp32tc
        flop_tile = products * (wide_chunks * 4 * 4 * (2 * 64 * 128 * 16) + OUT_CHUNKS * 4 * (2 * 64 * 16 * 16))
        r.set_profiling(True)
        for _ in range(args.warmup):
            r.render_rays_batch(K, T, x_rgb, sampled_pixels=pix, outputs="minimal")
        torch.cuda.synchronize()
        sampler = ClockSampler(_dev_index())
        sampler.start()
        ms = []
        for _ in range(args.steps):
            r.render_rays_batch(K, T, x_rgb, sampled_pixels=pix, outputs="minimal")
            ms.append(r.last_mlp_ms()[1])
        torch.cuda.synchronize()
        clocks = sampler.stop()
        kms = statistics.median(ms)
        l2_bytes = tiles * images / args.cluster
        print(json.dumps({
            "precision": prec, "kernel_ms": round(kms, 2), "kernel_ms_all": [round(m, 2) for m in ms],
            "tiles": tiles, "cluster": args.cluster, "image_bytes_per_tile": images,
            "l2_weight_bytes": l2_bytes, "l2_weight_gbs": round(l2_bytes / (kms * 1e-3) / 1e9, 1),
            "tensor_tflops": round(tiles * flop_tile / (kms * 1e-3) / 1e12, 1),
            **info, "sm_mhz_median": clocks["sm_mhz"], "clock_reasons": clocks["reasons"]}), flush=True)
        del r
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
