"""Timing of the novel-view colour metrics (csrc/color_metrics.cu, DESIGN.md 6.8) against the same work on the host.

    python tools/bench_color.py [--runs 20] [--host-runs 3] [--out DIR]

Device rows (CUDA events, median of --runs after warm-up, inputs already on the device), at 124x407 (KITTI's render) and
480x640 (BundleFusion's):
  * PSNR + SSIM of one pair (srf_psnr_ssim: two launches);
  * LPIPS-VGG of one pair (srf_lpips_vgg, random weights: the time does not depend on them), with the achieved TFLOP/s
    of the 26 convolutions from shape-computed FLOPs (VGG16 features[0:30]: 30.0 GFLOP per 124x407 image, 187.9 GFLOP
    per 480x640 image, two images per pair).
Host rows (wall clock, median of --host-runs): the scipy/numpy oracle of PSNR + SSIM (oracle/color_oracle.py, the
algorithm of skimage 0.18.1), and LPIPS-VGG as a torch float32 network on the CPU -- each named as such.
Prints one JSON line per row and the card's name, power limit and maximum SM clock, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import color_oracle as O  # noqa: E402
from scenerf_b200 import evaluation as E  # noqa: E402
from scenerf_b200.perceptual import LPIPSVGG  # noqa: E402
from test_color_eval import u8_image  # noqa: E402

SHAPES = ((124, 407), (480, 640))


def vgg_flops(h, w):
    """2 * 9 * Cin * Cout * H * W over the 13 convolutions of VGG16 features[0:30] (floor pooling), one image."""
    stages = ((2, 64), (2, 128), (3, 256), (3, 512), (3, 512))
    f, cin = 0, 3
    for s, (n, c) in enumerate(stages):
        if s:
            h, w = h // 2, w // 2
        for _ in range(n):
            f += 2 * 9 * cin * c * h * w
            cin = c
    return f


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    f = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")] if q.returncode == 0 and q.stdout.strip() else []
    return {"gpu": f[0] if f else torch.cuda.get_device_name(), "power_limit": f[1] if len(f) > 1 else None,
            "max_sm_clock": f[2] if len(f) > 2 else None}


def time_device(fn, runs):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def time_host(fn, runs):
    ts = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def torch_cpu_lpips(sd):
    """LPIPS-VGG as a float32 torch network on the CPU (the reference's network, minus CUDA)."""
    orc = O.LPIPSOracle(sd)
    feats = orc.features.float()
    lins = [l.float() for l in orc.lins]
    shift, scale = orc.shift.float(), orc.scale.float()

    @torch.no_grad()
    def run(a, b):
        x = [((torch.from_numpy(t).permute(2, 0, 1)[None] - 0.5) * 2 - shift) / scale for t in (a, b)]
        v = 0.0
        taps = [[], []]
        for k in range(2):
            y = x[k]
            for i, m in enumerate(feats):
                y = m(y)
                if i in O.TAPS:
                    taps[k].append(y)
        for f0, f1, lin in zip(taps[0], taps[1], lins):
            n0 = f0 / (f0.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            n1 = f1 / (f1.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            v += float(((n0 - n1) ** 2 * lin).sum(1).mean())
        return v
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--host-runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_color.py needs a CUDA device")
    info = card()
    print(json.dumps(info), flush=True)
    sd = O.random_lpips_state_dict(7)
    net = LPIPSVGG(sd, "cuda:0")
    cpu_lpips = torch_cpu_lpips(sd)
    rows = []
    for h, w in SHAPES:
        img, gt = u8_image(h, w, 1), u8_image(h, w, 2)
        di, dg = torch.from_numpy(img).cuda(), torch.from_numpy(gt).cuda()
        b = E.ColorErrorBuckets("kitti")
        rows.append({"row": "psnr+ssim %dx%d per pair" % (h, w), "device_ms": time_device(lambda: b.add(di, dg, 1.0), a.runs),
                     "host_ms": time_host(lambda: (O.psnr(img, gt), O.ssim(img, gt)), a.host_runs),
                     "host_impl": "scipy/numpy oracle (skimage 0.18.1 algorithm)"})
        ms = time_device(lambda: net(di, dg), a.runs)
        gflop = 2 * vgg_flops(h, w) / 1e9
        rows.append({"row": "lpips-vgg %dx%d per pair" % (h, w), "device_ms": ms, "conv_gflop": round(gflop, 1),
                     "achieved_tflops": round(gflop / ms, 1), "launches": net.launches,
                     "host_ms": time_host(lambda: cpu_lpips(img, gt), a.host_runs), "host_impl": "torch float32 CPU (%d threads)"
                     % torch.get_num_threads()})
    for r in rows:
        r.update(info)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_color.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
