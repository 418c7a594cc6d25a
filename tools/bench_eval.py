"""Timing of the device evaluation metrics (csrc/metrics.cu, DESIGN.md 6.7) against the same work on the host.

    python tools/bench_eval.py [--runs 20] [--out DIR]

Device rows (CUDA events, median of --runs after warm-up, inputs already on the device):
  * score_reconstruction_kitti on a KITTI-size 256x256x32 volume: occupancy, crop, whole-scene and FOV counts
    (eval_sr.py:79-87), including the one 4-byte read of max_z;
  * tsdf2occ_bf + SSCMetrics.add_batch on a BundleFusion-size 120x120x96 volume (eval_sc_bf.py:203-210);
  * DepthErrorBuckets.add on a 20 k-ray (gt, pred) pair (save_depth_metrics.py:122-131; no synchronisation).
Host rows (wall clock, median of fewer runs): the same work through the reference's own SSCMetrics and
compute_depth_errors when the reference tree is importable, otherwise through oracle/eval_oracle.py (named in the row).
Prints one JSON line per row and the card's name, power limit and maximum SM clock."""
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

import eval_cases as EC  # noqa: E402
from oracle import eval_oracle as O  # noqa: E402
from scenerf_b200 import evaluation as E  # noqa: E402


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


def host_impl():
    """The reference's SSCMetrics / compute_depth_errors where importable, else the oracle's restatement."""
    ref = os.environ.get("SCENERF_REFERENCE", "/root/reference")
    if os.path.isdir(os.path.join(ref, "scenerf")):
        sys.path.insert(0, ref)
        try:
            from scenerf.loss.sscMetrics import SSCMetrics
            from scenerf.loss.depth_metrics import compute_depth_errors
            return "reference", SSCMetrics, compute_depth_errors
        except ImportError:
            pass
    return "oracle", O.SSCMetricsOracle, O.compute_depth_errors


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--host-runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py needs a CUDA device")
    rows = []
    info = card()
    print(json.dumps(info), flush=True)

    tsdf = EC.tsdf_volume(EC.KITTI_SHAPE, 300, E.th_table_kitti(256), 0)
    target, fov = EC.labels(EC.KITTI_SHAPE, 301, top_z=20), EC.fov_mask(EC.KITTI_SHAPE, 303)
    d_tsdf, d_target, d_fov = (torch.from_numpy(x).cuda() for x in (tsdf, target, fov))
    m, fm = E.SSCMetrics(2), E.SSCMetrics(2)
    rows.append({"row": "kitti 256x256x32 score_reconstruction_kitti", "device_ms":
                 time_device(lambda: E.score_reconstruction_kitti(d_tsdf, d_target, d_fov, m, fm), a.runs)})

    tsdf_bf, target_bf = EC.tsdf_volume(EC.BF_SHAPE, 310, E.th_table_bf(96, 0.04, 0.1, 0.4, 0.04), 2), EC.labels(EC.BF_SHAPE, 311)
    d_bf, d_tbf = torch.from_numpy(tsdf_bf).cuda(), torch.from_numpy(target_bf).cuda()
    mb = E.SSCMetrics(2)
    rows.append({"row": "bf 120x120x96 tsdf2occ_bf + add_batch", "device_ms":
                 time_device(lambda: mb.add_batch(E.tsdf2occ_bf(d_bf, 0.04, 0.1, 0.4, 0.04), d_tbf), a.runs)})

    gt, pred = EC.depth_pair(0, 20000)
    d_gt, d_pred = torch.from_numpy(gt).cuda(), torch.from_numpy(pred).cuda()
    b = E.DepthErrorBuckets()
    rows.append({"row": "depth errors 20k rays (bucket add)", "device_ms": time_device(lambda: b.add(d_gt, d_pred, 1.5), a.runs)})

    which, SSC, cde = host_impl()

    def host_kitti():
        hm, hfm = SSC(2), SSC(2)
        t = np.copy(target)
        t[target == 255] = 0
        max_z = t.nonzero()[2].max()
        occ = O.tsdf2occ(tsdf, O.th_table_kitti(256), 0)
        occ[:, :, max_z:] = 0
        hm.add_batch(occ, target)
        hfm.add_batch(occ, target, fov)

    def host_bf():
        SSC(2).add_batch(O.tsdf2occ(tsdf_bf, O.th_table_bf(96, 0.04, 0.1, 0.4, 0.04), 2), target_bf)

    rows[0]["host_ms"] = time_host(host_kitti, a.host_runs)
    rows[1]["host_ms"] = time_host(host_bf, a.host_runs)
    rows[2]["host_ms"] = time_host(lambda: cde(gt.copy(), pred.copy()), max(a.host_runs, 20))
    for r in rows:
        r["host_impl"] = which
        r.update(info)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_eval.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
