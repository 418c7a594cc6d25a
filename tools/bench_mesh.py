"""Timing of the device mesh extraction (csrc/mesh.cu) on fused volumes of the reference's two reconstruction sizes:
KITTI 256x256x32 at 0.2 m (depth2tsdf.py:87-93) and BundleFusion 120x120x96 at 5 cm (depth2tsdf_bf.py:92-100), each
fused with TSDFVolume.integrate from seeded synthetic depth: a structured scene (ground plane + boxes) and hash noise.

    python tools/bench_mesh.py --out DIR [--runs 20]

Reports vertex / face counts, the device time of count + emit (CUDA events, median of --runs after warm-up), the
end-to-end get_mesh() wall time including the device-to-host copies, and the numpy oracle's time (a CPU figure).
There is no skimage figure: scikit-image is not a dependency, and its marching_cubes_lewiner was never timed here."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import mesh_oracle  # noqa: E402
from scenerf_b200 import _lib, synth  # noqa: E402
from scenerf_b200.tsdf import TSDFVolume  # noqa: E402

T_VELO2CAM = np.array([[0.0, -1.0, 0.0, 0.0], [0.0, 0.0, -1.0, -0.08], [1.0, 0.0, 0.0, -0.27], [0, 0, 0, 1.0]])


def scene_depth(K, H, W, cam_height, box_seed):
    """Ray-cast depth of a ground plane cam_height below the camera plus 6 seeded axis-aligned boxes (camera frame:
    x right, y down, z forward)."""
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    d = np.stack([(u - K[0, 2]) / K[0, 0], (v - K[1, 2]) / K[1, 1], np.ones_like(u)], -1)
    depth = np.where(d[..., 1] > 1e-6, cam_height / np.maximum(d[..., 1], 1e-6), 0.0)
    rng = np.random.default_rng(box_seed)
    zmax = depth.max() if depth.max() > 0 else 30.0
    for _ in range(6):
        c = np.array([rng.uniform(-0.4, 0.4), 0.0, rng.uniform(0.2, 0.8)]) * np.array([zmax * 0.5, 1, zmax * 0.6])
        half = np.array([rng.uniform(0.05, 0.15), 0.5, rng.uniform(0.05, 0.15)]) * np.array([zmax * 0.3, cam_height, zmax * 0.3])
        c[1] = cam_height - half[1]
        lo, hi = c - half, c + half
        with np.errstate(divide="ignore", invalid="ignore"):
            t0, t1 = lo / d, hi / d
        tn = np.nanmax(np.minimum(t0, t1), -1)
        tf = np.nanmin(np.maximum(t0, t1), -1)
        hit = (tn <= tf) & (tn > 0)
        depth = np.where(hit & ((depth == 0) | (tn < depth)), tn, depth)
    return depth.astype(np.float32)


def fused_volume(kind, scene, seed):
    if kind == "kitti":
        bnds = np.zeros((3, 2)); bnds[:, 0] = [0, -25.6, -2]; bnds[:, 1] = bnds[:, 0] + [51.2, 51.2, 6.4]
        vol, K, H, W, base, h = TSDFVolume(bnds, voxel_size=0.2), synth.KITTI_K, 370, 1220, np.linalg.inv(T_VELO2CAM), 1.73
        zr = (5.0, 30.0)
    else:
        bnds = np.array([[-3.0, 3.0], [-3.0, 3.0], [0.0, 4.8]])
        vol, K, H, W, base, h = TSDFVolume(bnds, voxel_size=0.05), synth.BF_K, 480, 640, np.eye(4), 1.2
        zr = (0.5, 4.0)
    for i, (yaw, tz) in enumerate(((0.0, 0.0), (10.0, 1.0), (-10.0, 2.0))):
        if scene == "structured":
            depth = scene_depth(K, H, W, h, seed + i)
        else:
            depth = (zr[0] + zr[1] * synth.hash_unit(seed + i, H * W)).reshape(H, W).astype(np.float32)
        rgb = np.floor(synth.hash_unit(seed + 50 + i, H * W * 3) * 256).reshape(H, W, 3).astype(np.float32)
        pose = base @ synth.yaw_translate(yaw, tz * (0.2 if kind == "bf" else 1.0)).astype(np.float64)
        vol.integrate(torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda(), K, pose)
    return vol


def device_ms(vol, runs):
    """Median device time of count + emit (CUDA events on the current stream)."""
    lib = vol.lib
    st = torch.cuda.current_stream()
    sp = C.c_void_p(st.cuda_stream)
    wsb = lib.srf_tsdf_mesh_workspace_bytes(vol._dims)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    nv, nf = C.c_longlong(0), C.c_longlong(0)
    _lib.check(lib.srf_tsdf_mesh_count_host(vol._tsdf.data_ptr(), None, vol._dims, ws.data_ptr(), wsb, C.byref(nv), C.byref(nf), sp))
    verts = torch.empty((nv.value, 3), device="cuda")
    norms = torch.empty((nv.value, 3), device="cuda")
    cols = torch.empty((nv.value, 3), dtype=torch.uint8, device="cuda")
    faces = torch.empty((nf.value, 3), dtype=torch.int32, device="cuda")
    origin = (C.c_float * 3)(*[float(v) for v in vol._vol_origin])
    times = []
    for r in range(runs + 3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(st)
        _lib.check(lib.srf_tsdf_mesh_count_host(vol._tsdf.data_ptr(), None, vol._dims, ws.data_ptr(), wsb, C.byref(nv),
                                                C.byref(nf), sp))
        _lib.check(lib.srf_tsdf_mesh_emit(vol._tsdf.data_ptr(), vol._color.data_ptr(), None, vol._dims, origin, vol._voxel_size,
                                          ws.data_ptr(), wsb, verts.data_ptr(), norms.data_ptr(), cols.data_ptr(),
                                          faces.data_ptr(), sp))
        b.record(st)
        b.synchronize()
        if r >= 3:
            times.append(a.elapsed_time(b))
    return float(np.median(times)), times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--runs", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh needs a CUDA device")
    os.makedirs(args.out, exist_ok=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True).stdout.strip()
    res = {"gpu": q, "runs": args.runs, "cases": []}
    for kind in ("kitti", "bf"):
        for scene, seed in (("structured", 300), ("noise", 400)):
            vol = fused_volume(kind, scene, seed)
            med, times = device_ms(vol, args.runs)
            walls = []
            for _ in range(5):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                v, f, n, c = vol.get_mesh()
                walls.append((time.perf_counter() - t0) * 1e3)
            tsdf, color = vol.get_volume()
            t0 = time.perf_counter()
            ov, of, on, oc = mesh_oracle.get_mesh(tsdf, color, vol._vol_origin, vol._voxel_size)
            cpu_ms = (time.perf_counter() - t0) * 1e3
            same = all(np.array_equal(x, y) for x, y in ((v, ov), (f, of), (n, on), (c, oc)))
            row = {"volume": kind, "dims": [int(d) for d in vol._vol_dim], "scene": scene, "verts": int(len(v)),
                   "faces": int(len(f)), "device_count_emit_ms_median": med, "device_ms_min": float(min(times)),
                   "device_ms_max": float(max(times)), "get_mesh_wall_ms_median": float(np.median(walls)),
                   "oracle_numpy_cpu_ms": cpu_ms, "equals_oracle": bool(same)}
            res["cases"].append(row)
            print(json.dumps(row))
    with open(os.path.join(args.out, "bench_mesh.json"), "w") as fh:
        json.dump(res, fh, indent=1)
    print(json.dumps({"gpu": q}))


if __name__ == "__main__":
    main()
