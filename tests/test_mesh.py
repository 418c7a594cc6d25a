"""Mesh extraction from the TSDF volume (csrc/mesh.cu, DESIGN.md 6.6).  CPU tests: the oracle's topology on analytic
fields, its vertices against an independent pass over the edge arrays, and its get_mesh / get_point_cloud against the
golden made by the reference's own TSDFVolume post-processing.  GPU tests: the CUDA path equals the oracle and the
golden bit for bit, arrays and order."""
import ctypes as C
from collections import Counter

import numpy as np
import pytest

from cases import load_golden
from oracle import mesh_oracle as M
from oracle.tsdf_oracle import TSDFVolumeOracle
from scenerf_b200 import _lib


def sphere_field(n=32, r=10.0, c=15.3):
    g = np.mgrid[0:n, 0:n, 0:n].astype(np.float32)
    return (np.sqrt(((g - np.float32(c)) ** 2).sum(0)) - np.float32(r)).astype(np.float32)


def torus_field(n=32, R=9.0, r=3.5):
    x, y, z = np.mgrid[0:n, 0:n, 0:n].astype(np.float64) - (n - 1) / 2.0
    return (np.sqrt((np.sqrt(x * x + y * y) - R) ** 2 + z * z) - r).astype(np.float32)


def trilinear_noise(seed=0, coarse=12, up=2):
    """Coarse Gaussian noise upsampled trilinearly: saddles inside the coarse cells put many ambiguous faces on the fine
    grid.  The border is set outside so that the surface is closed."""
    g = np.random.default_rng(seed).standard_normal((coarse,) * 3)
    t = np.linspace(0, coarse - 1, (coarse - 1) * up + 1)
    i0 = np.minimum(np.floor(t).astype(int), coarse - 2)
    fr = t - i0
    for ax in range(3):
        a = np.moveaxis(g, ax, 0)
        g = np.moveaxis(a[i0] * (1 - fr)[:, None, None] + a[i0 + 1] * fr[:, None, None], 0, ax)
    v = g.astype(np.float32)
    v[0] = v[-1] = v[:, 0] = v[:, -1] = v[:, :, 0] = v[:, :, -1] = 1.0
    return v


def ambiguous_faces(v):
    s = v < 0
    n = 0
    for a, b in ((0, 1), (0, 2), (1, 2)):
        w = np.moveaxis(s, (a, b), (0, 1))
        c00, c10, c11, c01 = w[:-1, :-1], w[1:, :-1], w[1:, 1:], w[:-1, 1:]
        n += int(((c00 == c11) & (c10 == c01) & (c00 != c10)).sum())
    return n


def edge_counts(faces):
    e = Counter()
    for a, b, c in faces.tolist():
        e[(a, b)] += 1
        e[(b, c)] += 1
        e[(c, a)] += 1
    return e


def assert_closed_oriented(faces):
    """Every directed edge once and its reverse once: watertight and consistently oriented."""
    e = edge_counts(faces)
    bad = [k for k, n in e.items() if n != 1 or e.get((k[1], k[0])) != 1]
    assert not bad, bad[:5]
    return e


def euler(verts, faces):
    und = {tuple(sorted(k)) for k in edge_counts(faces)}
    return len(verts) - len(und) + len(faces)


# ---------------------------------------------------------------------------------------------------- CPU: oracle
def test_oracle_sphere_closed_genus0_area():
    v, f, n, _ = M.marching_cubes(sphere_field())
    assert_closed_oriented(f)
    assert euler(v, f) == 2
    a = v[f[:, 1]] - v[f[:, 0]]
    b = v[f[:, 2]] - v[f[:, 0]]
    area = 0.5 * np.linalg.norm(np.cross(a.astype(np.float64), b.astype(np.float64)), axis=1).sum()
    assert abs(area / (4 * np.pi * 10.0 ** 2) - 1) < 0.02          # marching cubes cuts corners: within 2 % of 4 pi r^2


def test_oracle_torus_genus1():
    v, f, _, _ = M.marching_cubes(torus_field())
    assert_closed_oriented(f)
    assert euler(v, f) == 0


def test_oracle_trilinear_noise_interior_edges_shared_twice():
    vol = trilinear_noise()
    assert ambiguous_faces(vol) > 100
    v, f, _, _ = M.marching_cubes(vol)
    assert_closed_oriented(f)
    # without the outside border the surface is open, and its boundary edges lie on the volume faces only
    inner = vol[1:-1, 1:-1, 1:-1]
    v, f, _, _ = M.marching_cubes(inner)
    e = edge_counts(f)
    shape = np.array(inner.shape) - 1
    for (a, b), k in e.items():
        assert k == 1
        if e.get((b, a)) != 1:
            pa, pb = v[a], v[b]
            assert any((pa[d] == pb[d]) and pa[d] in (0, shape[d]) for d in range(3)), (pa, pb)


def test_oracle_vertices_are_the_edge_crossings():
    vol = trilinear_noise(seed=3)
    v, _, _, _ = M.marching_cubes(vol)
    X, Y, Z = vol.shape
    rows = []
    for a in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, -1), slice(1, None)
        f0, f1 = vol[tuple(lo)], vol[tuple(hi)]
        idx = np.argwhere((f0 < 0) != (f1 < 0))
        t = f0[tuple(idx.T)] / (f0[tuple(idx.T)] - f1[tuple(idx.T)])
        pos = idx.astype(np.float32)
        pos[:, a] += t
        key = (idx[:, 0] * Y + idx[:, 1]) * Z + idx[:, 2]
        rows.append((key * 3 + a, pos))
    keys = np.concatenate([r[0] for r in rows])
    pos = np.concatenate([r[1] for r in rows])[np.argsort(keys, kind="stable")]
    assert pos.dtype == np.float32 and np.array_equal(pos, v)


def test_oracle_orientation_follows_gradient():
    vol = sphere_field()
    v, f, n, _ = M.marching_cubes(vol)
    fn = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    grad = (v[f].mean(1) - np.float32(15.3))                       # +grad of |x - c| - r
    assert ((fn * grad).sum(1) > 0).mean() >= 0.99
    assert ((n[f].mean(1) * grad).sum(1) > 0).mean() >= 0.99
    assert np.allclose(np.linalg.norm(n, axis=1), 1.0, atol=1e-5)


def golden_frames():
    """The three frames the tsdf_mesh golden volume was fused from (those of the tsdf_fusion case)."""
    f = load_golden("tsdf_fusion")
    return f["K"], [(f["rgb%d" % i], f["depth%d" % i], f["pose%d" % i]) for i in range(3)]


def test_oracle_matches_reference_postprocessing_golden():
    g = load_golden("tsdf_mesh")
    K, frames = golden_frames()
    o = TSDFVolumeOracle(g["vol_bnds"], 0.2, 10)                     # the golden's volume is the reference's fusion
    for rgb, depth, pose in frames:
        o.integrate(rgb, depth, K, pose, 1.0)
    assert np.array_equal(o.tsdf, g["tsdf"]) and np.array_equal(o.color, g["color"])
    origin = g["vol_bnds"][:, 0].astype(np.float32)
    assert len(g["faces"]) > 1000 and len(g["mfaces"]) > 1000
    got = M.get_mesh(g["tsdf"], g["color"], origin, 0.2)
    for k, a in zip(("verts", "faces", "norms", "colors"), got):
        assert a.dtype == g[k].dtype and np.array_equal(a, g[k]), k
    got = M.get_mesh(g["tsdf"], g["color"], origin, 0.2, g["mask"])
    for k, a in zip(("mverts", "mfaces", "mnorms", "mcolors"), got):
        assert a.dtype == g[k].dtype and np.array_equal(a, g[k]), k
    pv, pc = M.get_point_cloud(g["tsdf"], g["color"], origin, 0.2)
    assert np.array_equal(pv, g["verts"]) and np.array_equal(pc, g["colors"])     # fusion.py:333-354: get_mesh's vertices


def test_mesh_abi_rejects_bad_arguments_without_gpu():
    lib = _lib.load()
    nv, nf = C.c_longlong(-1), C.c_longlong(-1)
    dims = (C.c_int * 3)(8, 8, 0)
    assert lib.srf_tsdf_mesh_count_host(None, None, dims, None, 0, C.byref(nv), C.byref(nf), None) == 1
    assert b"srf_tsdf_mesh_count_host" in lib.srf_last_error()
    assert lib.srf_tsdf_mesh_workspace_bytes(dims) == 0
    huge = (C.c_int * 3)(4096, 4096, 4096)
    assert lib.srf_tsdf_mesh_count_host(None, None, huge, None, 0, C.byref(nv), C.byref(nf), None) == 1
    assert b"int32" in lib.srf_last_error()
    dims = (C.c_int * 3)(8, 8, 4)
    need = lib.srf_tsdf_mesh_workspace_bytes(dims)
    assert need >= 8 * 8 * 4 * 9
    assert lib.srf_tsdf_mesh_count_host(None, None, dims, None, need, C.byref(nv), C.byref(nf), None) == 1
    assert lib.srf_tsdf_mesh_count_host(16, None, dims, 256, need - 1, C.byref(nv), C.byref(nf), None) == 2
    assert b"workspace" in lib.srf_last_error()
    origin = (C.c_float * 3)(0, 0, 0)
    assert lib.srf_tsdf_mesh_emit(16, None, None, dims, origin, 0.2, 256, need, 256, None, 256, None, None) == 1
    assert b"srf_tsdf_mesh_emit" in lib.srf_last_error()
    assert lib.srf_tsdf_mesh_emit(16, 16, None, dims, origin, 0.2, 256, need - 1, 256, None, None, None, None) == 2
    flat = (C.c_int * 3)(8, 1, 4)                                    # a dimension of 1: empty mesh, no device call
    assert lib.srf_tsdf_mesh_count_host(16, None, flat, None, 0, C.byref(nv), C.byref(nf), None) == 0
    assert nv.value == 0 and nf.value == 0


# ---------------------------------------------------------------------------------------------------- GPU
def volume_with(tsdf, color=None, origin=(0.0, -6.4, -2.0), voxel=0.2):
    """A TSDFVolume holding the given arrays (merged into the reset volume: exact for |tsdf| <= 255)."""
    import torch
    from scenerf_b200.tsdf import TSDFVolume
    assert np.abs(tsdf).max() <= 255
    shape = np.array(tsdf.shape)
    bnds = np.zeros((3, 2))
    bnds[:, 0] = origin
    bnds[:, 1] = bnds[:, 0] + (shape - 0.5) * voxel
    vol = TSDFVolume(bnds, voxel_size=voxel)
    assert tuple(vol._vol_dim) == tsdf.shape
    color = np.zeros_like(tsdf) if color is None else color
    vol.merge_(torch.from_numpy(tsdf), torch.ones(tsdf.shape), torch.from_numpy(color.astype(np.float32)))
    assert np.array_equal(vol.get_volume()[0], tsdf)
    return vol


def assert_same(got, want, names):
    for k, a, b in zip(names, got, want):
        assert a.dtype == b.dtype and a.shape == b.shape, (k, a.dtype, b.dtype, a.shape, b.shape)
        assert np.array_equal(a, b), (k, int((a != b).sum()))


def check_vol(vol, mask=None):
    """CUDA get_mesh / get_mesh(mask) / get_point_cloud == the oracle on the volume's own arrays."""
    tsdf, color = vol.get_volume()
    origin, vs = vol._vol_origin, vol._voxel_size
    names = ("verts", "faces", "norms", "colors")
    got = vol.get_mesh()
    assert_same(got, M.get_mesh(tsdf, color, origin, vs), names)
    if mask is not None:
        assert_same(vol.get_mesh(mask), M.get_mesh(tsdf, color, origin, vs, mask), names)
        assert np.array_equal(vol.get_volume()[0], tsdf)                 # the mask does not write into the volume
    assert_same(vol.get_point_cloud(), M.get_point_cloud(tsdf, color, origin, vs), ("verts", "colors"))
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("mask_as", ["numpy", "tensor"])
def test_cuda_mesh_matches_reference_golden(mask_as):
    import torch
    from scenerf_b200.tsdf import TSDFVolume
    g = load_golden("tsdf_mesh")
    K, frames = golden_frames()
    vol = TSDFVolume(g["vol_bnds"].copy(), voxel_size=0.2, trunc_margin=10)
    for rgb, depth, pose in frames:
        vol.integrate(torch.from_numpy(rgb).cuda(), torch.from_numpy(depth).cuda(), K, pose)
    assert np.array_equal(vol.get_volume()[0], g["tsdf"])
    assert_same(vol.get_point_cloud(), (g["verts"], g["colors"]), ("verts", "colors"))
    assert_same(vol.get_mesh(), (g["verts"], g["faces"], g["norms"], g["colors"]), ("verts", "faces", "norms", "colors"))
    mask = g["mask"] if mask_as == "numpy" else torch.from_numpy(g["mask"]).cuda()
    assert_same(vol.get_mesh(mask), (g["mverts"], g["mfaces"], g["mnorms"], g["mcolors"]),
                ("verts", "faces", "norms", "colors"))
    assert np.array_equal(vol.get_volume()[0], g["tsdf"])
    check_vol(vol, g["mask"])


@pytest.mark.gpu
def test_cuda_mesh_analytic_fields():
    rng = np.random.default_rng(4)
    for field, closed_chi in ((sphere_field(), 2), (torus_field(), 0), (trilinear_noise(), None)):
        color = np.floor(rng.random(field.shape) * 2 ** 24).astype(np.float32)
        vol = volume_with(field, color)
        v, f, _, _ = check_vol(vol, rng.random(field.shape) > 0.05)
        assert_closed_oriented(f)
        if closed_chi is not None:
            assert euler(v, f) == closed_chi


def kitti_volume():
    import torch
    from scenerf_b200.tsdf import TSDFVolume
    from scenerf_b200 import synth
    vol_bnds = np.zeros((3, 2)); vol_bnds[:, 0] = [0, -25.6, -2]; vol_bnds[:, 1] = vol_bnds[:, 0] + [51.2, 51.2, 6.4]
    T_velo2cam = np.array([[0.0, -1.0, 0.0, 0.0], [0.0, 0.0, -1.0, -0.08], [1.0, 0.0, 0.0, -0.27], [0, 0, 0, 1.0]])
    H, W = 370, 1220
    vol = TSDFVolume(vol_bnds, voxel_size=0.2)
    for i, (yaw, tz) in enumerate(((0.0, 0.0), (10.0, 2.0), (-10.0, 4.0))):
        depth = torch.from_numpy((5.0 + 30.0 * synth.hash_unit(80 + i, H * W)).reshape(H, W).astype(np.float32)).cuda()
        rgb = torch.from_numpy(np.floor(synth.hash_unit(90 + i, H * W * 3) * 256).reshape(H, W, 3).astype(np.float32)).cuda()
        vol.integrate(rgb, depth, synth.KITTI_K, np.linalg.inv(T_velo2cam) @ synth.yaw_translate(yaw, tz).astype(np.float64))
    return vol


@pytest.mark.gpu
def test_cuda_mesh_full_kitti_volume():
    vol = kitti_volume()
    assert vol.get_volume()[0].shape == (256, 256, 32)
    mask = np.random.default_rng(5).random((256, 256, 32)) > 0.02
    v, f, _, _ = check_vol(vol, mask)
    assert len(f) > 10000


@pytest.mark.gpu
def test_cuda_mesh_bf_volume():
    import torch
    from scenerf_b200.tsdf import TSDFVolume
    from scenerf_b200 import synth
    vol_bnds = np.array([[-3.0, 3.0], [-3.0, 3.0], [0.0, 4.8]])                   # 120 x 120 x 96 at 5 cm
    vol = TSDFVolume(vol_bnds, voxel_size=0.05, trunc_margin=10)
    H, W = 480, 640
    for i, (yaw, tz) in enumerate(((0.0, 0.0), (15.0, 0.4), (-15.0, 0.2))):
        depth = torch.from_numpy((0.5 + 4.0 * synth.hash_unit(110 + i, H * W)).reshape(H, W).astype(np.float32)).cuda()
        rgb = torch.from_numpy(np.floor(synth.hash_unit(120 + i, H * W * 3) * 256).reshape(H, W, 3).astype(np.float32)).cuda()
        vol.integrate(rgb, depth, synth.BF_K, synth.yaw_translate(yaw, tz).astype(np.float64))
    assert vol.get_volume()[0].shape == (120, 120, 96)
    v, f, _, _ = check_vol(vol, np.random.default_rng(6).random((120, 120, 96)) > 0.02)
    assert len(f) > 10000


@pytest.mark.gpu
def test_cuda_mesh_empty_and_flat_volumes():
    from scenerf_b200.tsdf import TSDFVolume
    vol = TSDFVolume(np.array([[0, 1.6], [0, 1.6], [0, 0.8]]), voxel_size=0.2)         # all 255: nothing observed
    v, f, n, c = vol.get_mesh()
    assert v.shape == (0, 3) and v.dtype == np.float32 and f.shape == (0, 3) and f.dtype == np.int32
    assert n.shape == (0, 3) and n.dtype == np.float32 and c.shape == (0, 3) and c.dtype == np.uint8
    pv, pc = vol.get_point_cloud()
    assert pv.shape == (0, 3) and pc.shape == (0, 3) and pc.dtype == np.uint8
    flat = np.full((6, 1, 5), -1.0, np.float32)
    flat[2:, :, :] = 1.0
    v, f, n, c = volume_with(flat).get_mesh()
    assert len(v) == 0 and len(f) == 0 and f.shape == (0, 3)


@pytest.mark.gpu
def test_depth2tsdf_sequence_and_sweep_volume():
    """depth2tsdf.py:93-107: construct, integrate, get_volume, get_mesh with scenerf_b200.tsdf.TSDFVolume; then a small
    NovelDepthSweep.reconstruct volume meshes like the oracle, into a surface whose interior edges are shared by exactly
    two faces."""
    import torch
    from scenerf_b200 import sweep
    from scenerf_b200.tsdf import TSDFVolume
    g = load_golden("tsdf_mesh")
    K, frames = golden_frames()
    tsdf_vol = TSDFVolume(g["vol_bnds"].copy(), voxel_size=0.2)
    for rgb, depth, pose in frames:
        tsdf_vol.integrate(rgb, depth, K, pose, obs_weight=1.)
    tsdf_grid, _ = tsdf_vol.get_volume()
    verts, faces, norms, colors = tsdf_vol.get_mesh()
    assert np.array_equal(tsdf_grid, g["tsdf"]) and np.array_equal(faces, g["faces"])

    from test_sweep import _renderer                                             # the small sweep of test_sweep.py
    sg = load_golden("sweep_kitti")
    cfg, r, x_rgb = _renderer("fp32")
    sw = sweep.NovelDepthSweep(r, torch.from_numpy(cfg.K).cuda(), x_rgb, img_size=(244, 74), scale=4)
    poses = sweep.sample_rel_poses(step=1.0, angle=10, max_distance=1.1)
    vol = sw.reconstruct(poses, sg["T_velo2cam"], sg["vol_bnds"])
    v, f, _, _ = check_vol(vol)
    e = edge_counts(f)
    shape = np.array(vol.get_volume()[0].shape) - 1
    vi = (v - vol._vol_origin) / np.float32(vol._voxel_size)
    for (a, b), k in e.items():
        assert k == 1
        if e.get((b, a)) != 1:                                                   # open only at the volume border
            assert any(np.isclose(vi[a][d], vi[b][d]) and min(abs(vi[a][d]), abs(vi[a][d] - shape[d])) < 1e-3 for d in range(3))
