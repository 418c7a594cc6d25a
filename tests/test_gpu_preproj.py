"""GPU: pre-projected latents (B200Renderer(preproject=True), srf_build_latent_table; SURVEY 7 hard part 3b).

SphericalMapping.from_pixels rounds the sphere coordinates (spherical_mapping.py:115), so lin_z[b](z) (resnetfc.py:148-150)
is a function of the integer sphere pixel; the table holds it for every pixel with a valid tap and the kernel adds table rows
instead of running the three lin_z GEMM passes of the main network.  Exact in real arithmetic -- checked here against
  * the dense path of the same precision mode on adversarial points (corners of every scale, zero-padding boundary,
    behind-camera sentinel, out-of-grid points: the zero row),
  * the reference's goldens at the unchanged tolerances of the mode (small grids and the full-size config-B grid),
and the table itself row by row against float64 (every row of two small grids, edge rows and a 1 % sample of the
full-size config-B grid); the layer checks of the table variants of the kernel are in test_gpu_tc_layers.py and
test_gpu_fp32tc.py."""
import numpy as np
import pytest

from cases import FULL_CASES, PREDICT_CASES, RENDER_CASES, load_golden, pyramid_for
from helpers import make_renderer, torch_pyramid
from test_gpu_parity import _compare_with_golden

import tc_mlp_emul as E

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("prec,tol", [("fp32tc", 3e-5), ("fp16", 1e-2)])
@pytest.mark.parametrize("name", sorted(PREDICT_CASES))
def test_table_vs_dense_on_adversarial_points(name, prec, tol):
    import torch
    cfg, seed = PREDICT_CASES[name]
    g = load_golden(name)
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    args = (torch.from_numpy(g["cam_pts"]), x_rgb, K, None, torch.from_numpy(g["viewdir"]))
    dense = make_renderer(cfg, prec).predict("mlp", *args, output_type="offset").cpu().numpy()
    r = make_renderer(cfg, prec, preproject=True)
    tab = r.predict("mlp", *args, output_type="offset").cpu().numpy()
    assert r.last_pack_launches == 36                       # per network: 15 GEMMs + 3 blend kernels built its table
    err = float(np.abs(tab - dense).max())
    mag = float(max(1.0, np.abs(dense).max()))
    print("%s/%s: table vs dense raw-output max-abs-err %.3e (max |out| %.3e)" % (name, prec, err, mag))
    assert np.isfinite(tab).all() and err <= tol * mag
    # the gaussian-proposal network has its own table (its own lin_z weights)
    og = r.predict("mlp_gaussian", *args, output_type="offset").cpu().numpy()
    od = make_renderer(cfg, prec).predict("mlp_gaussian", *args, output_type="offset").cpu().numpy()
    assert np.abs(og - od).max() <= tol * float(max(1.0, np.abs(od).max()))


@pytest.mark.parametrize("prec", ["fp32tc", "fp16"])
@pytest.mark.parametrize("name", sorted(RENDER_CASES))
def test_render_with_table_vs_reference_golden(name, prec):
    cfg, seed = RENDER_CASES[name]
    _compare_with_golden(name + "+table", cfg, load_golden(name), prec, pyramid_for(cfg, seed), preproject=True)


def test_full_size_B_with_table_vs_reference_golden():
    """config B at full size (1226x370 grid: 455 k table rows, 2.8 GB fp32 / 1.4 GB fp16) against the reference's outputs."""
    from scenerf_b200 import synth
    cfg, seed = FULL_CASES["full_B"]
    g = load_golden("full_B")
    pyr = synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H)
    for prec in ("fp32tc", "fp16"):
        _compare_with_golden("full_B+table", cfg, g, prec, pyr, preproject=True)


# ---------------------------------------------------------------------------------------------------------------
# The table itself, row by row.  Row (sx, sy), block b:
#   T = sum_s sum_taps w_tap * Q_s[tap] + c_b,   Q_s = feat_s . W_z,b[:, scale s]^T   (float32 SIMT GEMMs)
# with the tap weights of the float32 tap arithmetic.  Bound per entry: each Q entry is within C_s 2^-24 sum|f||w|
# (the SIMT GEMM bound of test_gpu_gemm.py), carried through the blend weights, plus the blend's float32 roundings:
# every term passes at most 10 of them (1 product, 3 tap adds, 5 scale adds, the bias add).
# ---------------------------------------------------------------------------------------------------------------
_SCALES = ("1_1", "1_2", "1_4", "1_8", "1_16")


def _tap_arrays(cfg, pyr, s, sx, sy):
    """float32 tap arithmetic (oracle.sample_feats_2d): texel index (n,4), in-range (n,4), weights (n,4)."""
    f32 = np.float32
    _, H, W = pyr[_SCALES[s]].shape
    g = lambda c, nrm: ((c.astype(f32) / f32(nrm)).astype(f32) * f32(2) - f32(1)).astype(f32)
    ix = ((g(sx, cfg.sphere_W // (1 << s)) + f32(1)) * f32(W / 2.0) - f32(0.5)).astype(f32)
    iy = ((g(sy, cfg.sphere_H // (1 << s)) + f32(1)) * f32(H / 2.0) - f32(0.5)).astype(f32)
    xw, yn = np.floor(ix), np.floor(iy)
    w, n = (ix - xw).astype(f32), (iy - yn).astype(f32)
    e, so = (f32(1) - w).astype(f32), (f32(1) - n).astype(f32)
    x0, y0 = xw.astype(np.int64), yn.astype(np.int64)
    idx, ok, wt = [], [], []
    for dx, dy, wgt in ((0, 0, so * e), (1, 0, so * w), (0, 1, n * e), (1, 1, n * w)):
        xx, yy = x0 + dx, y0 + dy
        good = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        idx.append(np.where(good, yy * W + xx, 0))
        ok.append(good)
        wt.append(wgt.astype(f32))
    return np.stack(idx, 1), np.stack(ok, 1), np.stack(wt, 1)


def _check_table(cfg, pyr, params, hdr, tab, rows, label):
    """Per-entry check of the table rows `rows` (indices < W1*H1) of all three blocks; returns the worst err/bound."""
    import torch
    dev = tab.device
    W1 = cfg.sphere_W + 1
    sx, sy = rows % W1, rows // W1
    taps = [_tap_arrays(cfg, pyr, s, sx, sy) for s in range(5)]
    worst = 0.0
    off = 0
    feats = []
    for key in _SCALES:
        C = pyr[key].shape[0]
        feats.append((off, C, torch.from_numpy(pyr[key].reshape(C, -1).T.copy()).to(dev).double()))
        off += C
    for b in range(3):
        Wz = torch.from_numpy(params["lin_z.%d.weight" % b]).to(dev).double()
        ref = hdr[b].double().expand(len(rows), -1).clone()
        mag = hdr[b].double().abs().expand(len(rows), -1).clone()
        gemm = torch.zeros_like(ref)
        for s, (o, C, f) in enumerate(feats):
            Q = f @ Wz[:, o:o + C].T
            Qa = f.abs() @ Wz[:, o:o + C].abs().T
            idx, ok, wt = (torch.from_numpy(a).to(dev) for a in taps[s])
            wq = (wt.double() * ok).unsqueeze(-1)
            ref += (wq * Q[idx]).sum(1)
            mag += (wq.abs() * Q[idx].abs()).sum(1)
            gemm += (wq.abs() * (C * E.U) * Qa[idx]).sum(1)
            del Q, Qa
        bound = gemm + 10 * E.U * (mag + gemm)
        rt = E.ratio(tab[torch.from_numpy(rows).to(dev), b], ref, bound)
        worst = max(worst, float(rt.max()))
    print("%s: latent table, %d rows x 3 blocks: worst err/bound %.3g" % (label, len(rows), worst))
    assert worst <= 1.0
    return worst


def _tables(cfg, seed, pyr):
    """fp32 table (fp32tc renderer) and fp16 table (fp16 renderer) of both networks, built from the same image."""
    import torch
    x_rgb = {k: torch.from_numpy(v).to("cuda:0") for k, v in pyr.items()}
    K = torch.from_numpy(cfg.K)
    out = {}
    for prec in ("fp32tc", "fp16"):
        r = make_renderer(cfg, prec, preproject=True)
        pts = torch.zeros((1, 1, 3))
        r.predict("mlp", pts, x_rgb, K, None, torch.zeros((1, 3)), output_type="offset")
        torch.cuda.synchronize()
        out[prec] = r
    return out


@pytest.mark.parametrize("name", ["kitti_mini", "bf_mini"])
def test_latent_table_rows_per_entry(name):
    import torch
    from cases import params_for
    cfg, seed = RENDER_CASES[name]
    pyr = pyramid_for(cfg, seed)
    rs = _tables(cfg, seed, pyr)
    W1, H1 = cfg.sphere_W + 1, cfg.sphere_H + 1
    edges = np.unique(np.concatenate([np.arange(W1), (H1 - 1) * W1 + np.arange(W1), np.arange(H1) * W1,
                                      np.arange(H1) * W1 + W1 - 1]))
    for i, which in enumerate(("mlp", "mlp_gaussian")):
        params = params_for(cfg)[i]
        net = getattr(rs["fp32tc"], which)
        hdr = E.blob_header(net.packed_split)
        t32 = E.table_of(rs["fp32tc"], which)
        t16raw = E.table_of(rs["fp16"], which)
        # the fp16 table is rn16 of the fp32 one (same arithmetic, only the store differs)
        assert torch.equal(t16raw.half().view(torch.int16), t32.half().view(torch.int16))
        # the outside row is c_b, bit for bit
        assert torch.equal(t32[W1 * H1].view(torch.int32), hdr[:3].view(torch.int32))
        _check_table(cfg, pyr, params, hdr, t32, edges, "%s %s edge rows" % (name, which))
        _check_table(cfg, pyr, params, hdr, t32, np.arange(W1 * H1), "%s %s all rows" % (name, which))


def test_latent_table_rows_full_size_B():
    """config B at full size: the edge rows and a seeded 1 % sample of the 455 k rows."""
    import torch
    from cases import params_for
    from scenerf_b200 import synth
    cfg, seed = FULL_CASES["full_B"]
    pyr = synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H)
    r = _tables(cfg, seed, pyr)["fp32tc"]
    W1, H1 = cfg.sphere_W + 1, cfg.sphere_H + 1
    edges = np.concatenate([np.arange(W1), (H1 - 1) * W1 + np.arange(W1), np.arange(H1) * W1, np.arange(H1) * W1 + W1 - 1])
    sample = np.random.default_rng(5).choice(W1 * H1, size=W1 * H1 // 100, replace=False)
    rows = np.unique(np.concatenate([edges, sample]))
    params = params_for(cfg)[0]
    hdr = E.blob_header(r.mlp.packed_split)
    t32 = E.table_of(r, "mlp")
    assert torch.equal(t32[W1 * H1].view(torch.int32), hdr[:3].view(torch.int32))
    _check_table(cfg, pyr, params, hdr, t32, rows, "full_B mlp")
