"""GPU parity tests (run on an H100: pytest -m gpu).  The CUDA path is called through the C ABI (via the ctypes
binding) on the same seeded inputs + recorded noise as the reference goldens and compared with
  * the goldens themselves (outputs of the unmodified reference, tests/golden/make_goldens.py), and
  * the CPU oracle for sizes/configs the goldens do not cover.
Stated tolerances (also in DESIGN.md):
  fp32 (SIMT) mode   : float32 round-off, abs <= 2e-6 + 2e-4 * max(1, |ref|max)
  fp32tc (wgmma)     : fp16 hi/lo split operands, fp32 accumulate -- float32-grade: the SAME tolerances as fp32
  fp16 (wgmma)       : fp16 operands / fp32 accumulate ("fast mode"): depth <= 3e-4 * max_sample_depth (3 cm of 100 m),
                       colour <= 1e-3, other per-sample quantities <= 1e-2 * max(1, |ref|max)
Discrete decisions (rounded sphere pixel, arg-min sample, SOM best-matching unit) are compared exactly where the
implementations agree on the decision and counted where a last-ulp difference flips it."""
import numpy as np
import pytest

from cases import RENDER_CASES, PREDICT_CASES, FULL_CASES, load_golden, params_for, pyramid_for
from helpers import make_renderer, torch_pyramid, max_err
from oracle import scenerf_oracle as orc          # checker only: arg-max margins of the RaySOM decisions

pytestmark = pytest.mark.gpu

TOL = {
    "fp32": dict(rtol=2e-4, atol=2e-6, depth=2e-4, color=2e-4),
    "fp32tc": dict(rtol=2e-4, atol=2e-6, depth=2e-4, color=2e-4),
    "fp16": dict(rtol=1e-2, atol=1e-4, depth=3e-4, color=1e-3),
}
PRECS = ["fp32", "fp32tc", "fp16"]
# RaySOM (ray_som_kl.py:10-78) picks a best-matching prototype per sample.  A ray may differ from the reference only
# if it contains a sample whose two best prototypes are closer (relative gap of p(z|c)) than the precision mode can
# resolve: the gap moves with the gaussian means/stds, which carry the mode's MLP error.
SOM_MARGIN = {"fp32": 1e-3, "fp32tc": 1e-3, "fp16": 0.25}
SOM_OFF_LIMIT = {"fp32": 0.2, "fp32tc": 0.2, "fp16": 0.3}


def _tol(b, prec, scale=None):
    t = TOL[prec]
    return t["atol"] + t["rtol"] * float(max(1.0, np.abs(b).max()) if scale is None else scale)


def _np(d):
    return {k: v.detach().cpu().numpy() for k, v in d.items()}


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", sorted(RENDER_CASES))
def test_render_rays_batch_vs_reference_golden(name, prec):
    cfg, seed = RENDER_CASES[name]
    _compare_with_golden(name, cfg, load_golden(name), prec, pyramid_for(cfg, seed))


@pytest.mark.parametrize("name", sorted(FULL_CASES))
def test_full_size_vs_reference_golden(name):
    """BASELINE.json configs B, B' and C at their FULL sphere-grid sizes and sample counts (1226x370 / 1500x452 /
    640x480; S = 128 / 128 / 96), 256 rays spread over the frame, all three precision modes against the outputs of
    the unmodified reference: index arithmetic at full size (tap offsets up to 80*370*1226, the 16-bit sphere
    coordinates kept in shared memory, (W//s,H//s) corners of the real grids)."""
    from scenerf_b200 import synth
    cfg, seed = FULL_CASES[name]
    g = load_golden(name)
    pyr = synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H)       # 190-420 MB, not cached
    for prec in PRECS:
        _compare_with_golden(name, cfg, g, prec, pyr)


def _compare_with_golden(name, cfg, g, prec, pyr_np, **renderer_kw):
    import torch
    r = make_renderer(cfg, prec, **renderer_kw)
    x_rgb = {k: torch.from_numpy(v).to("cuda:0") for k, v in pyr_np.items()}
    out = _np(r.render_rays_batch(torch.from_numpy(cfg.K), torch.from_numpy(cfg.T), x_rgb,
                                  sampled_pixels=torch.from_numpy(g["pixels"]), ray_batch_size=g["pixels"].shape[0],
                                  noise=(torch.from_numpy(g["noise_u"]), torch.from_numpy(g["noise_n"])), debug=True))
    assert r.last_launches > 0
    R, S, G = g["pixels"].shape[0], cfg.S, cfg.n_gaussians
    for k in ("depth", "color", "gaussian_means", "gaussian_stds", "weights_at_depth", "closest_pts_to_depths",
              "loss_kl", "alphas", "som_vars", "densities", "weights", "depth_volumes"):
        assert out[k].shape == g[k].shape, k
        assert np.isfinite(out[k]).all(), k
    flips_main = (out["dbg_sphere_main"] != g["main_sphere"]).any(axis=1).reshape(R, S).any(axis=1)
    flips_gauss = (out["dbg_sphere_gauss"] != g["gauss_sphere"]).any(axis=1).reshape(R, G).any(axis=1)
    clean = ~(flips_main | flips_gauss)
    assert clean.mean() > 0.95, "sphere-pixel rounding flips on %d of %d rays" % ((~clean).sum(), R)
    t = TOL[prec]
    d_err = max_err(out["depth"][clean], g["depth"][clean])
    c_err = max_err(out["color"][clean], g["color"][clean])
    print("%s/%s: depth max-abs-err %.3e m, colour max-abs-err %.3e, flipped rays %d/%d" % (
        name, prec, d_err, c_err, (~clean).sum(), R))
    assert d_err <= t["depth"] * cfg.max_sample_depth
    assert c_err <= t["color"]
    for k in ("gaussian_means", "gaussian_stds", "alphas", "densities", "weights", "depth_volumes"):
        assert max_err(out[k][clean], g[k][clean]) <= _tol(g[k], prec), k
    assert max_err(out["closest_pts_to_depths"][clean], g["closest_pts_to_depths"][clean]) <= _tol(
        g["depth_volumes"], prec, scale=np.abs(g["depth_volumes"]).max())
    # arg-min sample: compare where the decision has a margin
    dv = g["depth_volumes"]
    srt = np.sort(np.abs(g["depth"][:, None] - dv), axis=1)
    margin = srt[:, 1] - srt[:, 0]
    ok = clean & (margin > 50 * max(d_err, 1e-6))
    assert max_err(out["weights_at_depth"][ok], g["weights_at_depth"][ok]) <= _tol(g["weights"], prec)
    # RaySOM: arg-max near-ties are round-off decided in the reference itself (see tests/test_oracle.py): every ray
    # whose decisions all have a margin must match; rays with a near-tie are counted and bounded
    pm, pg = params_for(cfg)
    o = orc.OracleRenderer(cfg, pm, pg)
    o.render_rays_batch(cfg.K, cfg.T, pyr_np, g["pixels"], R, g["noise_u"], g["noise_n"])
    margin = o.debug["som_margin"]
    bad = np.zeros(R, bool)
    for k in ("loss_kl", "som_vars"):
        err = np.abs(out[k] - g[k]).reshape(R, -1).max(axis=1)
        bad |= err > _tol(g[k], prec) * (10 if prec == "fp16" else 1)
    bad &= clean
    print("%s/%s: RaySOM outputs off on %d of %d rays (%d of them without a near-tie)" % (
        name, prec, bad.sum(), R, (bad & (margin > SOM_MARGIN[prec])).sum()))
    assert not (bad & (margin > SOM_MARGIN[prec])).any(), "SOM outputs differ on rays without an arg-max near-tie"
    assert bad.mean() <= SOM_OFF_LIMIT[prec], "SOM outputs differ on %d of %d rays" % (bad.sum(), R)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("name", sorted(PREDICT_CASES))
def test_predict_adversarial_vs_reference_golden(name, prec):
    import torch
    cfg, seed = PREDICT_CASES[name]
    g = load_golden(name)
    r = make_renderer(cfg, prec)
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    dens, col, dbg = r.predict("mlp", torch.from_numpy(g["cam_pts"]), x_rgb, K, None, torch.from_numpy(g["viewdir"]),
                               debug=True)
    off = r.predict("mlp_gaussian", torch.from_numpy(g["cam_pts"]), x_rgb, K, None, torch.from_numpy(g["viewdir"]),
                    output_type="offset")
    dens, col, dbg, off = dens.cpu().numpy(), col.cpu().numpy(), dbg.cpu().numpy(), off.cpu().numpy()
    same = (dbg == g["sphere"]).all(axis=1).reshape(dens.shape)
    # far out-of-range coords are saturated by the kernel (they can only address zero padding): compare in-range only
    inr = ((np.abs(g["sphere"]) < 1_000_000).all(axis=1)).reshape(dens.shape)
    assert (same | ~inr).mean() > 0.97
    ok = same | ~inr
    assert max_err(dens[ok], g["density"][ok]) <= _tol(g["density"], prec)
    assert max_err(col[ok], g["color"][ok]) <= _tol(g["color"], prec)
    assert max_err(off[ok], g["offset"][ok]) <= _tol(g["offset"], prec)


def test_empty_and_ragged_batches():
    import torch
    cfg, seed = RENDER_CASES["kitti_mini"]
    r = make_renderer(cfg, "fp32")
    x_rgb = torch_pyramid(cfg, seed)
    K, T = torch.from_numpy(cfg.K), torch.from_numpy(cfg.T)
    out = r.render_rays_batch(K, T, x_rgb, sampled_pixels=torch.zeros(0, 2), ray_batch_size=8)
    assert out["depth"].shape == (0,) and out["alphas"].shape == (0, cfg.S)
    g = load_golden("kitti_mini")
    noise = (torch.from_numpy(g["noise_u"]), torch.from_numpy(g["noise_n"]))
    full = r.render_rays_batch(K, T, x_rgb, sampled_pixels=torch.from_numpy(g["pixels"]), noise=noise)
    for n in (1, 3, 33):          # ragged sizes: not a multiple of the warp / tile size
        part = r.render_rays_batch(K, T, x_rgb, sampled_pixels=torch.from_numpy(g["pixels"][:n]),
                                   noise=(noise[0][:n], noise[1][:n]))
        for k in ("depth", "color", "alphas", "loss_kl"):
            assert torch.equal(part[k], full[k][:n]), (n, k)     # rays are independent -> bit-identical
    with pytest.raises(ValueError):
        r.render_rays_batch(K, T, x_rgb, sampled_pixels=torch.zeros(5, 3))


def test_properties_at_scale_philox():
    """Size-independent properties on a larger batch with in-kernel RNG: sorted samples, weights in [0,1], sum <= 1,
    depth within the sampled range, determinism for a fixed seed."""
    import torch
    cfg, seed = RENDER_CASES["kitti_mini"]
    r = make_renderer(cfg, "fp32", rng="philox")
    x_rgb = torch_pyramid(cfg, seed)
    K, T = torch.from_numpy(cfg.K), torch.from_numpy(cfg.T)
    from scenerf_b200 import synth
    pix = torch.from_numpy(synth.random_pixels(77, 2000, cfg.img_W, cfg.img_H))
    r.seed = 123
    a = r.render_rays_batch(K, T, x_rgb, sampled_pixels=pix)
    r.seed = 123
    b = r.render_rays_batch(K, T, x_rgb, sampled_pixels=pix)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    dv, w = a["depth_volumes"], a["weights"]
    assert (dv[:, 1:] >= dv[:, :-1] - 1e-6).all()            # z = t * unit.z is monotone in the sorted distance
    assert (w >= 0).all() and (w.sum(1) <= 1 + 1e-4).all()
    assert (a["alphas"] >= 0).all() and (a["alphas"] <= 1).all()
    assert (a["depth"] <= dv.max(1).values + 1e-3).all() and (a["depth"] >= 0).all()
    assert (a["gaussian_stds"] >= 1.5).all() and (a["gaussian_means"] >= 1.5).all()
    m = a["gaussian_means"].mean(0).cpu().numpy()
    assert (np.diff(m) > 0).all()


def test_pyramid_cache_never_reuses_a_stale_pack():
    """Two different images through the SAME renderer must never share a pack: the cache key holds the caller's tensor objects
    (their storage cannot be recycled under the key), inputs that need a copy (fp16 / non-contiguous maps) included, and an
    in-place update bumps the version counter."""
    import torch
    cfg, seed = RENDER_CASES["kitti_mini"]
    g = load_golden("kitti_mini")
    K, T = torch.from_numpy(cfg.K), torch.from_numpy(cfg.T)
    pix = torch.from_numpy(g["pixels"])
    noise = (torch.from_numpy(g["noise_u"]), torch.from_numpy(g["noise_n"]))
    shared = make_renderer(cfg, "fp32")

    def fresh(x):
        return make_renderer(cfg, "fp32").render_rays_batch(K, T, x, sampled_pixels=pix, noise=noise)["depth"]

    def image(s, kind):
        x = {k: torch.from_numpy(v).to("cuda:0") for k, v in pyramid_for(cfg, seed).items()}
        x = {k: v * (1.0 + 0.25 * s) for k, v in x.items()}
        if kind == "half":
            return {k: v.half() for k, v in x.items()}                       # needs a dtype copy
        if kind == "strided":
            return {k: torch.cat([v, v], 2)[:, :, :v.shape[2]] for k, v in x.items()}      # non-contiguous view
        return x

    for i, kind in enumerate(["half", "half", "strided", "strided", "plain", "half"]):
        x = image(i, kind)
        got = shared.render_rays_batch(K, T, x, sampled_pixels=pix, noise=noise)["depth"]
        assert torch.equal(got, fresh(x)), (i, kind)
        del x                                                                 # the next image may be allocated at the same address
        torch.cuda.empty_cache()
    x = image(7, "plain")
    a = shared.render_rays_batch(K, T, x, sampled_pixels=pix, noise=noise)["depth"].clone()
    x["1_1"].mul_(1.5)                                                        # in-place: same storage, new version
    b = shared.render_rays_batch(K, T, x, sampled_pixels=pix, noise=noise)["depth"]
    assert not torch.equal(a, b) and torch.equal(b, fresh(x))
    x["1_1"].data.mul_(0.5)                                                   # bypasses the version counter: needs invalidate_pyramid()
    shared.invalidate_pyramid()
    assert torch.equal(shared.render_rays_batch(K, T, x, sampled_pixels=pix, noise=noise)["depth"], fresh(x))


@pytest.mark.parametrize("U,G,P", [(1, 1, 1), (16, 8, 4), (128, 8, 16), (7, 3, 5)])
def test_sample_count_extremes_vs_oracle(U, G, P):
    """Shapes the goldens do not cover, against the oracle (itself pinned to the reference): the smallest ray (S = 2), the maximum
    number of gaussians (8) and samples (S = 256, the documented cap), odd counts (S = 22: ragged warps, tiles straddling rays)."""
    import torch
    from scenerf_b200 import synth
    cfg = synth.config_A(name="extreme", sphere_W=300, sphere_H=90, yaw_deg=10.0, tz=1.0, n_pts_uni=U, n_gaussians=G, n_pts_per_gaussian=P)
    seed = 31
    pm, pg = params_for(cfg)
    R = 24
    pix = synth.random_pixels(55, R, cfg.img_W, cfg.img_H)
    rng = np.random.default_rng(3)
    nu = rng.random((R, U), dtype=np.float32)
    nn_ = rng.standard_normal((R, G * P)).astype(np.float32)
    pyr = pyramid_for(cfg, seed)
    ref = orc.OracleRenderer(cfg, pm, pg).render_rays_batch(cfg.K, cfg.T, pyr, pix, R, nu, nn_)
    x_rgb = torch_pyramid(cfg, seed)
    for prec in ("fp32", "fp32tc"):
        out = _np(make_renderer(cfg, prec).render_rays_batch(torch.from_numpy(cfg.K), torch.from_numpy(cfg.T), x_rgb,
                                                             sampled_pixels=torch.from_numpy(pix), ray_batch_size=R,
                                                             noise=(torch.from_numpy(nu), torch.from_numpy(nn_))))
        t = TOL[prec]
        assert out["alphas"].shape == (R, U + G * P) and out["gaussian_means"].shape == (R, G)
        assert max_err(out["depth"], ref["depth"]) <= t["depth"] * cfg.max_sample_depth, prec
        assert max_err(out["color"], ref["color"]) <= t["color"], prec
        for k in ("gaussian_means", "gaussian_stds", "alphas", "weights", "depth_volumes"):
            assert max_err(out[k], ref[k]) <= _tol(ref[k], prec), (prec, k)
    with pytest.raises(ValueError):
        big = synth.config_A(name="too_big", sphere_W=300, sphere_H=90, n_pts_uni=129, n_gaussians=8, n_pts_per_gaussian=16)   # S = 257
        make_renderer(big, "fp32").render_rays_batch(torch.from_numpy(cfg.K), torch.from_numpy(cfg.T), x_rgb, sampled_pixels=torch.from_numpy(pix))
