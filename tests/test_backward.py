"""Backward pass (hot-path contract row 8f-1).  Golden = gradients the reference itself produces under torch.autograd
for L = sum_k <out_k, C_k> with fixed cotangents (tests/golden/make_goldens.py `run_grad_case`): d L / d raw MLP outputs
in full, parameter gradients as digests (full for small tensors; G@u, G.T@v and G[::16, ::16] for the big ones), feature-
map gradients as per-channel sums, per-pixel sums and the first 4 channels.

Tolerance: the reference computes in float32; a unit whose pre-activation is within float32 round-off of zero has its
ReLU derivative decided by that round-off, and the flip changes whole gradient rows discontinuously.  The float64
oracle restatement (validated against float64 torch.autograd to 1e-15) differs from the float32 reference by up to
1.3e-2 (max, relative to the tensor's largest entry) and up to 8e-3 (relative L2 of a digest); the CUDA float32 path is held to the same
bounds against the golden AND against the float64 oracle."""
import numpy as np
import pytest

from cases import load_golden
from scenerf_b200 import synth

GRAD_KEYS = ("depth", "color", "gaussian_means", "gaussian_stds", "weights_at_depth", "closest_pts_to_depths", "loss_kl",
             "alphas", "densities", "weights", "depth_volumes")
CASES = {
    "grad_kitti": (lambda: synth.config_A(name="grad_kitti", sphere_W=300, sphere_H=90, yaw_deg=10.0, tz=1.0), 41),
    "grad_bf": (lambda: synth.config_C(name="grad_bf", sphere_W=160, sphere_H=120, n_pts_uni=32), 42),
}
MAX_REL, L2_REL = 3e-2, 2e-2


def cotangents(g):
    return {k: synth.hash_normalish(900 + i, int(np.prod(g[k].shape))).reshape(g[k].shape).astype(np.float32)
            for i, k in enumerate(GRAD_KEYS)}


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(1e-30, np.abs(b).max())
    l2 = np.linalg.norm(a - b) / max(1e-30, np.linalg.norm(b))
    return np.abs(a - b).max() / scale, l2


def check_param_grads(grads, g, tag, what):
    u = lambda n: synth.hash_normalish(700, n).astype(np.float64)
    v = lambda n: synth.hash_normalish(701, n).astype(np.float64)
    worst = (0.0, 0.0)
    for k, G in grads.items():
        G = np.asarray(G, np.float64)
        key = "%s.%s" % (tag, k)
        if "g:" + key in g:
            pairs = [(G, g["g:" + key])]
        else:
            pairs = [(G @ u(G.shape[1]), g["gu:" + key]), (G.T @ v(G.shape[0]), g["gv:" + key]), (G[::16, ::16], g["gs:" + key])]
        for a, b in pairs:
            mx, l2 = _rel(a, b)
            assert mx <= MAX_REL and l2 <= L2_REL, "%s %s: max-rel %.2e, L2-rel %.2e" % (what, key, mx, l2)
            worst = (max(worst[0], mx), max(worst[1], l2))
    return worst


def check_pyramid_grads(gp, g, what):
    for k, G in gp.items():
        G = np.asarray(G, np.float64)
        ref_abs = float(g["gpyr_abs:" + k])
        if ref_abs == 0.0:
            assert np.abs(G).max() == 0.0, "%s %s: reference gradient is identically zero (quirk Q2)" % (what, k)
            continue
        assert abs(np.abs(G).sum() - ref_abs) <= 2e-3 * ref_abs, (what, k)
        for a, b in ((G.sum((1, 2)), g["gpyr_chsum:" + k]), (G.sum(0), g["gpyr_pixsum:" + k]), (G[:4], g["gpyr_head:" + k])):
            mx, l2 = _rel(a, b)
            assert mx <= MAX_REL and l2 <= L2_REL, "%s %s: max-rel %.2e, L2-rel %.2e" % (what, k, mx, l2)


@pytest.mark.parametrize("name", sorted(CASES))
def test_backward_oracle_matches_reference_autograd(name):
    from oracle import scenerf_oracle as so, backward_oracle as bo
    g = load_golden(name)
    cfg, seed = CASES[name][0](), CASES[name][1]
    orc = so.OracleRenderer(cfg, *synth.make_model_params(cfg))
    pyr = synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H)
    r = bo.render_backward(orc, cfg.K, cfg.T, pyr, g["pixels"], g["noise_u"], g["noise_n"], cotangents(g))
    assert abs(r["loss"] - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    for k in ("graw_main", "graw_gauss"):
        mx, l2 = _rel(r[k], g[k])
        assert mx <= 2e-4 and l2 <= 2e-4, (k, mx, l2)
    check_param_grads(r["g_main"], g, "main", "oracle")
    check_param_grads(r["g_gauss"], g, "gauss", "oracle")
    check_pyramid_grads(r["g_pyr"], g, "oracle")


def test_mlp_backward_oracle_against_finite_differences():
    """Independent of any golden: central differences of the float64 ResnetFC restatement."""
    from oracle import backward_oracle as bo
    cfg = synth.config_A(name="fd")
    pm, _ = synth.make_model_params(cfg)
    rng = np.random.default_rng(1)
    n = 6
    z = (rng.standard_normal((n, 2480)) * 0.5).astype(np.float32)
    x = rng.standard_normal((n, 42)).astype(np.float32)
    gout = rng.standard_normal((n, 4))
    grads, dz, _ = bo.mlp_backward(pm, z, x, gout)
    f = lambda P, Z: float((bo.mlp_forward_saved(P, Z, x)[0] * gout).sum())
    eps = 1e-6
    for key, idx in (("lin_z.1.weight", (7, 100)), ("blocks.0.fc_0.weight", (3, 5)), ("lin_in.bias", (11,)), ("lin_out.weight", (2, 9))):
        P = {k: v.astype(np.float64).copy() for k, v in pm.items()}
        P[key][idx] += eps
        up = f(P, z)
        P[key][idx] -= 2 * eps
        fd = (up - f(P, z)) / (2 * eps)
        assert abs(fd - grads[key][idx]) <= 1e-5 * max(1.0, abs(fd)), (key, fd, grads[key][idx])
    Z = z.astype(np.float64).copy()
    Z[2, 33] += eps
    up = f(pm, Z)
    Z[2, 33] -= 2 * eps
    fd = (up - f(pm, Z)) / (2 * eps)
    assert abs(fd - dz[2, 33]) <= 1e-5 * max(1.0, abs(fd))


# ------------------------------------------------------------------------------------------------ GPU

def _run_cuda(name, save_activations=True, matmul="fp32"):
    import torch
    from helpers import hp_from_cfg
    from scenerf_b200.autograd import TrainableRenderer, PARAM_KEYS
    g = load_golden(name)
    cfg, seed = CASES[name][0](), CASES[name][1]
    pm, pg = synth.make_model_params(cfg)
    dev = torch.device("cuda:0")
    mk = lambda d: {k: torch.from_numpy(d[k]).to(dev).requires_grad_(True) for k in PARAM_KEYS}
    tm, tg = mk(pm), mk(pg)
    x_rgb = {k: torch.from_numpy(v).to(dev).requires_grad_(True) for k, v in synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H).items()}
    t = TrainableRenderer(hp_from_cfg(cfg), tm, tg, device=dev, save_activations=save_activations, matmul=matmul)
    out = t.render_rays_batch(torch.from_numpy(cfg.K), torch.from_numpy(cfg.T), x_rgb, sampled_pixels=torch.from_numpy(g["pixels"]),
                              ray_batch_size=g["pixels"].shape[0],
                              noise=(torch.from_numpy(g["noise_u"]), torch.from_numpy(g["noise_n"])))
    cot = cotangents(g)
    L = sum((out[k] * torch.from_numpy(cot[k]).to(dev)).sum() for k in GRAD_KEYS)
    L.backward()
    return g, cfg, seed, out, L, tm, tg, x_rgb, t


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_backward_matches_reference_autograd(name):
    g, cfg, seed, out, L, tm, tg, x_rgb, t = _run_cuda(name)
    assert not out["som_vars"].requires_grad and out["depth"].requires_grad
    assert abs(float(L) - float(g["loss"])) <= 2e-4 * abs(float(g["loss"]))
    assert t.renderer.last_backward_launches > 50
    np_ = lambda d: {k: v.grad.detach().cpu().numpy() for k, v in d.items()}
    w1 = check_param_grads(np_(tm), g, "main", "cuda")
    w2 = check_param_grads(np_(tg), g, "gauss", "cuda")
    check_pyramid_grads(np_(x_rgb), g, "cuda")
    print("%s: worst parameter-gradient error vs reference autograd: max-rel %.2e, L2-rel %.2e" % (
        name, max(w1[0], w2[0]), max(w1[1], w2[1])))


@pytest.mark.gpu
def test_cuda_backward_matches_float64_oracle_and_is_reproducible():
    """Against the float64 restatement entry by entry (no digests), and bit-reproducible parameter gradients."""
    from oracle import scenerf_oracle as so, backward_oracle as bo
    name = "grad_kitti"
    g, cfg, seed, out, L, tm, tg, x_rgb, t = _run_cuda(name)
    orc = so.OracleRenderer(cfg, *synth.make_model_params(cfg))
    r = bo.render_backward(orc, cfg.K, cfg.T, synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H), g["pixels"], g["noise_u"],
                           g["noise_n"], cotangents(g))
    for tag, tens, ref in (("main", tm, r["g_main"]), ("gauss", tg, r["g_gauss"])):
        for k, v in tens.items():
            mx, l2 = _rel(v.grad.cpu().numpy(), ref[k])
            assert mx <= MAX_REL and l2 <= L2_REL, (tag, k, mx, l2)
    for k, v in x_rgb.items():
        if np.abs(r["g_pyr"][k]).max() == 0:
            assert float(v.grad.abs().max()) == 0.0
            continue
        mx, l2 = _rel(v.grad.cpu().numpy(), r["g_pyr"][k])
        assert mx <= MAX_REL and l2 <= L2_REL, (k, mx, l2)
    g2, _, _, _, _, tm2, tg2, x2, _ = _run_cuda(name)
    for k in tm:
        assert (tm[k].grad == tm2[k].grad).all() and (tg[k].grad == tg2[k].grad).all(), k
    # recomputing the forward inside the backward (save_activations=False) is the same arithmetic: identical gradients
    g3, _, _, out3, _, tm3, tg3, x3, _ = _run_cuda(name, save_activations=False)
    assert all((out[k] == out3[k]).all() for k in out)
    for k in tm:
        assert (tm[k].grad == tm3[k].grad).all() and (tg[k].grad == tg3[k].grad).all(), k


@pytest.mark.gpu
def test_cuda_backward_partial_cotangents_and_chunking():
    """Only depth + colour losses (what an image loss uses), rays split into chunks like scenerf.py:419-433: the gradient of
    the chunked call equals the un-chunked one up to float32 summation order."""
    import torch
    from helpers import hp_from_cfg
    from scenerf_b200.autograd import TrainableRenderer, PARAM_KEYS
    g = load_golden("grad_kitti")
    cfg, seed = CASES["grad_kitti"][0](), 41
    pm, pg = synth.make_model_params(cfg)
    dev = torch.device("cuda:0")
    res = []
    for rbs in (48, 20):
        mk = lambda d: {k: torch.from_numpy(d[k]).to(dev).requires_grad_(True) for k in PARAM_KEYS}
        tm, tg = mk(pm), mk(pg)
        x_rgb = {k: torch.from_numpy(v).to(dev).requires_grad_(True) for k, v in synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H).items()}
        t = TrainableRenderer(hp_from_cfg(cfg), tm, tg, device=dev)
        out = t.render_rays_batch(torch.from_numpy(cfg.K), torch.from_numpy(cfg.T), x_rgb, sampled_pixels=torch.from_numpy(g["pixels"]),
                                  ray_batch_size=rbs, noise=(torch.from_numpy(g["noise_u"]), torch.from_numpy(g["noise_n"])))
        (out["depth"].abs().sum() * 0.01 + (out["color"] - 0.5).abs().sum()).backward()
        res.append((out, tm, tg, x_rgb))
    (o1, m1, g1, x1), (o2, m2, g2, x2) = res
    assert torch.equal(o1["depth"], o2["depth"]) and torch.equal(o1["color"], o2["color"])
    for k in m1:
        for a, b in ((m1[k].grad, m2[k].grad), (g1[k].grad, g2[k].grad)):
            assert float((a - b).abs().max()) <= 1e-4 * max(1e-12, float(a.abs().max())), k
    assert float(x1["1_1"].grad.abs().sum()) > 0
    assert float((x1["1_1"].grad - x2["1_1"].grad).abs().max()) <= 1e-4 * float(x1["1_1"].grad.abs().max())


def _full_tensor_check(tensors, ref, what, l2_max, cos_min):
    worst = (0.0, 1.0)
    for k, v in tensors.items():
        a, b = v.grad.detach().cpu().numpy().astype(np.float64).ravel(), np.asarray(ref[k], np.float64).ravel()
        if np.abs(b).max() == 0:
            assert np.abs(a).max() == 0, (what, k)
            continue
        l2 = np.linalg.norm(a - b) / np.linalg.norm(b)
        cos = float(a @ b / (np.linalg.norm(a) * np.linalg.norm(b)))
        assert l2 <= l2_max and cos >= cos_min, "%s %s: L2-rel %.3f cosine %.5f" % (what, k, l2, cos)
        worst = (max(worst[0], l2), min(worst[1], cos))
    return worst


def test_tf32_emulation_sets_the_tolerance():
    """CPU: the float64 oracle with tf32-truncated GEMM operands (what wgmma .tf32 feeds the multipliers) against the
    exact float64 oracle.  This is the deviation ANY tf32 implementation shows on these small cases (<= 3072 points, so a few
    hundred ReLU-derivative flips are visible): full-tensor relative L2 up to 0.10, cosine >= 0.995.  The GPU test below
    holds the CUDA tf32 mode to 2x that."""
    from oracle import scenerf_oracle as so, backward_oracle as bo
    name = "grad_bf"
    g = load_golden(name)
    cfg, seed = CASES[name][0](), CASES[name][1]
    orc = so.OracleRenderer(cfg, *synth.make_model_params(cfg))
    pyr = synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H)
    a = bo.render_backward(orc, cfg.K, cfg.T, pyr, g["pixels"], g["noise_u"], g["noise_n"], cotangents(g), tf32=True)
    b = bo.render_backward(orc, cfg.K, cfg.T, pyr, g["pixels"], g["noise_u"], g["noise_n"], cotangents(g), tf32=False)
    assert abs(a["loss"] - b["loss"]) <= 2e-4 * abs(b["loss"])
    worst = 0.0
    for tag in ("g_main", "g_gauss"):
        for k in a[tag]:
            x, y = a[tag][k].ravel(), b[tag][k].ravel()
            worst = max(worst, np.linalg.norm(x - y) / np.linalg.norm(y))
    assert 0.01 <= worst <= 0.15, worst


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_cuda_backward_tf32_mode(name):
    """matmul="tf32": the GEMMs of forward and backward on wgmma .tf32 (float32 storage, 10-bit mantissa operands,
    float32 accumulate).  Bounds from the emulation above: loss 2e-3 relative, depth 1.5e-3 * max_sample_depth, every
    gradient tensor within relative L2 0.2 / cosine 0.98 of the exact (float64) gradient.  The strict float32 mode keeps the
    tight bounds of the tests above."""
    from oracle import scenerf_oracle as so, backward_oracle as bo
    g, cfg, seed, out, L, tm, tg, x_rgb, t = _run_cuda(name, matmul="tf32")
    assert abs(float(L.detach()) - float(g["loss"])) <= 2e-3 * abs(float(g["loss"]))
    d = np.abs(out["depth"].detach().cpu().numpy() - g["depth"]).max()
    assert d <= 1.5e-3 * cfg.max_sample_depth
    orc = so.OracleRenderer(cfg, *synth.make_model_params(cfg))
    r = bo.render_backward(orc, cfg.K, cfg.T, synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H), g["pixels"], g["noise_u"],
                           g["noise_n"], cotangents(g))
    w1 = _full_tensor_check(tm, r["g_main"], "cuda-tf32 main", 0.2, 0.98)
    w2 = _full_tensor_check(tg, r["g_gauss"], "cuda-tf32 gauss", 0.2, 0.98)
    w3 = _full_tensor_check(x_rgb, r["g_pyr"], "cuda-tf32 maps", 0.2, 0.98)
    print("%s tf32: depth err %.2e m; gradients vs float64: worst L2-rel %.3f, min cosine %.5f" % (
        name, d, max(w1[0], w2[0], w3[0]), min(w1[1], w2[1], w3[1])))


def _edge_inputs(R):
    """R random rays of grad_kitti with seeded noise and a fixed loss (cotangents)."""
    cfg, seed = CASES["grad_kitti"][0](), 43
    pm, pg = synth.make_model_params(cfg)
    pix = synth.random_pixels(50 + R, R, cfg.img_W, cfg.img_H)
    rng = np.random.default_rng(R)
    nu = rng.random((R, cfg.n_pts_uni)).astype(np.float32)
    nn_ = rng.standard_normal((R, cfg.n_gaussians * cfg.n_pts_per_gaussian)).astype(np.float32)
    pyr = synth.make_pyramid(seed, cfg.sphere_W, cfg.sphere_H)
    cot = {"depth": np.full(R, 0.05, np.float32), "color": np.full((R, 3), 1.0, np.float32), "loss_kl": np.ones(R, np.float32),
           "gaussian_means": np.full((R, cfg.n_gaussians), 0.01, np.float32)}
    return cfg, pm, pg, pix, nu, nn_, pyr, cot


def edge_case_grads(R, matmul, save_activations=True):
    """The CUDA gradients of _edge_inputs(R): (main MLP tensors, gaussian MLP tensors, feature maps, renderer)."""
    import torch
    from helpers import hp_from_cfg
    from scenerf_b200.autograd import TrainableRenderer, PARAM_KEYS
    cfg, pm, pg, pix, nu, nn_, pyr, cot = _edge_inputs(R)
    dev = torch.device("cuda:0")
    mk = lambda d: {k: torch.from_numpy(d[k]).to(dev).requires_grad_(True) for k in PARAM_KEYS}
    tm, tg = mk(pm), mk(pg)
    x_rgb = {k: torch.from_numpy(v).to(dev).requires_grad_(True) for k, v in pyr.items()}
    t = TrainableRenderer(hp_from_cfg(cfg), tm, tg, device=dev, save_activations=save_activations, matmul=matmul)
    out = t.render_rays_batch(torch.from_numpy(cfg.K), torch.from_numpy(cfg.T), x_rgb, sampled_pixels=torch.from_numpy(pix),
                              ray_batch_size=R, noise=(torch.from_numpy(nu), torch.from_numpy(nn_)))
    sum((out[k] * torch.from_numpy(c).to(dev)).sum() for k, c in cot.items()).backward()
    return tm, tg, x_rgb, t


def check_edge_case(R, matmul, tm, tg, x_rgb):
    """edge_case_grads against the float64 oracle."""
    from oracle import scenerf_oracle as so, backward_oracle as bo
    cfg, pm, pg, pix, nu, nn_, pyr, cot = _edge_inputs(R)
    orc = so.OracleRenderer(cfg, pm, pg)
    r = bo.render_backward(orc, cfg.K, cfg.T, pyr, pix, nu, nn_, cot)
    l2, cos = (0.25, 0.97) if matmul == "tf32" else (2e-2, 0.9995)
    if R == 1:
        l2, cos = 5e-2, 0.999          # 64 points: a single ReLU flip is a visible fraction of a tensor
    w1 = _full_tensor_check(tm, r["g_main"], "main", l2, cos)
    w2 = _full_tensor_check(tg, r["g_gauss"], "gauss", l2, cos)
    w3 = _full_tensor_check(x_rgb, r["g_pyr"], "maps", l2, cos)
    print("R=%d %s: worst L2-rel %.2e, min cosine %.6f" % (R, matmul, max(w1[0], w2[0], w3[0]), min(w1[1], w2[1], w3[1])))


@pytest.mark.gpu
@pytest.mark.parametrize("R,matmul", [(1, "fp32"), (150, "fp32"), (150, "tf32")])
def test_cuda_backward_edge_sizes(R, matmul):
    """One ray (a single partial tile everywhere) and 150 rays = 9600 sample points in one training chunk (split-K
    remainders, ragged TMA boxes) against the float64 oracle.  test_backward_chunks.py runs the 150-ray case in 10 chunks."""
    tm, tg, x_rgb, _ = edge_case_grads(R, matmul)
    check_edge_case(R, matmul, tm, tg, x_rgb)
