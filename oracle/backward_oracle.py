"""TEST INFRASTRUCTURE ONLY: numpy restatement of the BACKWARD pass of the hot path -- what torch.autograd computes for
the reference's `SceneRF.render_rays_batch` (/root/reference/scenerf/models/scenerf.py:392-748) -- written out by hand.

Forward decisions (rounded sphere pixels, sort order, arg-min sample, SOM mask) come from the float32 forward oracle
(oracle/scenerf_oracle.py); the derivative arithmetic is done in float64.  Pinned against gradients produced by the
reference itself under torch.autograd (tests/golden/grad_kitti.npz, grad_bf.npz; make_goldens.py `run_grad_case`).

Gradient structure reproduced (file:line of the forward op whose derivative it is):
  * main MLP inputs are detached (scenerf.py:662) -> no gradient into the sampled points through the MLP;
  * sorted sensor distances / depth volumes keep their dependence on the gaussian means / stds
    (utils.py:204-214, the 0.1 clamp kills the gradient of clamped samples; uniform samples are constants);
  * compositing scenerf.py:704-748 (cumprod backward as torch: reverse cumsum of grad*out divided by the input);
  * RaySOM: loss_kl differentiates only gauss_means / gauss_stds (ray_som_kl.py:17-19,71: everything else detached);
    `som_vars` is treated as NON-differentiable (its only consumer logs it detached, scenerf.py:222-227);
  * heads: sigmoid colour, softplus(x-1) density (scenerf.py:533-536,473-481); means = relu(m0+o0)+c, stds = relu(o1+std)+c;
  * ResnetFC backward (resnetfc.py:133-164), grid_sample(bilinear, zeros) backward w.r.t. the feature maps
    (utils.py:232-247) for the 5 scales with the reference's normalisation quirk."""
import math

import numpy as np

from . import scenerf_oracle as so

f32, f64 = np.float32, np.float64

GRAD_KEYS = ("depth", "color", "gaussian_means", "gaussian_stds", "weights_at_depth", "closest_pts_to_depths", "loss_kl",
             "alphas", "densities", "weights", "depth_volumes")


def taps_2d(coords, norm_size, H, W):
    """Indices / validity / weights of the 4 bilinear taps exactly as sample_feats_2d computes them."""
    gx = ((coords[:, 0].astype(f32) / f32(norm_size[0])).astype(f32) * f32(2) - f32(1)).astype(f32)
    gy = ((coords[:, 1].astype(f32) / f32(norm_size[1])).astype(f32) * f32(2) - f32(1)).astype(f32)
    ix = ((gx + f32(1)) * f32(W / 2.0) - f32(0.5)).astype(f32)
    iy = ((gy + f32(1)) * f32(H / 2.0) - f32(0.5)).astype(f32)
    x_w, y_n = np.floor(ix), np.floor(iy)
    w = (ix - x_w).astype(f32)
    e = (f32(1) - w).astype(f32)
    n = (iy - y_n).astype(f32)
    s = (f32(1) - n).astype(f32)
    x0, y0 = x_w.astype(np.int64), y_n.astype(np.int64)
    out = []
    for dx, dy, wt in ((0, 0, s * e), (1, 0, s * w), (0, 1, n * e), (1, 1, n * w)):
        xx, yy = x0 + dx, y0 + dy
        ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        out.append((np.where(ok, yy * W + xx, 0), ok, wt.astype(f32)))
    return out


def tf32_trunc(a):
    """Operand rounding of the tf32 tensor-core MMA (wgmma .tf32): the float32 value with its low 13 mantissa bits dropped."""
    u = np.ascontiguousarray(a, dtype=f32).view(np.uint32) & np.uint32(0xFFFFE000)
    return u.view(f32).astype(f64)


def _mm(a, b, tf32):
    """a @ b in float64; tf32=True emulates the tensor-core mode of csrc/gemm_tf32.cu (operands truncated to tf32,
    products and sums exact/float32-accumulated on the device -- float64 here)."""
    return (tf32_trunc(a) @ tf32_trunc(b)) if tf32 else (a @ b)


def mlp_forward_saved(params, z, x, n_blocks=3, tf32=False):
    """resnetfc.py:133-164 in float64 keeping what the backward needs.  tf32: the GEMMs the CUDA tf32 mode runs on tensor
    cores (everything except lin_in / lin_out) use truncated operands."""
    P = {k: v.astype(f64) for k, v in params.items()}
    z, x = z.astype(f64), x.astype(f64)
    h = x @ P["lin_in.weight"].T + P["lin_in.bias"]
    saved = []
    for b in range(n_blocks):
        pre = h + _mm(z, P["lin_z.%d.weight" % b].T, tf32) + P["lin_z.%d.bias" % b]
        net = _mm(np.maximum(pre, 0), P["blocks.%d.fc_0.weight" % b].T, tf32) + P["blocks.%d.fc_0.bias" % b]
        h = pre + _mm(np.maximum(net, 0), P["blocks.%d.fc_1.weight" % b].T, tf32) + P["blocks.%d.fc_1.bias" % b]
        saved.append((pre, net))
    out = np.maximum(h, 0) @ P["lin_out.weight"].T + P["lin_out.bias"]
    return out, saved, h, P


def mlp_backward(params, z, x, g_out, n_blocks=3, tf32=False):
    """-> (dict of parameter gradients, dz (n, d_latent))."""
    out, saved, h3, P = mlp_forward_saved(params, z, x, n_blocks, tf32)
    z64, x64 = z.astype(f64), x.astype(f64)
    g = {}
    g_out = g_out.astype(f64)
    g["lin_out.weight"] = g_out.T @ np.maximum(h3, 0)
    g["lin_out.bias"] = g_out.sum(0)
    dh = (g_out @ P["lin_out.weight"]) * (h3 > 0)
    dz = np.zeros_like(z64)
    for b in reversed(range(n_blocks)):
        pre, net = saved[b]
        g["blocks.%d.fc_1.weight" % b] = _mm(dh.T, np.maximum(net, 0), tf32)
        g["blocks.%d.fc_1.bias" % b] = dh.sum(0)
        dnet = _mm(dh, P["blocks.%d.fc_1.weight" % b], tf32) * (net > 0)
        g["blocks.%d.fc_0.weight" % b] = _mm(dnet.T, np.maximum(pre, 0), tf32)
        g["blocks.%d.fc_0.bias" % b] = dnet.sum(0)
        dpre = dh + _mm(dnet, P["blocks.%d.fc_0.weight" % b], tf32) * (pre > 0)
        g["lin_z.%d.weight" % b] = _mm(dpre.T, z64, tf32)
        g["lin_z.%d.bias" % b] = dpre.sum(0)
        dz += _mm(dpre, P["lin_z.%d.weight" % b], tf32)
        dh = dpre
    g["lin_in.weight"] = dh.T @ x64
    g["lin_in.bias"] = dh.sum(0)
    return g, dz, out


def scatter_latent_grad(dz, coords, x_rgb, sphere_W, sphere_H, grads):
    """grid_sample backward w.r.t. the inputs: grads[key] (C,H,W) += taps^T dz   (scenerf.py:522-527 normalisation)."""
    off = 0
    for s in (1, 2, 4, 8, 16):
        key = "1_%d" % s
        C, H, W = x_rgb[key].shape
        norm = (sphere_W, sphere_H) if s == 1 else (sphere_W // s, sphere_H // s)
        flat = grads[key].reshape(C, H * W)
        part = dz[:, off:off + C]
        for idx, ok, wt in taps_2d(coords, norm, H, W):
            sel = np.nonzero(ok)[0]
            if sel.size:
                np.add.at(flat.T, idx[sel], part[sel] * wt[sel].astype(f64)[:, None])
        off += C


def render_backward(orc: "so.OracleRenderer", K, T, x_rgb, pixels, noise_u, noise_n, cot: dict, tf32: bool = False):
    """One chunk (all rays) of render_rays_batch, forward + backward.  cot: cotangents for GRAD_KEYS (missing = 0).
    Returns dict(out=forward outputs, g_main=..., g_gauss=... parameter grads, g_pyr={key: (C,H,W)}, graw_main, graw_gauss)."""
    cfg = orc.cfg
    K, T = K.astype(f32), T.astype(f32)
    inv_K = np.linalg.inv(K).astype(f32)
    orc._inv_K = inv_K
    pix = pixels.astype(f32)
    R = pix.shape[0]
    U, G, Pn = cfg.n_pts_uni, cfg.n_gaussians, cfg.n_pts_per_gaussian
    # ---------------- forward (float32 oracle, keeping intermediates) -------------------------------------------
    pts_u, depth_u, t_u, viewdir, unit = so.sample_rays_viewdir(inv_K, T, pix, U, cfg.max_sample_depth, noise_u)
    step = cfg.max_sample_depth * 1.0 / G
    m0 = so.torch_linspace(step / 2, cfg.max_sample_depth - step / 2, G)
    gpts = so.cam_pts_2_cam_pts((m0[None, :, None] * unit[:, None, :]).astype(f32).reshape(-1, 3), T)

    def inputs_of(p, n_per):
        pixp = so.cam_pts_2_pix(p, K)
        coords, _ = so.sphere_coords_from_pixels(pixp, inv_K, cfg.angles(), cfg.sphere_W, cfg.sphere_H)
        z = so.gather_latent(x_rgb, coords, cfg.sphere_W, cfg.sphere_H)
        x = np.concatenate([so.positional_encoding(p), np.repeat(viewdir.astype(f32), n_per, axis=0)], axis=1)
        return coords, z, x

    gp_coords, gp_lat, gp_x = inputs_of(gpts, G)
    fwd = (lambda P_, z_, x_: mlp_forward_saved(P_, z_, x_, tf32=True)[0].astype(f32)) if tf32 else so.resnetfc
    g_raw = fwd(orc.pg, gp_lat, gp_x).reshape(R, G, 2)
    pre_mean = (m0[None, :] + g_raw[:, :, 0]).astype(f32)
    pre_std = (g_raw[:, :, 1] + f32(cfg.std)).astype(f32)
    means = (np.maximum(pre_mean, 0) + orc.add_const).astype(f32)
    stds = (np.maximum(pre_std, 0) + orc.add_const).astype(f32)
    t_g_raw = (np.repeat(means, Pn, axis=1) + noise_n.astype(f32) * np.repeat(stds, Pn, axis=1)).astype(f32)
    clamped = t_g_raw < f32(0.1)
    pts_g, depth_g, t_g = so.sample_rays_gaussian(T, unit, means, stds, Pn, noise_n)
    pts = np.concatenate([pts_u, pts_g], axis=1)
    depth = np.concatenate([depth_u, depth_g], axis=1)
    t = np.concatenate([t_u, t_g], axis=1)
    order = np.argsort(t, axis=1, kind="stable")
    t = np.take_along_axis(t, order, 1)
    zc = np.take_along_axis(depth, order, 1)
    pts = np.take_along_axis(pts, order[:, :, None], 1)
    S = t.shape[1]
    mp_coords, mp_lat, mp_x = inputs_of(pts.reshape(-1, 3), S)
    m_raw = fwd(orc.pm, mp_lat, mp_x)
    colors = so.sigmoid(m_raw[:, :3]).reshape(R, S, 3)
    sigma = so.softplus(m_raw[:, 3] - f32(1)).reshape(R, S)
    ro = orc.render_depth_and_color(sigma, t, zc, colors)
    loss_kl, som_means, som_vars = orc.ray_som(means, stds, np.where(t < 0, f32(0), t), ro["alphas"])
    out = dict(depth=ro["depth"], color=ro["color"], gaussian_means=means, gaussian_stds=stds,
               weights_at_depth=ro["weights_at_depth"], closest_pts_to_depths=ro["closest_pts_to_depth"], loss_kl=loss_kl,
               alphas=ro["alphas"], som_vars=som_vars, densities=sigma, weights=ro["weights"], depth_volumes=zc)

    # ---------------- backward ----------------------------------------------------------------------------------
    c = {k: (np.zeros(out[k].shape, f64) if cot.get(k) is None else np.asarray(cot[k], f64)) for k in GRAD_KEYS}
    t64, z64, sg, col = t.astype(f64), zc.astype(f64), sigma.astype(f64), colors.astype(f64)
    delta = np.empty_like(t64)
    delta[:, 0] = t64[:, 0]
    delta[:, 1:] = t64[:, 1:] - t64[:, :-1]
    E = np.exp(-delta * sg)
    alpha = 1 - E
    s_ = 1 - alpha + 1e-10
    Tj = np.cumprod(np.concatenate([np.ones((R, 1)), s_], axis=1), axis=1)[:, :-1]      # transmittance before sample j
    w = alpha * Tj
    d_out = (w * z64).sum(1)
    jstar = np.abs(d_out[:, None] - z64).argmin(1)
    rows = np.arange(R)
    g_depth = c["depth"].copy()
    g_w = c["weights"].copy()
    g_z = c["depth_volumes"].copy()
    g_alpha = c["alphas"].copy()
    g_sigma = c["densities"].copy()
    sgn = np.sign(d_out - z64[rows, jstar])
    g_depth += sgn * c["closest_pts_to_depths"]
    g_z[rows, jstar] -= sgn * c["closest_pts_to_depths"]
    g_w[rows, jstar] += c["weights_at_depth"]
    g_w += g_depth[:, None] * z64 + (c["color"][:, None, :] * col).sum(-1)
    g_z += g_depth[:, None] * w
    g_col = c["color"][:, None, :] * w[:, :, None]
    g_alpha += g_w * Tj
    g_T = g_w * alpha
    gTT = g_T * Tj
    suffix = np.cumsum(gTT[:, ::-1], axis=1)[:, ::-1] - gTT                             # sum_{j>k} g_T[j] T[j]
    g_alpha -= suffix / s_
    g_delta = g_alpha * sg * E
    g_sigma += g_alpha * delta * E
    g_t = g_delta.copy()
    g_t[:, :-1] -= g_delta[:, 1:]
    g_t = g_t * (t64 >= 0)                                                              # scenerf.py:707 (never active)
    g_t += g_z * unit[:, 2:3].astype(f64)                                               # depth_volume = t * unit_z for gaussian samples
    # route to the un-sorted samples; only unclamped gaussian samples carry gradient
    g_t_unsorted = np.zeros_like(g_t)
    np.put_along_axis(g_t_unsorted, order, g_t, 1)
    # uniform samples: depth_volume grad does not reach any parameter; gaussian: through t
    gg = g_t_unsorted[:, U:] * (~clamped)
    g_mean = c["gaussian_means"] + gg.reshape(R, G, Pn).sum(-1)
    g_std = c["gaussian_stds"] + (gg * noise_n.astype(f64)).reshape(R, G, Pn).sum(-1)
    # RaySOM KL (ray_som_kl.py:64-92): constants m2 = new_means, s2 = max(sqrt(new_vars), 1.5), mask
    var = (stds ** 2).astype(f32)
    mean_diffs = np.abs(means - som_means)
    var_diffs = np.abs(np.sqrt(var) - np.sqrt(som_vars))
    mask = ((mean_diffs > 0.1) & (som_vars > 0)) & ((var_diffs > 0.1) & (som_vars > 0))
    s2 = np.maximum(np.sqrt(som_vars).astype(f32), f32(1.5)).astype(f64)
    m1, s1, m2 = means.astype(f64), stds.astype(f64), som_means.astype(f64)
    gk = c["loss_kl"][:, None] * mask / G
    g_mean += gk * (m1 - m2) / s2 ** 2
    g_std += gk * (-(s2 / s1 ** 2) / (s2 / s1 + 1e-8) + s1 / s2 ** 2)
    graw_gauss = np.stack([g_mean * (pre_mean > 0), g_std * (pre_std > 0)], axis=-1).reshape(-1, 2)
    # heads of the main MLP
    x3 = m_raw[:, 3].astype(f64) - 1.0
    dsoft = np.where(x3 > 20.0, 1.0, 1.0 / (1.0 + np.exp(-x3)))
    graw_main = np.concatenate([(g_col * col * (1 - col)).reshape(-1, 3), (g_sigma.reshape(-1) * dsoft)[:, None]], axis=1)
    # MLPs + feature maps
    g_main, dz_main, _ = mlp_backward(orc.pm, mp_lat, mp_x, graw_main, tf32=tf32)
    g_gauss, dz_gauss, _ = mlp_backward(orc.pg, gp_lat, gp_x, graw_gauss, tf32=tf32)
    g_pyr = {k: np.zeros(v.shape, f64) for k, v in x_rgb.items()}
    scatter_latent_grad(dz_main, mp_coords, x_rgb, cfg.sphere_W, cfg.sphere_H, g_pyr)
    scatter_latent_grad(dz_gauss, gp_coords, x_rgb, cfg.sphere_W, cfg.sphere_H, g_pyr)
    return dict(out=out, g_main=g_main, g_gauss=g_gauss, g_pyr=g_pyr, graw_main=graw_main, graw_gauss=graw_gauss,
                loss=float(sum((c[k] * out[k].astype(f64)).sum() for k in GRAD_KEYS)))
