"""GPU: the wgmma tile program checked layer by layer.  After each accumulator-complete point of the fused kernel
the raw fp32 accumulator is dumped (srf_debug_tc_layer) and compared with a float64 emulation that applies the
same fp16 operand rounding (oracle geometry / gather / positional encoding + numpy matmuls).  This localises a wrong
shared-memory descriptor, swizzle, weight image or epilogue to the exact layer."""
import numpy as np
import pytest

from cases import PREDICT_CASES, RENDER_CASES, load_golden, params_for, pyramid_for
from helpers import make_renderer, torch_pyramid
from oracle import scenerf_oracle as orc

pytestmark = pytest.mark.gpu


def q16(a):
    return np.asarray(a, dtype=np.float32).astype(np.float16).astype(np.float64)


def emulate(cfg, params, pts, viewdir, x_rgb):
    """dict layer -> expected accumulator (n,512) with fp16-rounded operands, float64 accumulation."""
    p = pts.reshape(-1, 3).astype(np.float32)
    inv_K = np.linalg.inv(cfg.K).astype(np.float32)
    coords, _ = orc.sphere_coords_from_pixels(orc.cam_pts_2_pix(p, cfg.K), inv_K, cfg.angles(), cfg.sphere_W, cfg.sphere_H)
    # tensor-core mode stores the packed pyramid as fp16 (features rounded once at pack time)
    x16 = {k: np.asarray(v, dtype=np.float32).astype(np.float16).astype(np.float32) for k, v in x_rgb.items()}
    z = q16(orc.gather_latent(x16, coords, cfg.sphere_W, cfg.sphere_H))
    x = q16(np.concatenate([orc.positional_encoding(p), np.repeat(viewdir, pts.shape[1], axis=0)], axis=1))
    W = lambda n: q16(params[n])
    b = lambda n: params[n].astype(np.float64)
    out = {}
    acc = x @ W("lin_in.weight").T + z @ W("lin_z.0.weight").T
    out[1] = acc
    h = acc + b("lin_in.bias") + b("lin_z.0.bias")
    for blk in range(3):
        # default tensor-core mode (SRF_FLAG_HIDDEN_FP16): the residual hidden state is stored as fp16 between blocks;
        # the activation fed to fc_0 is relu(h) rounded to fp16, identical with or without that storage rounding
        h_act = h
        h = q16(h)
        acc = q16(np.maximum(h_act, 0)) @ W("blocks.%d.fc_0.weight" % blk).T
        out[2 + 3 * blk] = acc
        net = acc + b("blocks.%d.fc_0.bias" % blk)
        acc = q16(np.maximum(net, 0)) @ W("blocks.%d.fc_1.weight" % blk).T
        if blk < 2:
            acc = acc + z @ W("lin_z.%d.weight" % (blk + 1)).T
            out[4 + 3 * blk] = acc
            h = h + acc + b("blocks.%d.fc_1.bias" % blk) + b("lin_z.%d.bias" % (blk + 1))
        else:
            out[9] = acc
            h = h + acc + b("blocks.%d.fc_1.bias" % blk)
    o = q16(np.maximum(h, 0)) @ W("lin_out.weight").T
    out[10] = o
    out["final"] = o + b("lin_out.bias")
    return out


@pytest.mark.parametrize("which", ["mlp", "mlp_gaussian"])
def test_tile_program_layer_by_layer(which):
    import torch
    cfg, seed = PREDICT_CASES["predict_adversarial_kitti"]
    g = load_golden("predict_adversarial_kitti")
    pts, vd = g["cam_pts"][:41], g["viewdir"][:41]        # 41 x 8 = 328 points: 6 tiles of 64, last one ragged
    pm, pg = params_for(cfg)
    params = pm if which == "mlp" else pg
    exp = emulate(cfg, params, pts, vd, pyramid_for(cfg, seed))
    r = make_renderer(cfg, "fp16")
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    n = pts.shape[0] * pts.shape[1]
    for layer in (1, 2, 4, 5, 7, 8, 9, 10):
        acc = r.debug_tc_layer(which, torch.from_numpy(pts), x_rgb, K, torch.from_numpy(vd), layer)
        torch.cuda.synchronize()
        got = acc.cpu().numpy()[:n]
        want = exp[layer]
        ncol = want.shape[1]
        scale = float(np.abs(want).max())
        err = float(np.abs(got[:, :ncol] - want).max())
        print("%s layer %2d: max|acc| %.3e  max-abs-err %.3e" % (which, layer, scale, err))
        assert err <= 2e-3 * scale + 1e-4, "layer %d: err %.3e (scale %.3e)" % (layer, err, scale)
    raw = r.predict(which, torch.from_numpy(pts), x_rgb, K, None, torch.from_numpy(vd), output_type="offset")
    got = raw.reshape(n, -1).cpu().numpy()
    want = exp["final"]
    assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max() + 1e-4


def test_fp16_vs_fp32_device_paths_large_ragged():
    """tensor-core path against the strict fp32 SIMT path on the device, many tiles + ragged tail + more tiles than SMs."""
    import torch
    from scenerf_b200 import synth
    cfg, seed = RENDER_CASES["kitti_mini"]
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    n_cols, n_per = 2611, 8                                   # 20888 points = 326 tiles of 64 + 24 rows
    u = synth.hash_uniform(91, n_cols * n_per * 3).reshape(n_cols, n_per, 3)
    pts = np.stack([u[..., 0] * 25, u[..., 1] * 4, u[..., 2] * 45 + 46], axis=-1).astype(np.float32)
    vd = (synth.hash_uniform(92, n_cols * 3).reshape(n_cols, 3) * 0.7).astype(np.float32)
    outs = {}
    for prec in ("fp32", "fp16"):
        r = make_renderer(cfg, prec)
        d, c = r.predict("mlp", torch.from_numpy(pts), x_rgb, K, None, torch.from_numpy(vd))
        torch.cuda.synchronize()
        outs[prec] = (d.cpu().numpy(), c.cpu().numpy())
    assert np.isfinite(outs["fp16"][0]).all()
    d_err = np.abs(outs["fp16"][0] - outs["fp32"][0]).max()
    c_err = np.abs(outs["fp16"][1] - outs["fp32"][1]).max()
    print("fp16 vs fp32: density max-abs-err %.3e (max %.3e), colour max-abs-err %.3e" % (d_err, outs["fp32"][0].max(), c_err))
    assert d_err <= 1e-2 * max(1.0, outs["fp32"][0].max()) and c_err <= 5e-3


def test_skip_zero_chunks_is_bit_identical():
    import torch
    cfg, seed = PREDICT_CASES["predict_adversarial_kitti"]
    g = load_golden("predict_adversarial_kitti")
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    a = make_renderer(cfg, "fp16").predict("mlp", torch.from_numpy(g["cam_pts"]), x_rgb, K, None,
                                            torch.from_numpy(g["viewdir"]), output_type="offset")
    b = make_renderer(cfg, "fp16", skip_zero_chunks=True).predict("mlp", torch.from_numpy(g["cam_pts"]), x_rgb, K, None,
                                                                  torch.from_numpy(g["viewdir"]), output_type="offset")
    torch.cuda.synchronize()
    assert torch.equal(a, b)


def test_fp16_and_fp32_pyramid_storage_agree():
    """tensor-core mode with the packed pyramid stored as fp16 (default) vs fp32: both within the fp16-mode tolerance
    of the strict fp32 path; the storage format must not change a sphere-pixel decision."""
    import torch
    cfg, seed = PREDICT_CASES["predict_adversarial_kitti_full"]
    g = load_golden("predict_adversarial_kitti_full")
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    pts, vd = torch.from_numpy(g["cam_pts"]), torch.from_numpy(g["viewdir"])
    ref = make_renderer(cfg, "fp32").predict("mlp", pts, x_rgb, K, None, vd, output_type="offset").cpu().numpy()
    outs = {}
    for fp16_pyr, fp16_hid in ((True, True), (False, False), (True, False)):
        r = make_renderer(cfg, "fp16", pyramid_fp16=fp16_pyr, hidden_fp16=fp16_hid)
        raw, dbg = r.predict("mlp", pts, x_rgb, K, None, vd, output_type="offset", debug=True)
        outs[(fp16_pyr, fp16_hid)] = (raw.cpu().numpy(), dbg.cpu().numpy())
    assert (outs[(True, True)][1] == outs[(False, False)][1]).all()
    scale = max(1.0, np.abs(ref).max())
    for k, (raw, _) in outs.items():
        assert np.abs(raw - ref).max() <= 1e-2 * scale, k
