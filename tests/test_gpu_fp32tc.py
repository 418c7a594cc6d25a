"""GPU: the float32-grade tensor-core mode (precision="fp32tc", SRF_PREC_FP32_TC).

Every fp32 operand of the ResnetFC GEMMs (resnetfc.py:54-63,133-164) is carried as an fp16 hi/lo pair; the tile holds 32
points whose high parts are MMA rows 0-31 and low parts rows 32-63, every weight image is followed by the image of its
low parts, and the epilogue adds accumulator rows r and r+32.  Checked here:
  * layer by layer against a float64 evaluation of the UNROUNDED operands (the raw accumulator dump is recombined as
    (D[r] + D[r+32]) / 2^s) -- localises a wrong image order / scale / lane pairing to the layer;
  * against the strict fp32 SIMT path on many tiles with a ragged tail, at float32 round-off tolerance;
  * zero-chunk skipping stays bit-identical; ragged batches are bit-equal to the prefix of the full batch.
Golden parity of the whole render at the fp32 tolerances is in test_gpu_parity.py (precision "fp32tc")."""
import numpy as np
import pytest

from cases import PREDICT_CASES, RENDER_CASES, load_golden, params_for, pyramid_for
from helpers import make_renderer, torch_pyramid
from oracle import scenerf_oracle as orc

pytestmark = pytest.mark.gpu


def exact_layers(cfg, params, pts, viewdir, x_rgb):
    """dict layer -> accumulator (n,512) in float64 from the float32 operands (no operand rounding)."""
    p = pts.reshape(-1, 3).astype(np.float32)
    inv_K = np.linalg.inv(cfg.K).astype(np.float32)
    coords, _ = orc.sphere_coords_from_pixels(orc.cam_pts_2_pix(p, cfg.K), inv_K, cfg.angles(), cfg.sphere_W, cfg.sphere_H)
    z = orc.gather_latent(x_rgb, coords, cfg.sphere_W, cfg.sphere_H).astype(np.float64)
    x = np.concatenate([orc.positional_encoding(p), np.repeat(viewdir, pts.shape[1], axis=0)], axis=1).astype(np.float64)
    W = lambda n: params[n].astype(np.float64)
    out = {}
    acc = x @ W("lin_in.weight").T + z @ W("lin_z.0.weight").T
    out[1] = acc
    h = acc + W("lin_in.bias") + W("lin_z.0.bias")
    for blk in range(3):
        acc = np.maximum(h, 0) @ W("blocks.%d.fc_0.weight" % blk).T
        out[2 + 3 * blk] = acc
        net = acc + W("blocks.%d.fc_0.bias" % blk)
        acc = np.maximum(net, 0) @ W("blocks.%d.fc_1.weight" % blk).T
        if blk < 2:
            acc = acc + z @ W("lin_z.%d.weight" % (blk + 1)).T
            out[4 + 3 * blk] = acc
            h = h + acc + W("blocks.%d.fc_1.bias" % blk) + W("lin_z.%d.bias" % (blk + 1))
        else:
            out[9] = acc
            h = h + acc + W("blocks.%d.fc_1.bias" % blk)
    o = np.maximum(h, 0) @ W("lin_out.weight").T
    out[10] = o
    out["final"] = o + W("lin_out.bias")
    return out


def blob_scale(net):
    """2^s of a split weight blob (header row 7, entry 256: csrc/mlp_tc.cu kScaleSlot)."""
    import torch
    hdr = net.packed_split[:8 * 512 * 4].view(torch.float32)
    return float(hdr[7 * 512 + 256].item()), float(hdr[7 * 512 + 257].item())


@pytest.mark.parametrize("which", ["mlp", "mlp_gaussian"])
def test_split_tile_program_layer_by_layer(which):
    import torch
    cfg, seed = PREDICT_CASES["predict_adversarial_kitti"]
    g = load_golden("predict_adversarial_kitti")
    pts, vd = g["cam_pts"][:41], g["viewdir"][:41]        # 328 points: 10 tiles of 32 + a ragged one of 8
    pm, pg = params_for(cfg)
    params = pm if which == "mlp" else pg
    exp = exact_layers(cfg, params, pts, vd, pyramid_for(cfg, seed))
    r = make_renderer(cfg, "fp32tc")
    net = r.mlp if which == "mlp" else r.mlp_gaussian
    scale, inv = blob_scale(net)
    wmax = max(float(np.abs(v).max()) for k, v in params.items() if k.endswith("weight"))
    assert scale * inv == 1.0 and 2.0 ** 13 <= wmax * scale < 2.0 ** 14, (scale, wmax)
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    n = pts.shape[0] * pts.shape[1]
    for layer in (1, 2, 4, 5, 7, 8, 9, 10):
        acc = r.debug_tc_layer(which, torch.from_numpy(pts), x_rgb, K, torch.from_numpy(vd), layer)
        torch.cuda.synchronize()
        raw = acc.cpu().numpy().astype(np.float64).reshape(-1, 2, 32, 512)        # (tile, hi/lo part, row, col)
        got = ((raw[:, 0] + raw[:, 1]) * inv).reshape(-1, 512)[:n]
        want = exp[layer]
        ncol = want.shape[1]
        mag = float(np.abs(want).max())
        err = float(np.abs(got[:, :ncol] - want).max())
        lo_share = float(np.abs(raw[:, 1]).max() / max(np.abs(raw[:, 0]).max(), 1e-30))
        print("%s layer %2d: max|acc| %.3e  max-abs-err %.3e (rel %.1e), low-part rows / high-part rows %.1e"
              % (which, layer, mag, err, err / mag, lo_share))
        assert err <= 2e-5 * mag + 1e-6, "layer %d: err %.3e (scale %.3e)" % (layer, err, mag)
        assert lo_share < 2e-3                                 # rows 32..63 really are the 2^-11-sized low parts
    raw = r.predict(which, torch.from_numpy(pts), x_rgb, K, None, torch.from_numpy(vd), output_type="offset")
    got = raw.reshape(n, -1).cpu().numpy()
    want = exp["final"]
    assert np.abs(got - want).max() <= 2e-5 * np.abs(want).max() + 1e-6


def test_fp32tc_vs_fp32_device_paths_large_ragged():
    """split tensor-core path against the strict fp32 SIMT path on the device: 653 tiles of 32 + ragged tail."""
    import torch
    from scenerf_b200 import synth
    cfg, seed = RENDER_CASES["kitti_mini"]
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    n_cols, n_per = 2611, 8                                   # 20888 points
    u = synth.hash_uniform(91, n_cols * n_per * 3).reshape(n_cols, n_per, 3)
    pts = np.stack([u[..., 0] * 25, u[..., 1] * 4, u[..., 2] * 45 + 46], axis=-1).astype(np.float32)
    vd = (synth.hash_uniform(92, n_cols * 3).reshape(n_cols, 3) * 0.7).astype(np.float32)
    outs = {}
    for prec in ("fp32", "fp32tc"):
        r = make_renderer(cfg, prec)
        raw, dbg = r.predict("mlp", torch.from_numpy(pts), x_rgb, K, None, torch.from_numpy(vd), output_type="offset", debug=True)
        torch.cuda.synchronize()
        outs[prec] = (raw.cpu().numpy(), dbg.cpu().numpy())
    assert (outs["fp32"][1] == outs["fp32tc"][1]).all()      # same geometry code -> same sphere pixels
    a, b = outs["fp32tc"][0], outs["fp32"][0]
    assert np.isfinite(a).all()
    err = float(np.abs(a - b).max())
    print("fp32tc vs fp32 SIMT: raw MLP output max-abs-err %.3e (max |out| %.3e)" % (err, np.abs(b).max()))
    assert err <= 2e-5 * max(1.0, float(np.abs(b).max()))


def test_fp32tc_skip_zero_and_single_cta_variants_bit_identical():
    import torch
    cfg, seed = PREDICT_CASES["predict_adversarial_kitti"]
    g = load_golden("predict_adversarial_kitti")
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    args = (torch.from_numpy(g["cam_pts"]), x_rgb, K, None, torch.from_numpy(g["viewdir"]))
    a = make_renderer(cfg, "fp32tc").predict("mlp", *args, output_type="offset")
    b = make_renderer(cfg, "fp32tc", skip_zero_chunks=True).predict("mlp", *args, output_type="offset")
    c = make_renderer(cfg, "fp32tc").predict("mlp", args[0][:1, :3], *args[1:4], args[4][:1], output_type="offset")   # 3 points: 1 tile -> single-CTA kernel
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert torch.equal(c, a[:1, :3])


def test_fp32tc_ragged_batches_bit_equal():
    import torch
    cfg, seed = RENDER_CASES["kitti_mini"]
    r = make_renderer(cfg, "fp32tc")
    x_rgb = torch_pyramid(cfg, seed)
    K, T = torch.from_numpy(cfg.K), torch.from_numpy(cfg.T)
    g = load_golden("kitti_mini")
    noise = (torch.from_numpy(g["noise_u"]), torch.from_numpy(g["noise_n"]))
    full = r.render_rays_batch(K, T, x_rgb, sampled_pixels=torch.from_numpy(g["pixels"]), noise=noise)
    for n in (1, 3, 33):
        part = r.render_rays_batch(K, T, x_rgb, sampled_pixels=torch.from_numpy(g["pixels"][:n]),
                                   noise=(noise[0][:n], noise[1][:n]))
        for k in ("depth", "color", "alphas", "loss_kl"):
            assert torch.equal(part[k], full[k][:n]), (n, k)
