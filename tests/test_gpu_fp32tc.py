"""GPU: the float32-grade tensor-core mode (precision="fp32tc", SRF_PREC_FP32_TC).

Every fp32 operand of the ResnetFC GEMMs (resnetfc.py:54-63,133-164) is carried as an fp16 hi/lo pair along K: a
tile holds 64 points, every A chunk exists as a hi and a lo part, every weight image (of W 2^s) is followed by the
image of its low parts, and each fc layer sums its K in two halves.  Checked here:
  * entry by entry, layer by layer, against the chain-cut emulation of tests/tc_mlp_emul.py (all four hi/lo
    products in float64, bound ACC_C m_L 2^-24 sum|a||w| + 2^-24 |ref| for the two-half add), dense and with the
    latent table, both networks, the shapes of test_gpu_tc_layers.py (ragged tiles, 13 and 1 points per view
    direction, 2 SMs + 1 tiles);
  * against the strict fp32 SIMT path on many tiles with a ragged tail, at float32 round-off tolerance;
  * zero-chunk skipping stays bit-identical; ragged batches are bit-equal to the prefix of the full batch.
Golden parity of the whole render at the fp32 tolerances is in test_gpu_parity.py (precision "fp32tc")."""
import numpy as np
import pytest

import tc_mlp_emul as E
from cases import PREDICT_CASES, RENDER_CASES, load_golden
from helpers import make_renderer, torch_pyramid
from test_gpu_tc_layers import SHAPES, _sms

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("which", ["mlp", "mlp_gaussian"])
@pytest.mark.parametrize("table", [False, True], ids=["dense", "table"])
def test_split_tile_program_per_entry(table, which, shape):
    cfg, seed, pts, vd = E.shape_case(shape, _sms())
    E.check_variant(cfg, seed, "fp32tc", which, pts, vd, pre=table, label=shape)


def test_split_skip_zero_chunks_multitile_per_entry_and_bit_identical():
    import torch
    cfg, seed, pts, vd = E.shape_case("multitile", _sms())
    _, d0, r0 = E.check_variant(cfg, seed, "fp32tc", "mlp", pts, vd, skip=False, label="multitile")
    _, d1, r1 = E.check_variant(cfg, seed, "fp32tc", "mlp", pts, vd, skip=True, label="multitile")
    for L in E.LAYERS:
        assert torch.equal(d0[L].view(torch.int32), d1[L].view(torch.int32)), L
    assert torch.equal(r0, r1)


def test_fp32tc_vs_fp32_device_paths_large_ragged():
    """split tensor-core path against the strict fp32 SIMT path on the device: 326 tiles of 64 + a ragged one of 24."""
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
    """zero-chunk skipping on the adversarial points; 3 points (one tile, one CTA) equal the prefix of the full batch."""
    import torch
    cfg, seed = PREDICT_CASES["predict_adversarial_kitti"]
    g = load_golden("predict_adversarial_kitti")
    x_rgb = torch_pyramid(cfg, seed)
    K = torch.from_numpy(cfg.K)
    args = (torch.from_numpy(g["cam_pts"]), x_rgb, K, None, torch.from_numpy(g["viewdir"]))
    a = make_renderer(cfg, "fp32tc").predict("mlp", *args, output_type="offset")
    b = make_renderer(cfg, "fp32tc", skip_zero_chunks=True).predict("mlp", *args, output_type="offset")
    c = make_renderer(cfg, "fp32tc").predict("mlp", args[0][:1, :3], *args[1:4], args[4][:1], output_type="offset")   # 3 points: 1 tile -> a grid of one CTA
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
