"""GPU: the fp16 wgmma tile program (csrc/mlp_tc.cu, precision "fp16") checked entry by entry, layer by layer.

After each accumulator-complete point of the fused kernel the raw fp32 accumulator is dumped (srf_debug_tc_layer) and
every entry is compared with the chain-cut emulation of tests/tc_mlp_emul.py: the layer's A operand is rebuilt in
float32 from the dumps of the layers before it, the reference and the bound ACC_C m_L 2^-24 sum|a||w| are float64.
All four fp16 kernel variants (fp16 / fp32 hidden state, dense / latent table), both networks, shapes that hit the
kernel's edges: the adversarial goldens, n = 1, n % 64 of 1 and 63, 13 and 1 points per view direction, and 2 SMs + 1
tiles whose CTAs run tiles with different live lin_z chunks."""
import numpy as np
import pytest

import tc_mlp_emul as E
from cases import PREDICT_CASES, RENDER_CASES, load_golden
from helpers import make_renderer, torch_pyramid

pytestmark = pytest.mark.gpu

SHAPES = ("adv_kitti", "adv_bf", "n1", "n65_per13", "n127_per1", "multitile")


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("which", ["mlp", "mlp_gaussian"])
@pytest.mark.parametrize("h16,table", [(True, False), (False, False), (True, True), (False, True)],
                         ids=["h16", "h32", "h16-table", "h32-table"])
def test_tile_program_per_entry(h16, table, which, shape):
    cfg, seed, pts, vd = E.shape_case(shape, _sms())
    E.check_variant(cfg, seed, "fp16", which, pts, vd, h16=h16, pre=table, label=shape)


def test_skip_zero_chunks_multitile_per_entry_and_bit_identical():
    """2 SMs + 1 tiles with different live lin_z chunks per tile: with and without zero-chunk skipping both pass the
    per-entry check, and every dump and the output are bit-identical."""
    import torch
    cfg, seed, pts, vd = E.shape_case("multitile", _sms())
    _, d0, r0 = E.check_variant(cfg, seed, "fp16", "mlp", pts, vd, skip=False, label="multitile")
    _, d1, r1 = E.check_variant(cfg, seed, "fp16", "mlp", pts, vd, skip=True, label="multitile")
    for L in E.LAYERS:
        assert torch.equal(d0[L].view(torch.int32), d1[L].view(torch.int32)), L
    assert torch.equal(r0, r1)


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
