"""Novel-view colour evaluation (csrc/color_metrics.cu, scenerf_b200.evaluation / perceptual, DESIGN.md 6.8).  CPU: the
oracle's restatement of skimage's SSIM against a direct box-sum restatement, its edge cases, the LPIPS state-dict parser,
bucket keys and argument validation of the C entries.  GPU: PSNR / SSIM / LPIPS against the oracle, the render presets,
the bucket table, and two ranks."""
import ctypes as C
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np
import pytest

from oracle import color_oracle as O
from scenerf_b200 import _lib
from scenerf_b200.evaluation import color_bucket_key

PSNR_SSIM_SHAPES = ((124, 407), (480, 640), (7, 7), (9, 13))
LPIPS_SHAPES = ((124, 407), (480, 640), (33, 47), (16, 16))     # 16 x 16: stage 5 convolves a 1 x 1 map (only the centre tap)


def u8_image(h, w, seed):
    """A smooth 8-bit image / 255 (what the reference reads from a PNG), with saturated pixels."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = 0.5 + 0.45 * np.sin(x[..., None] / (3.0 + np.arange(3)) + y[..., None] / 5.0 + rng.uniform(0, 6, 3))
    img = np.clip(base + rng.normal(0, 0.05, (h, w, 3)), 0, 1)
    img[rng.random((h, w)) < 0.02] = 1.0
    img[rng.random((h, w)) < 0.02] = 0.0
    return np.floor(img * 255).astype(np.float32) / np.float32(255.0)


def color_pairs(h, w, seed):
    """(img, gt) pairs with all-0 / all-1 channels, constant images (zero variance), saturated pixels and one-ulp
    differences."""
    gt = u8_image(h, w, seed)
    img = u8_image(h, w, seed + 1)
    pairs = [("noisy", img, gt)]
    a = img.copy()
    a[..., 0] = 0.0
    a[..., 2] = 1.0
    pairs.append(("channels_0_1", a, gt))
    pairs.append(("constant", np.full((h, w, 3), 0.25, np.float32), np.full((h, w, 3), 0.75, np.float32)))
    pairs.append(("constant_vs_image", np.full((h, w, 3), 0.5, np.float32), gt))
    ulp = gt.copy()
    flip = np.random.default_rng(seed + 2).random((h, w, 3)) < 0.3
    ulp[flip] = np.nextafter(ulp[flip], np.float32(2.0))
    pairs.append(("one_ulp", ulp, gt))
    return pairs


def box_sum_ssim(X, Y):
    """Direct restatement of skimage 0.18.1 SSIM: 7x7 float64 window sums at the kept interior only."""
    from numpy.lib.stride_tricks import sliding_window_view as win
    out = []
    for ch in range(X.shape[2]):
        x, y = X[..., ch].astype(np.float64), Y[..., ch].astype(np.float64)
        m = lambda z: win(z, (7, 7)).sum(axis=(2, 3)) / 49.0
        ux, uy, uxx, uyy, uxy = m(x), m(y), m(x * x), m(y * y), m(x * y)
        cn = 49 / 48
        vx, vy, vxy = cn * (uxx - ux * ux), cn * (uyy - uy * uy), cn * (uxy - ux * uy)
        C1, C2 = 0.01 ** 2, 0.03 ** 2
        S = ((2 * ux * uy + C1) * (2 * vxy + C2)) / ((ux ** 2 + uy ** 2 + C1) * (vx + vy + C2))
        out.append(S.mean())
    return float(np.mean(out))


def rel(a, b):
    return abs(a - b) / max(abs(b), 1e-300)


# --- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", PSNR_SSIM_SHAPES)
def test_oracle_ssim_equals_direct_box_sum(shape):
    for name, a, b in color_pairs(*shape, seed=sum(shape)):
        assert rel(O.ssim(a, b), box_sum_ssim(a, b)) <= 1e-13, name


def test_oracle_identical_images():
    a = u8_image(33, 47, 5)
    assert O.ssim(a, a) == 1.0
    assert O.psnr(a, a) == np.inf
    assert O.LPIPSOracle(O.random_lpips_state_dict(0))(a, a) == 0.0
    assert O.psnr(a, np.clip(a + np.float32(1 / 255), 0, 1)) > 40


def test_side_below_seven_raises():
    a = np.zeros((6, 20, 3), np.float32)
    with pytest.raises(ValueError):
        O.ssim(a, a)
    with pytest.raises(ValueError):
        O.ssim(a.transpose(1, 0, 2), a.transpose(1, 0, 2))
    from scenerf_b200 import evaluation as E
    with pytest.raises(ValueError):                          # rejected before any device work
        E.compute_ssim(a, a, device="cpu")


def test_lpips_state_dict_parser():
    from scenerf_b200.perceptual import parse_state_dict
    for dropout_index in (True, False):
        sd = O.random_lpips_state_dict(1, dropout_index=dropout_index, with_scaling=dropout_index)
        convs, lins, shift, scale = parse_state_dict(sd)
        assert len(convs) == 13 and [l.numel() for l in lins] == [64, 128, 256, 512, 512]
        assert np.allclose(shift.numpy(), O.SHIFT) and np.allclose(scale.numpy(), O.SCALE)
    sd = O.random_lpips_state_dict(1)
    for key in ("net.slice3.14.weight", "net.slice5.28.bias", "lin4.model.1.weight"):
        broken = dict(sd)
        del broken[key]
        with pytest.raises(KeyError):
            parse_state_dict(broken)
    both = dict(sd)
    both["lin2.model.0.weight"] = sd["lin2.model.1.weight"]
    with pytest.raises(KeyError):
        parse_state_dict(both)


def test_bucket_keys_keep_the_file_name_quirks():
    assert color_bucket_key("kitti", 3.001) == 3 and color_bucket_key("kitti", 3.006) == 4
    assert color_bucket_key("kitti", "3.00") == 3 and color_bucket_key("kitti", 0.0) == 0
    assert color_bucket_key("bf", 2) == "2.00" and color_bucket_key("bf", -10) == "10.00"
    assert sorted([color_bucket_key("bf", 2), color_bucket_key("bf", 10)]) == ["10.00", "2.00"]
    agg = [defaultdict(float) for _ in range(3)] + [defaultdict(int)]
    for k, v in (("10.00", 1.0), ("2.00", 2.0)):
        for j in range(3):
            agg[j][k] += v
        agg[3][k] += 1
    t = O.print_metrics("bf", *agg).splitlines()
    assert t[1].startswith("|10.00|") and t[2].startswith("|2.00|") and t[3] == "|All     |1.500000|1.500000|1.500000|2.000000|"


def test_color_abi_validation():
    lib = _lib.load()
    fake = C.c_void_p(0x1000)
    assert lib.srf_psnr_ssim_workspace_bytes(6, 100) == 0 and lib.srf_psnr_ssim_workspace_bytes(7, 7) > 0
    ws = lib.srf_psnr_ssim_workspace_bytes(124, 407)
    ok = dict(img=fake, gt=fake, h=124, w=407, ws=fake, bytes=ws, rows=fake, slot=0, frame=None, stream=None)
    args = lambda **kw: [kw.get(k, v) for k, v in ok.items()]
    for bad in (dict(img=None), dict(gt=None), dict(h=6), dict(w=6), dict(rows=None), dict(slot=-1)):
        assert lib.srf_psnr_ssim(*args(**bad)) == 1, bad
    assert lib.srf_psnr_ssim(*args(bytes=ws - 1)) == 2 and lib.srf_psnr_ssim(*args(ws=None)) == 2
    assert b"srf_psnr_ssim" in lib.srf_last_error()
    assert lib.srf_lpips_workspace_bytes(15, 100) == 0 and lib.srf_lpips_workspace_bytes(16, 16) > 0
    p13, p5 = (C.c_void_p * 13)(*([0x1000] * 13)), (C.c_void_p * 5)(*([0x1000] * 5))
    sh, sc = (C.c_float * 3)(*O.SHIFT), (C.c_float * 3)(*O.SCALE)
    lws = lib.srf_lpips_workspace_bytes(33, 47)
    good = [fake, fake, 33, 47, p13, p13, p5, sh, sc, fake, lws, fake, None]
    for i, v in ((0, None), (1, None), (2, 15), (3, 9000), (4, None), (7, None), (11, None)):
        a = list(good)
        a[i] = v
        assert lib.srf_lpips_vgg(*a) == 1, i
    a = list(good)
    a[4] = (C.c_void_p * 13)(*([0x1000] * 12 + [0]))
    assert lib.srf_lpips_vgg(*a) == 1 and b"conv 12" in lib.srf_last_error()
    a = list(good)
    a[10] = lws - 1
    assert lib.srf_lpips_vgg(*a) == 2
    # colour mode 3 passes the mode check (then fails for having no buffers); modes 4 and 5 do not
    assert lib.srf_upsample_render(None, None, 4, 4, 8, 8, None, None, 3, None) == 1 and b"nothing to do" in lib.srf_last_error()
    for mode in (4, 5):
        assert lib.srf_upsample_render(None, None, 4, 4, 8, 8, None, None, mode, None) == 1 and b"mode" in lib.srf_last_error()


# --- GPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", PSNR_SSIM_SHAPES)
def test_gpu_psnr_ssim_match_oracle(shape):
    import torch
    from scenerf_b200 import evaluation as E
    for name, a, b in color_pairs(*shape, seed=sum(shape)):
        da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        p, s = E.compute_psnr(da, db), E.compute_ssim(da, db)
        assert rel(p, O.psnr(a, b)) <= 1e-12, (name, p, O.psnr(a, b))
        assert rel(s, O.ssim(a, b)) <= 1e-12, (name, s, O.ssim(a, b))
        assert E.compute_psnr(da, db) == p and E.compute_ssim(da, db) == s          # bit-identical reruns
    a = color_pairs(*shape, seed=1)[0][1]
    assert E.compute_ssim(a, a) == 1.0 and E.compute_psnr(a, a) == np.inf


@pytest.fixture(scope="module")
def lpips_nets():
    import torch
    from scenerf_b200.perceptual import LPIPSVGG
    sd = O.random_lpips_state_dict(7)
    return LPIPSVGG(sd, "cuda:0"), O.LPIPSOracle(sd, device="cuda:0"), torch


@pytest.mark.gpu
@pytest.mark.parametrize("shape", LPIPS_SHAPES)
def test_gpu_lpips_matches_float64_oracle(lpips_nets, shape):
    net, orc, torch = lpips_nets
    gt = u8_image(*shape, 11)
    rng = np.random.default_rng(12)
    rows = []
    for noise in (0.01, 0.05, 0.2):
        img = np.floor(np.clip(gt + noise * rng.standard_normal(gt.shape), 0, 1) * 255).astype(np.float32) / np.float32(255)
        da, db = torch.from_numpy(img).cuda(), torch.from_numpy(gt).cuda()
        v = net(da, db)
        got = float(v.item())
        want, want_tf32 = orc(img, gt), orc(img, gt, tf32=True)
        rows.append((noise, got, want, want_tf32))
        print("lpips %s noise %.2f: gpu %.8g  float64 %.8g (rel %.2e)  tf32-emulated %.8g (rel %.2e)" % (
            shape, noise, got, want, rel(got, want), want_tf32, rel(got, want_tf32)))
        assert abs(got - want) <= max(3e-4 * abs(want), 1e-7), (noise, got, want)
        assert float(net(da, db).item()) == got                                      # bit-identical reruns
    assert float(net(torch.from_numpy(gt).cuda(), torch.from_numpy(gt).cuda()).item()) == 0.0


def _preset_renderer(dataset):
    import torch
    from helpers import make_renderer
    from scenerf_b200 import synth
    cfg = synth.config_A(name="color_kitti") if dataset == "kitti" else synth.config_C(name="color_bf")
    r = make_renderer(cfg, precision="fp16")
    x_rgb = {k: torch.from_numpy(v).cuda() for k, v in synth.make_pyramid(21, cfg.sphere_W, cfg.sphere_H).items()}
    return cfg, r, x_rgb


@pytest.mark.gpu
@pytest.mark.parametrize("dataset", ["kitti", "bf"])
def test_gpu_render_presets(dataset):
    import torch
    from scenerf_b200 import sweep, synth
    cfg, r, x_rgb = _preset_renderer(dataset)
    preset = sweep.RENDER_COLORS_KITTI if dataset == "kitti" else sweep.RENDER_COLORS_BF
    K = torch.from_numpy(cfg.K).cuda()
    sw = sweep.NovelDepthSweep(r, K, x_rgb, **preset)
    R = sw.pixels.shape[0]
    assert R == (407 * 124 if dataset == "kitti" else 320 * 240)
    g = torch.Generator().manual_seed(3)
    noise = (torch.rand(R, cfg.n_pts_uni, generator=g), torch.randn(R, cfg.n_gaussians * cfg.n_pts_per_gaussian, generator=g))
    T = torch.from_numpy(np.ascontiguousarray(cfg.T, dtype=np.float32)).cuda()
    out = r.render_rays_batch(K, T, x_rgb, sampled_pixels=sw.pixels, ray_batch_size=sw.ray_batch_size, noise=noise, outputs="minimal")
    color = out["color"].cpu()
    _, img = sw.render(T, sweep.COLOR_EVAL, noise)
    _, from_rays = sweep.rays_to_images(None, out["color"], sw.grid, sw.out_size, sweep.COLOR_EVAL)
    assert torch.equal(img, from_rays)                     # the render itself repeats with the same noise
    img = img.cpu().numpy()
    if dataset == "kitti":
        assert img.shape == (124, 407, 3)
        # render_colors.py:123-127 + plt.imsave + eval_color.py:93-94
        c = color.reshape(407, 124, 3).transpose(0, 1).clamp(0, 1)
        want = ((c * 255).to(torch.uint8).to(torch.float32) / 255).numpy()
        assert np.array_equal(img, want)
    else:
        assert img.shape == (480, 640, 3)
        c = torch.nn.functional.interpolate(color.reshape(320, 240, 3).permute(2, 1, 0)[None], scale_factor=2, mode="bilinear")
        c = c.clamp(0, 1)[0].permute(1, 2, 0)
        want = ((c * 255).to(torch.uint8).to(torch.float32) / 255).numpy()
        assert (img != want).mean() <= 1e-4                # test_sweep's allowance: 1-ulp blends can cross an integer
        assert np.abs(img - want).max() <= 1 / 255 + 1e-7


def _score_all(dataset, pairs, net, torch):
    """The reference's loop on the oracle's accumulators, fed the device's per-pair values."""
    from scenerf_b200 import evaluation as E
    b = E.ColorErrorBuckets(dataset)
    acc = [defaultdict(float), defaultdict(float), defaultdict(float), defaultdict(int)]
    for img, gt, d in pairs:
        da, db = torch.from_numpy(img).cuda(), torch.from_numpy(gt).cuda()
        lp = net(da, db)
        b.add(da, db, d, lpips=lp)
        name = d if isinstance(d, str) else "{:.2f}".format(d)
        k = O.bucket_key(dataset, name)
        acc[0][k] += E.compute_psnr(da, db)
        acc[1][k] += E.compute_ssim(da, db)
        acc[2][k] += lp.item()
        acc[3][k] += 1
    return b, acc


def color_eval_pairs(dataset, n=6, shape=(40, 56)):
    dists = (3.001, 3.006, 0.4, 3.001, 1.0, 0.0) if dataset == "kitti" else ("2.00", "10.00", "2.00", "0.00", "10.00", "4.00")
    out = []
    for i in range(n):
        gt = u8_image(*shape, 50 + i)
        img = gt if i == 3 else u8_image(*shape, 60 + i)
        out.append((img, gt, dists[i]))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dataset", ["kitti", "bf"])
def test_gpu_bucket_table_equals_reference_text(lpips_nets, dataset):
    net, _, torch = lpips_nets
    b, acc = _score_all(dataset, color_eval_pairs(dataset), net, torch)
    assert b.table() == O.print_metrics(dataset, *acc)
    keys = [line.split("|")[1] for line in b.table().splitlines()[1:-1]]
    if dataset == "kitti":
        assert keys == ["00000000", "00000001", "00000003", "00000004"]
    else:
        assert keys == ["0.00", "10.00", "2.00", "4.00"]
    half = [_score_all(dataset, color_eval_pairs(dataset)[i::2], net, torch)[0] for i in (0, 1)]
    merged = half[0].merge(half[1]).as_dicts()
    for j in range(3):
        for k, v in acc[j].items():
            assert merged[j][k] == pytest.approx(v, rel=1e-12, abs=0) or (np.isinf(v) and merged[j][k] == v)
    assert merged[3] == dict(acc[3])


@pytest.mark.gpu
def test_gpu_two_ranks_get_identical_rows():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29747", os.path.join(here, "_color_dist_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "COLOR_DIST_OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
