"""The decoder's two kernels entry by entry, through the C ABI (csrc/conv_tf32.cu).

srf_conv3x3_hwc against a float64 convolution of the same tf32 operands, every output entry under the bound
    |got - y| <= tf32_gamma(9 Cin) |scale| S + 2^-22 (|acc scale| + |shift| + |res|),   S = conv(|x|, |w|),
at the edges of the implicit GEMM: Cin not a multiple of the 32-float k-block (TMA zero fill), Cout not a multiple of
the 128-column N tile, ragged and single-pixel M tiles at x0 > 0, dilations that reach past the map, H = 1, W = 1 and
channel strides larger than Cout.  Its output paths bit for bit: round_out, the fp16 copy, stores that leave padding
channels and the row past the end untouched, reruns.  srf_upsample_concat_hwc bit for bit against the oracle.
The CPU tests show that the bound rejects the mistakes such a kernel makes (a dropped tap, k-step or channel block, a
shifted tile, a wrong dilation, a residual read from the wrong pixel)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import tf32_gamma, tf32_rn

EPI = 2.0 ** -22              # float32 epilogue: fmaf(acc, scale, shift), residual add, LeakyReLU
SENT32, SENT16 = 0x7FC0DEAD, 0x7E5A    # NaN bit patterns neither kernel writes

# H, W, Cin (= ld_in), Cout, dil, residual, LeakyReLU slope, operands, padding of ld32 / ld_res (ld16 = Cout + 2 * pad)
CASES = [
    (1, 1, 4, 4, 1, False, 1.0, "tf32", 0),          # one pixel: every tap but the centre reads padding
    (1, 129, 28, 132, 2, True, 0.01, "tf32", 4),     # H = 1; Cin < one k-block; Cout = 128 + 4; a 1-pixel tile at x0 = 128
    (5, 127, 36, 64, 3, True, 0.0, "tf32", 8),       # a second k-block of 4 channels; W one short of a tile
    (3, 128, 128, 256, 1, False, 0.01, "tf32", 4),   # one full M tile, two N tiles
    (2, 385, 260, 4, 3, True, 0.01, "tf32", 4),      # dil >= H: only the middle row of taps sees data; last tile 1 pixel
    (3, 1226, 128, 64, 2, True, 0.01, "tf32", 0),    # config B's level-1_1 width: 9 full tiles and one of 74
    (3, 1226, 36, 132, 3, True, 1.0, "tf32", 4),     # the same width with both channel tails
    (1, 129, 4, 64, 130, False, 0.0, "tf32", 4),     # dil >= W: only the centre tap sees data
    (5, 1, 28, 4, 1, True, 0.01, "tf32", 4),         # W = 1
    (2, 385, 512, 256, 2, True, 0.01, "tf32", 0),    # Cin = 512
    (3, 385, 512, 64, 1, True, 0.01, "nonneg", 4),   # post-ReLU regime: partial sums grow to S, round-off at its worst
    (3, 385, 128, 132, 1, False, 0.01, "fp32", 4),   # unrounded operands: the tensor core reads 10 mantissa bits of each
]


def case_id(c):
    return "%dx%d-cin%d-cout%d-d%d%s-s%g-%s" % (c[0], c[1], c[2], c[3], c[4], "-res" if c[5] else "", c[6], c[7])


def make_case(case, seed=0):
    """CPU float32 operands of one case: x (H,W,Cin), w9 (9,Cout,Cin), scale, shift (Cout), res (H,W,Cout+pad) or None."""
    H, W, cin, cout, dil, has_res, slope, ops, pad = case
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    x, w = rn(H, W, cin), rn(9, cout, cin) / math.sqrt(9 * cin)
    scale = (0.5 + torch.rand(cout, generator=g)) * torch.where(torch.rand(cout, generator=g) < 0.3, -1.0, 1.0)
    shift = 0.1 * rn(cout)
    res = None
    if has_res:
        res = 1e4 + rn(H, W, cout + pad)                  # padding channels far outside the bound, should they be read
        res[..., :cout] = rn(H, W, cout)
    if ops == "nonneg":
        x, w, scale, shift = x.abs(), w.abs(), scale.abs(), shift.abs()
        res = res.abs() if res is not None else None
    if ops != "fp32":                                     # what every production caller feeds the kernel
        x, w = tf32_rn(x), tf32_rn(w)
        res = tf32_rn(res) if res is not None else None
    return dict(x=x, w=w, scale=scale, shift=shift, res=res, dil=dil, slope=slope, cout=cout, cin=cin, pad=pad)


def conv64(x, w, dil):
    """float64 3x3 convolution, padding = dilation = dil: x (H,W,Cin), w (9,Cout,Cin) -> (H,W,Cout)."""
    cout, cin = w.shape[1], w.shape[2]
    xd = x.double().permute(2, 0, 1)[None]
    wd = w.double().view(3, 3, cout, cin).permute(2, 3, 0, 1)          # [tap = ky*3 + kx][co][ci] -> [co][ci][ky][kx]
    return F.conv2d(xd, wd, padding=dil, dilation=dil)[0].permute(1, 2, 0)


def epilogue(acc, d, res):
    pre = acc * d["scale"].double() + d["shift"].double()
    if res is not None:
        pre = pre + res[..., :d["cout"]].double()
    return torch.where(pre > 0, pre, pre * d["slope"])


def accuracy_bound(acc, S, d):
    """Per-entry bound of the float32 result: tf32 accumulation over the k-steps plus the float32 epilogue."""
    sc = d["scale"].double().abs()
    epi = (acc * sc).abs() + d["shift"].double().abs()
    if d["res"] is not None:
        epi = epi + d["res"][..., :d["cout"]].double().abs()
    return tf32_gamma(9 * d["cin"]) * sc * S + EPI * epi, EPI * epi


def ratio(err, bound):
    return float(torch.where(bound > 0, err / bound.clamp(min=1e-300), torch.where(err > 0, math.inf, 0.0)).max())


# --- CPU: the bound rejects the mistakes a tiled implicit GEMM makes -------------------------------------------------
def _shift_x(t):
    """t read one pixel further right: t'[:, x] = t[:, x + 1], zeros past the row."""
    out = torch.zeros_like(t)
    out[:, :-1] = t[:, 1:]
    return out


def _drop_tap(d):
    w = d["w"].clone()
    w[0] = 0                                              # tap (ky, kx) = (0, 0)
    return epilogue(conv64(d["x"], w, d["dil"]), d, d["res"])


def _tile_shift(d):
    y = epilogue(conv64(d["x"], d["w"], d["dil"]), d, d["res"])
    y[:, 128] = epilogue(conv64(_shift_x(d["x"]), d["w"], d["dil"]), d, d["res"])[:, 128]
    return y


def _drop_last_block(d):
    x = d["x"].clone()
    x[..., (d["cin"] - 1) // 32 * 32:] = 0
    return epilogue(conv64(x, d["w"], d["dil"]), d, d["res"])


def _dil_minus_one(d):
    return epilogue(conv64(d["x"], d["w"], d["dil"] - 1), d, d["res"])


def _res_neighbour(d):
    H, W, ld = d["res"].shape
    return epilogue(conv64(d["x"], d["w"], d["dil"]), d, d["res"].reshape(H * W, ld).roll(-1, 0).reshape(H, W, ld))


def _drop_kstep(d):
    w = d["w"].clone()
    w[4, :, 264:272] = 0                                  # centre tap, channels 264..271: one m64n128k8 step
    return epilogue(conv64(d["x"], w, d["dil"]), d, d["res"])


MUTATIONS = [
    ("one tap dropped", _drop_tap, CASES[5]),
    ("one tap dropped", _drop_tap, CASES[2]),
    ("taps of the pixel at x = 128 shifted by one", _tile_shift, CASES[5]),
    ("taps of the pixel at x = 128 shifted by one", _tile_shift, CASES[1]),
    ("last 32-channel block dropped", _drop_last_block, CASES[4]),
    ("last 32-channel block dropped", _drop_last_block, CASES[3]),
    ("dil - 1 in place of dil", _dil_minus_one, CASES[2]),
    ("dil - 1 in place of dil", _dil_minus_one, CASES[5]),
    ("residual read from the neighbouring pixel", _res_neighbour, CASES[1]),
    ("one 8-wide k-step dropped at Cin = 512", _drop_kstep, CASES[9]),
    ("one 8-wide k-step dropped at Cin = 512", _drop_kstep, CASES[10]),
]


@pytest.mark.parametrize("name,mutate,case", MUTATIONS, ids=["%s@%s" % (m[0], case_id(m[2])) for m in MUTATIONS])
def test_bound_rejects_a_wrong_convolution(name, mutate, case):
    d = make_case(case)
    acc = conv64(d["x"], d["w"], d["dil"])
    bound, _ = accuracy_bound(acc, conv64(d["x"].abs(), d["w"].abs(), d["dil"]), d)
    margin = ratio((mutate(d) - epilogue(acc, d, d["res"])).abs(), bound)
    print("%s at %s: rejected, worst err / bound = %.3g" % (name, case_id(case), margin))
    assert margin > 1, (name, margin)


# --- GPU ------------------------------------------------------------------------------------------------------------
def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _conv_gpu(lib, dev, d, H, W, round_out):
    """One srf_conv3x3_hwc call into sentinel-filled out32 / out16 buffers with one guard row; returns their bits."""
    from scenerf_b200 import _lib
    cout, pad = d["cout"], d["pad"]
    ld32, ld16 = cout + pad, cout + 2 * pad
    o32 = torch.full(((H * W + 1) * ld32,), SENT32, dtype=torch.int32, device="cuda")
    o16 = torch.full(((H * W + 1) * ld16,), SENT16, dtype=torch.int16, device="cuda")
    res = dev["res"]
    _lib.check(lib.srf_conv3x3_hwc(dev["x"].data_ptr(), H, W, d["cin"], dev["w"].data_ptr(), cout, d["dil"], dev["scale"].data_ptr(),
                                   dev["shift"].data_ptr(), res.data_ptr() if res is not None else None,
                                   res.shape[-1] if res is not None else 0, d["slope"], round_out, o32.data_ptr(), ld32,
                                   o16.data_ptr(), ld16, _stream()))
    torch.cuda.synchronize()
    return o32.cpu().view(H * W + 1, ld32), o16.cpu().view(H * W + 1, ld16)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_gpu_conv3x3_matches_float64(case):
    from scenerf_b200 import _lib
    lib = _lib.load()
    H, W, cin, cout, dil, _, _, ops, _ = case
    d = make_case(case)
    dev = {k: (d[k].cuda() if d[k] is not None else None) for k in ("x", "w", "scale", "shift", "res")}
    a32, a16 = _conv_gpu(lib, dev, d, H, W, 0)
    b32, b16 = _conv_gpu(lib, dev, d, H, W, 1)
    r32, r16 = _conv_gpu(lib, dev, d, H, W, 0)

    # stores: the padding channels and the row past the end keep their sentinel; reruns are bit-identical
    for buf in (a32, b32):
        assert bool((buf[:, cout:] == SENT32).all()) and bool((buf[-1] == SENT32).all())
    for buf in (a16, b16):
        assert bool((buf[:, cout:] == SENT16).all()) and bool((buf[-1] == SENT16).all())
    assert torch.equal(a32, r32) and torch.equal(a16, r16)
    got_bits = a32[:-1, :cout].contiguous()
    got = got_bits.view(torch.float32)
    # the fp16 copy is fp16_rn of the unrounded float32 result; round_out = 1 stores round_tf32 of it and leaves fp16 alone
    assert torch.equal(a16[:-1, :cout], got.half().view(torch.int16))
    assert torch.equal(b32[:-1, :cout], tf32_rn(got).view(torch.int32))
    assert torch.equal(b16, a16)

    acc = conv64(d["x"], d["w"], dil)
    S = conv64(d["x"].abs(), d["w"].abs(), dil)
    y = epilogue(acc, d, d["res"])
    err = (got.double().view(H, W, cout) - y).abs()
    bound, epi = accuracy_bound(acc, S, d)
    sc_S = d["scale"].double().abs() * S
    if ops == "fp32":
        # unrounded operands: only the tf32 operand precision is promised; show which rounding the tensor core applies
        worst = float((err / sc_S.clamp(min=1e-300)).max())
        trunc = lambda t: (t.contiguous().view(torch.int32) & -8192).view(torch.float32)
        emu = {"truncating": epilogue(conv64(trunc(d["x"]), trunc(d["w"]), dil), d, d["res"]),
               "round-to-nearest": epilogue(conv64(tf32_rn(d["x"]), tf32_rn(d["w"]), dil), d, d["res"])}
        print("%s: max err / (|scale| S) = %.3g vs float64 of the fp32 operands (bound 2^-10 = %.3g); %s" % (
            case_id(case), worst, 2.0 ** -10, ", ".join("%.3g vs a %s tf32 emulation" % (
                float(((got.double().view(H, W, cout) - e).abs() / sc_S.clamp(min=1e-300)).max()), k) for k, e in emu.items())))
        assert worst <= 2.0 ** -10
        return
    unit = math.ceil(9 * cin / 8) * 2.0 ** -24 * sc_S
    c_seen = float(torch.where(unit > 0, (err - epi).clamp(min=0) / unit.clamp(min=1e-300), torch.zeros_like(unit)).max())
    worst = ratio(err, bound)
    y_r = b32[:-1, :cout].contiguous().view(torch.float32).double().view(H, W, cout)
    worst_r = ratio((y_r - y).abs(), bound + 2.0 ** -11 * y.abs())      # round_out = 1: half a tf32 ulp more
    print("%s: worst err / bound = %.3g (round_out: %.3g), accumulation constant seen c = %.3g" % (case_id(case), worst, worst_r, c_seen))
    assert worst <= 1 and worst_r <= 1


# h, w, Cx, ld_x, Cs, ld_skip, H, W, ld_out
UP_CASES = [
    (1, 1, 8, 8, 4, 4, 5, 7, 12),           # one source pixel broadcast
    (4, 6, 5, 8, 3, 4, 1, 1, 12),           # one target pixel
    (9, 13, 6, 6, 0, 0, 4, 5, 8),           # target smaller than the source (align_corners allows it); no skip channels
    (1, 5, 4, 4, 4, 4, 1, 9, 8),            # h = H = 1
    (6, 1, 4, 6, 4, 8, 11, 1, 12),          # w = W = 1
    (3, 10, 16, 20, 12, 16, 6, 20, 32),     # strides larger than the channel counts everywhere
    (23, 77, 12, 12, 4, 4, 46, 153, 16),    # a decoder level: 2x up, W past one 128-pixel tile
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", UP_CASES, ids=["%dx%d-to-%dx%d-cx%d-cs%d" % (c[0], c[1], c[6], c[7], c[2], c[4]) for c in UP_CASES])
def test_gpu_upsample_concat_bit_exact(case):
    from oracle.decoder_oracle import upsample_bilinear_ac
    from scenerf_b200 import _lib
    lib = _lib.load()
    h, w, cx, ldx, cs, lds, H, W, ld = case
    rng = np.random.default_rng(sum(case))
    x = (1e6 + rng.standard_normal((h, w, ldx))).astype(np.float32)        # padding channels: garbage, never read
    x[..., :cx] = rng.standard_normal((h, w, cx))
    skip = (1e6 + rng.standard_normal((H, W, max(lds, 1)))).astype(np.float32)
    skip[..., :cs] = rng.standard_normal((H, W, cs))
    out = torch.full((H * W * ld,), SENT32, dtype=torch.int32, device="cuda")
    dx, ds = torch.from_numpy(x).cuda(), torch.from_numpy(skip).cuda()
    _lib.check(lib.srf_upsample_concat_hwc(dx.data_ptr(), h, w, cx, ldx, ds.data_ptr(), cs, lds, H, W, out.data_ptr(), ld, _stream()))
    torch.cuda.synchronize()
    got = out.cpu().numpy().view(np.uint32).reshape(H, W, ld)
    up = upsample_bilinear_ac(np.ascontiguousarray(x[..., :cx].transpose(2, 0, 1)), H, W).transpose(1, 2, 0)
    want = np.concatenate([up, skip[..., :cs]], axis=2).astype(np.float32)
    want = (want.view(np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)    # RN-tf32, ties away from zero
    bad = int((got[..., :cx + cs] != want).sum())
    assert bad == 0, "%d of %d entries differ" % (bad, want.size)
    assert (got[..., cx + cs:] == 0).all()                                    # padding channels: +0.0
