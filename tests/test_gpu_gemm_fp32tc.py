"""The split 3xTF32 GEMM (srf_debug_gemm(..., use_tf32=2), the kernel of matmul="fp32tc") against float64 matmul, entry by
entry, on RAW float32 operands -- handling operands that are not tf32 values is what the split is for.

Bound.  The kernel computes a.b as hi_a hi_b + hi_a lo_b + lo_a hi_b with hi = trunc_tf32(x) (what wgmma .tf32 reads of
x) and lo = x - hi, itself truncated to tf32 by the tensor core (csrc/tma.cuh).  |lo| < 2^-10 |x| and that truncation
loses < 2^-20 |x|, so the dropped lo_a lo_b and the two truncated lo operands leave < 3 2^-20 |a||b| per product.  The
tensor core's accumulator truncates once per MMA (tf32_gamma's TF32_ACC_C per MMA); the kernel runs the 12 MMAs of a
32-wide k-block into a fresh partial and adds the partials in float32, rounded to nearest: <= 2 ceil(K/32) such adds on
a path through the sum, split-K's fixed-order reduce included.  Per entry:
    |err| <= (3 2^-20 + (12 TF32_ACC_C + 2 ceil(K/32)) 2^-24) (|A||B|^T) + 2^-22 |epilogue terms|
-- tighter than the SIMT kernel's K 2^-24 (|A||B|^T) from K = 96 on.  Non-vacuity: the plain tf32 kernel (use_tf32=1) on
the same raw operands breaks it on every shape, so a split kernel that dropped its correction products would fail here."""
import ctypes as C
import math

import pytest

from helpers import TF32_ACC_C, tf32_rn
from test_gpu_gemm import EPI, SHAPES


def split_gamma(K):
    return 3.0 * 2.0 ** -20 + (12 * TF32_ACC_C + 2 * math.ceil(K / 32)) * 2.0 ** -24


def _gemm(lib, A, B, Cm, lda, M, N, K, kernel, b=None, mk=None, R=None, accumulate=False, ws=None):
    import torch
    from scenerf_b200 import _lib
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(lib.srf_debug_gemm(p(A), lda, p(B), lda, p(Cm), N, M, N, K, p(b), p(mk), N, p(R), N, 1 if accumulate else 0, p(ws),
                                  ws.numel() if ws is not None else 0, kernel, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()


def _run(kernel, M, N, K, bias=False, mask=False, res=False, accumulate=False, splitk=False, lda=None, seed=0):
    """Raw float32 operands (columns K..lda-1 NaN, never read).  Returns (worst err / split bound, max |err| / max_ij
    |A_i||B_j|)."""
    import torch
    from scenerf_b200 import _lib
    lib = _lib.load()
    lda = lda or K
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.full((M, lda), math.nan, device="cuda")
    B = torch.full((N, lda), math.nan, device="cuda")
    A[:, :K] = torch.randn(M, K, device="cuda", generator=g)
    B[:, :K] = torch.randn(N, K, device="cuda", generator=g)
    Cm = torch.randn(M, N, device="cuda", generator=g)
    C0 = Cm.clone()
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    mk = torch.randn(M, N, device="cuda", generator=g) if mask else None
    R = torch.randn(M, N, device="cuda", generator=g) if res else None
    ws = torch.empty(4 * 512 * 2528, device="cuda") if splitk else None
    _gemm(lib, A, B, Cm, lda, M, N, K, kernel, b, mk, R, accumulate, ws)
    A64, B64 = A[:, :K].double(), B[:, :K].double()
    acc = A64 @ B64.T
    keep = (mk > 0).double() if mask else torch.ones_like(acc)
    bias64 = b.double().expand_as(acc) if bias else torch.zeros_like(acc)
    ref = keep * (acc + bias64)
    epi = torch.zeros_like(acc)
    if res:
        ref, epi = ref + R.double(), epi + R.double().abs()
    if accumulate:
        ref, epi = ref + C0.double(), epi + C0.double().abs()
    err = (Cm.double() - ref).abs()
    bound = keep * (split_gamma(K) * (A64.abs() @ B64.abs().T) + EPI * (acc.abs() + bias64.abs())) + EPI * epi
    normwise = float(err.max()) / float((A64.norm(dim=1)[:, None] * B64.norm(dim=1)[None, :]).max())
    return float((err / bound).max()), normwise


NORMWISE = 1e-5       # the split kernel stays below ~3e-6 here, the plain tf32 kernel on raw operands above ~3e-5


@pytest.mark.gpu
def test_split_gemm_meets_the_float32_grade_bound():
    """Every shape of test_gpu_gemm.SHAPES: ragged M / N / K, the forward fc shape with bias + residual, split-K, the whole
    epilogue offered a split-K workspace, M = 1."""
    for shape in SHAPES:
        worst, normwise = _run(2, **shape)
        print("fp32tc %s: worst err / bound %.3g, norm-relative err %.3g" % (shape, worst, normwise))
        assert worst <= 1 and normwise <= NORMWISE, shape


@pytest.mark.gpu
def test_plain_tf32_breaks_the_split_bound_on_raw_operands():
    """Non-vacuity: hi.hi alone (the tf32 kernel), whose operand truncation costs ~1.4e-3 |result| on average, on the
    same raw operands: every shape breaks the per-entry bound, and the norm-relative error separates the two kernels."""
    for shape in SHAPES:
        worst, normwise = _run(1, **shape)
        print("tf32 on raw operands %s: worst err / split bound %.3g, norm-relative err %.3g" % (shape, worst, normwise))
        assert worst > 1 and normwise > NORMWISE, shape


@pytest.mark.gpu
def test_split_gemm_non_finite_entries_match_simt():
    """Inf and NaN in A (and an Inf in B) give the SIMT kernel's non-finite entries, with the same signs: Inf * 0 = NaN
    where an operand is 0, +-Inf where the partner is a tf32 value (its lo part would be exactly 0) or any other finite
    value.  The finite entries stay within the split bound."""
    import torch
    from scenerf_b200 import _lib
    lib = _lib.load()
    M, N, K = 96, 136, 100
    g = torch.Generator(device="cuda").manual_seed(5)
    A = torch.randn(M, K, device="cuda", generator=g)
    B = torch.randn(N, K, device="cuda", generator=g)
    B[: N // 2] = tf32_rn(B[: N // 2])                   # rows whose lo part is 0
    A[5, 17], A[9, 3], A[20, 40] = math.inf, -math.inf, math.nan
    B[2, 17] = 0.0                                       # (5, 2): Inf * 0
    B[100, 60] = math.inf                                # column 100: Inf; (11, 100): 0 * Inf; (12, 100): a tf32 value
    A[11, 60], A[12, 60] = 0.0, 1.5
    out = {}
    for kernel in (0, 2):
        Cm = torch.zeros(M, N, device="cuda")
        _gemm(lib, A, B, Cm, K, M, N, K, kernel)
        out[kernel] = Cm
    s, f = out[0], out[2]
    assert torch.isnan(s[5, 2]) and torch.isnan(s[11, 100]) and torch.isnan(s[20]).all()
    assert torch.isinf(s[5, 0]) and torch.isinf(s[12, 100]) and torch.isinf(s[9, N // 2 - 1])
    for what in (torch.isnan, torch.isposinf, torch.isneginf):
        assert torch.equal(what(f), what(s)), what.__name__
    fin = torch.isfinite(s)
    assert int((~fin).sum()) >= 3 * N + M - 3
    A64, B64 = A.double(), B.double()
    A64[~torch.isfinite(A64)] = 0
    B64[~torch.isfinite(B64)] = 0
    acc = A64 @ B64.T
    err = (f.double() - acc).abs()[fin]
    bound = (split_gamma(K) * (A64.abs() @ B64.abs().T) + EPI * acc.abs())[fin]
    assert float((err / bound).max()) <= 1
