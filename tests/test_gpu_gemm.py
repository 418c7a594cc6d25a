"""The two GEMM kernels of the training path against float64 matmul (through the C ABI: srf_debug_gemm), entry by entry.
float32 SIMT: |err| <= K 2^-24 (|A||B|^T) + 2^-22 |epilogue terms|.  wgmma .tf32 on operands that are tf32 values (what the
training path feeds it): |err| <= tf32_gamma(K) (|A||B|^T) + 2^-22 |epilogue terms| (helpers.tf32_gamma, the bound of
test_gpu_conv.py).  The norm-relative error of the first version of this test, max |err| / max_ij |A_i||B_j|, stays
asserted as well; at the weight-gradient shape it admits a whole dropped k-step (test_old_bound_misses_a_dropped_k_step)."""
import ctypes as C
import math

import numpy as np
import pytest

from helpers import tf32_gamma, tf32_rn

EPI = 2.0 ** -22


def per_entry_bound(A, B, acc, use_tf32, keep, epi_kept, epi):
    """float64 bound of each entry: accumulation (scaled by |A||B|^T) and epilogue; `keep` zeroes what the ReLU mask drops."""
    K = A.shape[1]
    gamma = tf32_gamma(K) if use_tf32 else K * 2.0 ** -24
    return keep * (gamma * (A.abs() @ B.abs().T) + EPI * (acc.abs() + epi_kept)) + EPI * epi


def _run(M, N, K, use_tf32, bias=False, mask=False, res=False, accumulate=False, splitk=False, lda=None, seed=0):
    """Returns (worst err / per-entry bound, max |err| / max_ij |A_i||B_j|)."""
    import torch
    from scenerf_b200 import _lib
    lib = _lib.load()
    lda = lda or K                                        # also ldb; columns K..lda-1 hold NaN and must never be read
    g = torch.Generator(device="cuda").manual_seed(seed)
    rt = tf32_rn if use_tf32 else (lambda t: t)
    A = torch.full((M, lda), math.nan, device="cuda")
    B = torch.full((N, lda), math.nan, device="cuda")
    A[:, :K] = rt(torch.randn(M, K, device="cuda", generator=g))
    B[:, :K] = rt(torch.randn(N, K, device="cuda", generator=g))
    Cm = rt(torch.randn(M, N, device="cuda", generator=g))
    C0 = Cm.clone()
    b = rt(torch.randn(N, device="cuda", generator=g)) if bias else None
    mk = torch.randn(M, N, device="cuda", generator=g) if mask else None
    R = rt(torch.randn(M, N, device="cuda", generator=g)) if res else None
    ws = torch.empty(4 * 512 * 2528, device="cuda") if splitk else None
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(lib.srf_debug_gemm(p(A), lda, p(B), lda, p(Cm), N, M, N, K, p(b), p(mk), N, p(R), N, 1 if accumulate else 0, p(ws),
                                  ws.numel() if ws is not None else 0, 1 if use_tf32 else 0,
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
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
    bound = per_entry_bound(A64, B64, acc, use_tf32, keep, bias64.abs(), epi)
    normwise = float(err.max()) / float((A64.norm(dim=1)[:, None] * B64.norm(dim=1)[None, :]).max())
    return float((err / bound).max()), normwise


SHAPES = [
    dict(M=300, N=512, K=512),                                       # ragged M
    dict(M=9472, N=512, K=512, bias=True, res=True),                 # forward fc shape
    dict(M=1024, N=2480, K=512, mask=True, accumulate=True),         # N not a tile multiple (dz shape)
    dict(M=512, N=512, K=9472, accumulate=True, splitk=True),        # weight-gradient shape, split-K
    dict(M=512, N=240, K=1000, splitk=True),                         # K tail (not a multiple of 32), ragged N
    dict(M=128, N=128, K=32),                                        # single stage
    dict(M=300, N=132, K=4),                                         # one partial k-block; N = 128 + 4
    dict(M=200, N=4, K=33, lda=36),                                  # K tail inside the first k-block; N = 4
    dict(M=1, N=256, K=512),                                         # M = 1
    dict(M=200, N=132, K=512, lda=516),                              # row stride K + 4
    # workspace offered with the whole epilogue: the kernel must not split (the slices carry no epilogue)
    dict(M=512, N=512, K=9472, bias=True, mask=True, res=True, accumulate=True, splitk=True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("use_tf32,tol", [(0, 2e-6), (1, 2e-3)])
def test_gemm_shapes(use_tf32, tol):
    for shape in SHAPES:
        worst, normwise = _run(use_tf32=use_tf32, **shape)
        print("%s %s: worst err / bound %.3g, norm-relative err %.3g" % ("tf32" if use_tf32 else "simt", shape, worst, normwise))
        assert worst <= 1 and normwise <= tol, shape


def test_old_bound_misses_a_dropped_k_step():
    """CPU: at the weight-gradient K, a result with one 8-wide k-step missing passes the norm-relative bound and fails
    the per-entry one."""
    import torch
    g = torch.Generator().manual_seed(0)
    M, N, K = 64, 64, 9472
    A, B = tf32_rn(torch.randn(M, K, generator=g)).double(), tf32_rn(torch.randn(N, K, generator=g)).double()
    acc = A @ B.T
    B_drop = B.clone()
    B_drop[:, 4096:4104] = 0
    err = (A @ B_drop.T - acc).abs()
    normwise = float(err.max()) / float((A.norm(dim=1)[:, None] * B.norm(dim=1)[None, :]).max())
    ones = torch.ones_like(acc)
    margin = float((err / per_entry_bound(A, B, acc, True, ones, 0 * ones, 0 * ones)).max())
    print("dropped k-step at K = %d: norm-relative err %.3g (old bound 2e-3: accepted), worst err / per-entry bound %.3g (rejected)"
          % (K, normwise, margin))
    assert normwise <= 2e-3 and margin > 1
