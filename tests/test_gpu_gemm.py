"""The two GEMM kernels of the training path against float64 matmul (through the C ABI: srf_debug_gemm).
float32 SIMT: round-off (1e-5 of the row/column norms); wgmma .tf32: 10-bit mantissa operands, bound 2e-3."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _run(M, N, K, use_tf32, bias=False, mask=False, res=False, accumulate=False, splitk=False, seed=0):
    import torch
    from scenerf_b200 import _lib
    lib = _lib.load()
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, K, device="cuda", generator=g)
    B = torch.randn(N, K, device="cuda", generator=g)
    Cm = torch.randn(M, N, device="cuda", generator=g)
    C0 = Cm.clone()
    b = torch.randn(N, device="cuda", generator=g) if bias else None
    mk = torch.randn(M, N, device="cuda", generator=g) if mask else None
    R = torch.randn(M, N, device="cuda", generator=g) if res else None
    ws = torch.empty(4 * 512 * 2528, device="cuda") if splitk else None
    p = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    _lib.check(lib.srf_debug_gemm(p(A), K, p(B), K, p(Cm), N, M, N, K, p(b), p(mk), N, p(R), N, 1 if accumulate else 0, p(ws),
                                  ws.numel() if ws is not None else 0, 1 if use_tf32 else 0,
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    ref = A.double() @ B.double().T
    if bias:
        ref = ref + b.double()
    if mask:
        ref = torch.where(mk > 0, ref, torch.zeros_like(ref))
    if res:
        ref = ref + R.double()
    if accumulate:
        ref = ref + C0.double()
    scale = float((A.double().norm(dim=1)[:, None] * B.double().norm(dim=1)[None, :]).max())
    return float((Cm.double() - ref).abs().max()) / scale


@pytest.mark.parametrize("use_tf32,tol", [(0, 2e-6), (1, 2e-3)])
def test_gemm_shapes(use_tf32, tol):
    assert _run(300, 512, 512, use_tf32) <= tol                                   # ragged M
    assert _run(9472, 512, 512, use_tf32, bias=True, res=True) <= tol             # forward fc shape
    assert _run(1024, 2480, 512, use_tf32, mask=True, accumulate=True) <= tol     # N not a tile multiple (dz shape)
    assert _run(512, 512, 9472, use_tf32, accumulate=True, splitk=True) <= tol    # weight-gradient shape, split-K
    assert _run(512, 240, 1000, use_tf32, splitk=True) <= tol                     # K tail (not a multiple of 32), ragged N
    assert _run(128, 128, 32, use_tf32) <= tol                                    # single stage
