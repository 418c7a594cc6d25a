"""CPU tests of the fp32tc training engine's boundary (SRF_FLAG_FP32TC_MATMUL, matmul="fp32tc"): the flag value, the
Python options, and the argument checks that refuse a bad call before any device work."""
import ctypes as C
import os
import re

import pytest

from scenerf_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(flags):
    cfg = _lib.Config()
    cfg.n_gaussians, cfg.n_pts_uni, cfg.n_pts_per_gaussian = 4, 32, 8
    cfg.sphere_W, cfg.sphere_H = 300, 90
    cfg.precision = _lib.PREC_FP32
    cfg.flags = flags
    return cfg


def _pyramid():
    pyr = _lib.Pyramid()
    for i in range(5):                                   # plausible, never dereferenced
        pyr.hwc[i], pyr.C[i], pyr.H[i], pyr.W[i] = 256, 16, 8, 8
    pyr.format = _lib.PYR_FP32
    return pyr


def test_flag_value_matches_header():
    txt = open(os.path.join(ROOT, "include", "scenerf_b200.h")).read()
    m = re.search(r"#define\s+SRF_FLAG_FP32TC_MATMUL\s+(\d+)", txt)
    assert m and int(m.group(1)) == _lib.FLAG_FP32TC_MATMUL == 16
    assert _lib.FLAG_FP32TC_MATMUL & (_lib.FLAG_TF32_MATMUL | _lib.FLAG_SAVE_ACTIVATIONS | _lib.FLAG_HIDDEN_FP16 |
                                      _lib.FLAG_SKIP_ZERO_CHUNKS) == 0


def test_trainable_renderer_accepts_fp32tc():
    """The matmul option is checked before the renderer is built: "fp32tc" gets past it (and then meets the refusal of a
    CPU device), an unknown engine does not."""
    from scenerf_b200.autograd import TrainableRenderer
    with pytest.raises(RuntimeError, match="CUDA device"):
        TrainableRenderer({}, {}, {}, device="cpu", matmul="fp32tc")
    with pytest.raises(ValueError, match="fp32tc"):
        TrainableRenderer({}, {}, {}, device="cpu", matmul="fp64")


def test_debug_gemm_refuses_unknown_kernel():
    lib = _lib.load()
    p = C.c_void_p(1 << 20)                              # aligned, never dereferenced
    for bad in (3, -1):
        rc = lib.srf_debug_gemm(p, 4, p, 4, p, 4, 4, 4, 4, None, None, 0, None, 0, 0, None, 0, bad, None)
        assert rc == 1 and b"use_tf32" in lib.srf_last_error(), bad


def test_both_matmul_flags_are_refused_before_the_device():
    lib = _lib.load()
    both = _lib.FLAG_SAVE_ACTIVATIONS | _lib.FLAG_TF32_MATMUL | _lib.FLAG_FP32TC_MATMUL
    cfg, pyr, out = _cfg(both), _pyramid(), _lib.Outputs()
    gw = _lib.MlpWeights()
    gp = (C.c_void_p * 5)()
    rc = lib.srf_render_rays_backward(C.byref(cfg), C.byref(pyr), None, None, 4, None, C.byref(out), C.byref(out), None, 0,
                                      C.byref(gw), C.byref(gw), gp, None, 0, None)
    assert rc == 1 and b"SRF_FLAG_FP32TC_MATMUL" in lib.srf_last_error()
    rc = lib.srf_render_rays(C.byref(cfg), C.byref(pyr), None, None, None, 4, None, None, C.byref(out), None, 0, None)
    assert rc == 1 and b"SRF_FLAG_FP32TC_MATMUL" in lib.srf_last_error()
    # one engine flag alone passes this check and stops at the next one (the NULL weights)
    cfg.flags = _lib.FLAG_SAVE_ACTIVATIONS | _lib.FLAG_FP32TC_MATMUL
    rc = lib.srf_render_rays_backward(C.byref(cfg), C.byref(pyr), None, None, 4, None, C.byref(out), C.byref(out), None, 0,
                                      C.byref(gw), C.byref(gw), gp, None, 0, None)
    assert rc == 1 and b"MATMUL" not in lib.srf_last_error()
