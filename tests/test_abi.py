"""CPU tests of the drop-in boundary: the shared library builds/loads without a GPU and exports exactly the symbols
include/scenerf_b200.h declares; argument validation works without touching the device."""
import ctypes as C
import os
import re

import pytest

from scenerf_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    txt = open(os.path.join(ROOT, "include", "scenerf_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return set(re.findall(r"\b(srf_[a-z0-9_]+)\s*\(", txt))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    declared = _declared_symbols()
    assert declared, "header parse found nothing"
    assert declared == set(_lib.SYMBOLS), "binding and header disagree: %s" % (declared ^ set(_lib.SYMBOLS))
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.srf_abi_version() == _lib.ABI_VERSION == 2


def test_struct_layouts_match_header_sizes():
    # the library reports sizeof() of each ABI struct; the ctypes mirror must agree (guards against binding drift)
    lib = _lib.load()
    for which, st in enumerate((_lib.Config, _lib.Pyramid, _lib.MlpWeights, _lib.Outputs)):
        assert lib.srf_sizeof(which) == C.sizeof(st), st.__name__
    assert C.sizeof(_lib.Outputs) == 15 * 8


def test_argument_validation_without_gpu():
    lib = _lib.load()
    cfg = _lib.Config()
    cfg.n_gaussians = 99
    cfg.n_pts_uni = 32
    cfg.n_pts_per_gaussian = 8
    out = _lib.Outputs()
    rc = lib.srf_render_rays(C.byref(cfg), None, None, None, None, 4, None, None, C.byref(out), None, 0, None)
    assert rc == 1 and b"n_gaussians" in lib.srf_last_error()
    with pytest.raises(ValueError):
        _lib.check(rc)
    cfg.n_gaussians = 4
    cfg.sphere_W, cfg.sphere_H = 300, 90
    cfg.precision = 7
    rc = lib.srf_render_rays(C.byref(cfg), None, None, None, None, 4, None, None, C.byref(out), None, 0, None)
    assert rc == 1 and b"precision" in lib.srf_last_error()
    cfg.precision = 0
    assert lib.srf_render_workspace_bytes(C.byref(cfg), 1024) > 1024 * 64 * 4 * 9


def test_renderer_refuses_cpu():
    import torch
    from scenerf_b200.renderer import B200Renderer
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        B200Renderer({}, {}, {}, device="cpu")


def test_argument_validation_of_the_next_rows_without_gpu():
    """TSDF, sweep glue, sphere resampling, backward and the diagnostic GEMM reject bad arguments before any device call."""
    lib = _lib.load()
    dims = (C.c_int * 3)(8, 8, 4)
    assert lib.srf_tsdf_reset(None, None, None, dims, None) == 1 and b"srf_tsdf_reset" in lib.srf_last_error()
    origin = (C.c_float * 3)(0, 0, 0)
    assert lib.srf_tsdf_integrate(None, None, None, dims, origin, 0.2, None, None, None, None, 0, 4, 4, 10.0, 1.0, None) == 1
    assert lib.srf_tsdf_merge(None, None, None, None, None, None, dims, None) == 1
    assert lib.srf_upsample_render(None, None, 4, 4, 8, 8, None, None, 5, None) == 1 and b"mode" in lib.srf_last_error()
    assert lib.srf_upsample_render(None, None, 4, 4, 8, 8, None, None, 1, None) == 1 and b"nothing to do" in lib.srf_last_error()
    w, h = C.c_int(0), C.c_int(0)
    lib.srf_sphere_feature_dims(1500, 452, 8, C.byref(w), C.byref(h))          # round(187.5) = 188, round(56.5) = 56 (half to even)
    assert (w.value, h.value) == (188, 56)
    lib.srf_sphere_feature_dims(1500, 452, 16, C.byref(w), C.byref(h))
    assert (w.value, h.value) == (94, 28)
    assert lib.srf_sphere_feature(None, 4, 4, 4, None, None, 0, 1, 16, 16, None, 0, None, 0, None) == 1
    assert lib.srf_debug_gemm(None, 4, None, 4, None, 4, 4, 4, 4, None, None, 0, None, 0, 0, None, 0, 1, None) == 1
    # the convolution launches one CTA per 128-pixel row segment in gridDim.y (at most 65535): a 4096 x 2048 map (65536
    # segments, inside the sphere grid's 16384 limit) is refused before any tensor map is encoded; the aligned pointers
    # are never dereferenced
    p = C.c_void_p(1 << 20)
    for H, W in ((4096, 2048), (65536, 1), (1, 1 << 30)):
        rc = lib.srf_conv3x3_hwc(p, H, W, 64, p, 64, 1, p, p, None, 0, 1.0, 0, p, 64, None, 0, None)
        assert rc == 1 and b"65535" in lib.srf_last_error(), (H, W)
    cfg = _lib.Config()
    cfg.n_gaussians, cfg.n_pts_uni, cfg.n_pts_per_gaussian = 4, 32, 8
    cfg.sphere_W, cfg.sphere_H = 300, 90
    cfg.precision = 1                                                           # tensor-core inference precision
    pyr, out = _lib.Pyramid(), _lib.Outputs()
    for i in range(5):                                                          # a plausible (never dereferenced) pyramid
        pyr.hwc[i], pyr.C[i], pyr.H[i], pyr.W[i] = 256, 16, 8, 8
    gw = _lib.MlpWeights()
    gp = (C.c_void_p * 5)()
    rc = lib.srf_render_rays_backward(C.byref(cfg), C.byref(pyr), None, None, 4, None, C.byref(out), C.byref(out), None, 0,
                                      C.byref(gw), C.byref(gw), gp, None, 0, None)
    assert rc == 1 and b"float32" in lib.srf_last_error()
    cfg.precision = 0
    assert lib.srf_render_backward_workspace_bytes(C.byref(cfg), 1200) > 100 << 20
    cfg.flags = _lib.FLAG_SAVE_ACTIVATIONS
    plain = lib.srf_render_workspace_bytes(C.byref(cfg), 1200)
    cfg.flags = 0
    assert plain - lib.srf_render_workspace_bytes(C.byref(cfg), 1200) > 1200 * 64 * 24000      # 24.4 KB per sample point
