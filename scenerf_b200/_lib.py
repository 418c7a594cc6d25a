"""ctypes binding of libscenerf_b200.so (C ABI: include/scenerf_b200.h).  No torch types cross this boundary --
only raw pointers, sizes and POD structs.  The library is built in-tree by scenerf_b200/build.py; if it is missing
and nvcc is unavailable the import of the renderer fails loudly (there is no CPU fallback)."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
# SCENERF_B200_LIB: load another build of the library (kernel experiments: `python -m scenerf_b200.build --variant NAME -DFLAG`)
LIB_PATH = os.environ.get("SCENERF_B200_LIB") or os.path.join(HERE, "libscenerf_b200.so")
_DEFAULT_LIB = os.path.join(HERE, "libscenerf_b200.so")

ABI_VERSION = 2
NUM_SCALES = 5
NUM_BLOCKS = 3

PREC_FP32 = 0
PREC_FP16_TC = 1
PREC_FP32_TC = 2
FLAG_SKIP_ZERO_CHUNKS = 1
FLAG_HIDDEN_FP16 = 2
FLAG_SAVE_ACTIVATIONS = 4
FLAG_TF32_MATMUL = 8
PYR_FP32 = 0
PYR_FP16 = 1

c_float_p = C.POINTER(C.c_float)
c_int32_p = C.POINTER(C.c_int32)


class MlpWeights(C.Structure):
    _fields_ = [("d_out", C.c_int), ("d_latent", C.c_int),
                ("lin_in_w", C.c_void_p), ("lin_in_b", C.c_void_p),
                ("lin_z_w", C.c_void_p * NUM_BLOCKS), ("lin_z_b", C.c_void_p * NUM_BLOCKS),
                ("fc0_w", C.c_void_p * NUM_BLOCKS), ("fc0_b", C.c_void_p * NUM_BLOCKS),
                ("fc1_w", C.c_void_p * NUM_BLOCKS), ("fc1_b", C.c_void_p * NUM_BLOCKS),
                ("lin_out_w", C.c_void_p), ("lin_out_b", C.c_void_p),
                ("tc_packed", C.c_void_p), ("tc_split_packed", C.c_void_p)]


class Pyramid(C.Structure):
    _fields_ = [("hwc", C.c_void_p * NUM_SCALES), ("C", C.c_int * NUM_SCALES), ("H", C.c_int * NUM_SCALES),
                ("W", C.c_int * NUM_SCALES), ("format", C.c_int), ("latent_table", C.c_void_p),
                ("latent_table_gauss", C.c_void_p), ("latent_table_format", C.c_int)]


class Config(C.Structure):
    _fields_ = [("dataset", C.c_int), ("n_pts_uni", C.c_int), ("n_gaussians", C.c_int),
                ("n_pts_per_gaussian", C.c_int), ("max_sample_depth", C.c_float), ("base_std", C.c_float),
                ("som_sigma", C.c_float), ("sphere_W", C.c_int), ("sphere_H", C.c_int), ("d_latent", C.c_int),
                ("v_angle_min", C.c_float), ("v_angle_max", C.c_float), ("h_angle_min", C.c_float),
                ("h_angle_max", C.c_float), ("K", C.c_float * 9), ("inv_K", C.c_float * 9), ("T", C.c_float * 16),
                ("precision", C.c_int), ("seed", C.c_uint64), ("flags", C.c_int), ("ray_offset", C.c_int)]


OUTPUT_FIELDS = ("depth", "color", "gaussian_means", "gaussian_stds", "weights_at_depth", "closest_pts_to_depths",
                 "loss_kl", "alphas", "som_vars", "densities", "weights", "depth_volumes", "som_means",
                 "dbg_sphere_main", "dbg_sphere_gauss")


class Outputs(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in OUTPUT_FIELDS]


# every symbol include/scenerf_b200.h declares: name -> (restype, argtypes)
SYMBOLS = {
    "srf_abi_version": (C.c_int, []),
    "srf_last_error": (C.c_char_p, []),
    "srf_last_launch_count": (C.c_int, []),
    "srf_sizeof": (C.c_size_t, [C.c_int]),
    "srf_debug_watchdog_flag": (C.c_int, []),
    "srf_set_profiling": (None, [C.c_int]),
    "srf_last_mlp_ms": (C.c_int, [C.POINTER(C.c_float), C.POINTER(C.c_float)]),
    "srf_pyramid_bytes": (C.c_size_t, [C.POINTER(C.c_int)] * 3 + [C.c_int]),
    "srf_pack_pyramid": (C.c_int, [C.POINTER(C.c_void_p), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                   C.c_int, C.c_void_p, C.c_size_t, C.POINTER(Pyramid), C.c_void_p]),
    "srf_tc_weights_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "srf_pack_weights_tc": (C.c_int, [C.POINTER(MlpWeights), C.c_void_p, C.c_size_t, C.c_void_p]),
    "srf_tc_split_weights_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "srf_pack_weights_tc_split": (C.c_int, [C.POINTER(MlpWeights), C.c_void_p, C.c_size_t, C.c_void_p]),
    "srf_latent_table_bytes": (C.c_size_t, [C.POINTER(Config), C.c_int]),
    "srf_latent_table_workspace_bytes": (C.c_size_t, [C.POINTER(Pyramid)]),
    "srf_build_latent_table": (C.c_int, [C.POINTER(Config), C.POINTER(Pyramid), C.POINTER(MlpWeights), C.c_int, C.c_void_p,
                                         C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]),
    "srf_render_workspace_bytes": (C.c_size_t, [C.POINTER(Config), C.c_int]),
    "srf_render_rays": (C.c_int, [C.POINTER(Config), C.POINTER(Pyramid), C.POINTER(MlpWeights), C.POINTER(MlpWeights),
                                  C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(Outputs), C.c_void_p,
                                  C.c_size_t, C.c_void_p]),
    "srf_render_host_workspace_bytes": (C.c_size_t, [C.POINTER(Config), C.c_int]),
    "srf_render_rays_host": (C.c_int, [C.POINTER(Config), C.POINTER(Pyramid), C.POINTER(MlpWeights),
                                       C.POINTER(MlpWeights), C.c_void_p, C.c_int, C.POINTER(Outputs), C.c_void_p,
                                       C.c_size_t, C.c_void_p]),
    "srf_predict_workspace_bytes": (C.c_size_t, [C.POINTER(Config), C.c_int]),
    "srf_predict": (C.c_int, [C.POINTER(Config), C.POINTER(Pyramid), C.POINTER(MlpWeights), C.c_void_p, C.c_void_p,
                              C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                              C.c_size_t, C.c_void_p]),
    "srf_render_backward_workspace_bytes": (C.c_size_t, [C.POINTER(Config), C.c_int]),
    "srf_render_rays_backward": (C.c_int, [C.POINTER(Config), C.POINTER(Pyramid), C.POINTER(MlpWeights), C.POINTER(MlpWeights),
                                           C.c_int, C.c_void_p, C.POINTER(Outputs), C.POINTER(Outputs), C.c_void_p, C.c_size_t,
                                           C.POINTER(MlpWeights), C.POINTER(MlpWeights), C.POINTER(C.c_void_p), C.c_void_p,
                                           C.c_size_t, C.c_void_p]),
    "srf_tsdf_reset": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p]),
    "srf_tsdf_integrate": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_float), C.c_double,
                                     C.POINTER(C.c_double), C.POINTER(C.c_float), C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                     C.c_int, C.c_double, C.c_float, C.c_void_p]),
    "srf_tsdf_merge": (C.c_int, [C.c_void_p] * 6 + [C.POINTER(C.c_int), C.c_void_p]),
    "srf_tsdf_mesh_workspace_bytes": (C.c_size_t, [C.POINTER(C.c_int)]),
    "srf_tsdf_mesh_count_host": (C.c_int, [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_void_p, C.c_size_t,
                                           C.POINTER(C.c_longlong), C.POINTER(C.c_longlong), C.c_void_p]),
    "srf_tsdf_mesh_emit": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_float), C.c_double,
                                     C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "srf_eval_hist_len": (C.c_size_t, [C.POINTER(C.c_int), C.c_int, C.c_int]),
    "srf_eval_confusion": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int,
                                     C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "srf_eval_sc_label": (C.c_int, [C.c_void_p, C.POINTER(C.c_int), C.c_double, C.c_void_p, C.c_void_p]),
    "srf_resize_bilinear": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "srf_depth_errors_workspace_bytes": (C.c_size_t, []),
    "srf_depth_errors": (C.c_int, [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p,
                                   C.c_void_p]),
    "srf_upsample_render":(C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_int, C.c_void_p]),
    "srf_psnr_ssim_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "srf_psnr_ssim": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p,
                                C.c_void_p]),
    "srf_lpips_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "srf_lpips_vgg": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                C.POINTER(C.c_void_p), C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_void_p, C.c_size_t, C.c_void_p,
                                C.c_void_p]),
    "srf_sphere_feature_dims": (None, [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "srf_sphere_feature": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                     C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p]),
    "srf_upsample_concat_hwc": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.c_void_p, C.c_int, C.c_void_p]),
    "srf_conv3x3_hwc": (C.c_int, [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p]),
    "srf_debug_gemm": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                 C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]),
    "srf_debug_tc_layer": (C.c_int, [C.POINTER(Config), C.POINTER(Pyramid), C.POINTER(MlpWeights), C.c_void_p,
                                     C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t,
                                     C.c_void_p]),
}

_lib = None


def load(build_if_missing: bool = True):
    """Loads (building first if needed) the shared library and declares all prototypes."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if not build_if_missing:
            raise RuntimeError("libscenerf_b200.so is missing: run `python -m scenerf_b200.build`")
        from . import build as _build
        _build.build()
    elif build_if_missing and LIB_PATH == _DEFAULT_LIB:
        # an edited csrc/*.cu must never run as the old binary: rebuild when a source is newer than the library
        # (skipped silently where nvcc does not exist, e.g. a deployment box that only ships the .so)
        from . import build as _build
        if _build._stale() and _build.have_nvcc():
            _build.build()
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.srf_abi_version() != ABI_VERSION:
        raise RuntimeError("libscenerf_b200.so ABI version %d != %d (stale build? run python -m scenerf_b200.build --force)"
                           % (lib.srf_abi_version(), ABI_VERSION))
    for which, st in enumerate((Config, Pyramid, MlpWeights, Outputs)):
        if lib.srf_sizeof(which) != C.sizeof(st):
            raise RuntimeError("struct %s: binding %d bytes, library %d" % (st.__name__, C.sizeof(st), lib.srf_sizeof(which)))
    _lib = lib
    return lib


class SrfError(RuntimeError):
    pass


def check(rc: int):
    if rc != 0:
        msg = load().srf_last_error().decode("utf-8", "replace")
        if rc == 1:
            raise ValueError("scenerf_b200: " + msg)
        raise SrfError("scenerf_b200 (code %d): %s" % (rc, msg))
