"""Shared test helpers: build a B200Renderer from a synth.SceneConfig and compare dicts against goldens; tf32 rounding
and the accumulation bound of the wgmma .tf32 kernels."""
import math

import numpy as np

from cases import params_for, pyramid_for

# Accumulation constant of the wgmma .tf32 kernels (conv_tf32.cu, gemm_tf32.cu).  With operands that are tf32 values the
# products are exact, and an entry's float32 accumulation error stays under
#   tf32_gamma(K) * sum_k |a_k| |b_k|,   tf32_gamma(K) = TF32_ACC_C * ceil(K / 8) * 2^-24,
# one rounding per 8-wide k-step of the tensor core.  The accumulator truncates (the unrounded-operand case of
# tests/test_gpu_conv.py matches a truncating emulation), so a step may lose up to one float32 ulp, 2^-23 of the partial
# sum: c = 2.  Measured by tests/test_gpu_conv.py on an H100 80GB HBM3 (700 W power limit): c = 1.06 where every operand
# is >= 0 (Cin = 512, the partial sums grow to S), at most 0.093 on signed operands.
TF32_ACC_C = 2.0


def tf32_gamma(k):
    return TF32_ACC_C * math.ceil(k / 8) * 2.0 ** -24


def tf32_rn(t):
    """float32 torch tensor -> nearest tf32 value (ties away from zero): the integer trick of decoder.py::_pack and of
    round_tf32 in conv_tf32.cu."""
    import torch
    return ((t.contiguous().view(torch.int32) + 0x1000) & -8192).view(torch.float32)


def hp_from_cfg(cfg):
    v_min, v_max, h_min, h_max = cfg.angles()
    return dict(dataset=cfg.dataset, n_pts_uni=cfg.n_pts_uni, n_gaussians=cfg.n_gaussians,
                n_pts_per_gaussian=cfg.n_pts_per_gaussian, std=cfg.std, max_sample_depth=cfg.max_sample_depth,
                out_img_W=cfg.sphere_W, out_img_H=cfg.sphere_H, som_sigma=cfg.som_sigma, v_angle_min=v_min,
                v_angle_max=v_max, h_angle_min=h_min, h_angle_max=h_max)


def make_renderer(cfg, precision, device="cuda:0", **kw):
    import torch
    from scenerf_b200.renderer import B200Renderer
    pm, pg = params_for(cfg)
    to = lambda d: {k: torch.from_numpy(v) for k, v in d.items()}
    return B200Renderer(hp_from_cfg(cfg), to(pm), to(pg), device=device, precision=precision, **kw)


def torch_pyramid(cfg, seed, device="cuda:0"):
    import torch
    return {k: torch.from_numpy(v).to(device) for k, v in pyramid_for(cfg, seed).items()}


def max_err(a, b):
    return float(np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64)).max()) if np.size(a) else 0.0
