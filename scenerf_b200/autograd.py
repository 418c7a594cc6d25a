"""Training drop-in for the ray-render path: `render_rays_batch` as a differentiable function of the two ResnetFC
parameter sets and the five feature maps ("next" row 8f-1 of the hot-path contract).

Reference: torch.autograd through SceneRF.render_rays_batch (/root/reference/scenerf/models/scenerf.py:392-748); the
consumers of its gradients are the losses of scenerf.py:243-320 (`process_single_source`, `step`).  The forward is the
strict float32 CUDA path (`srf_render_rays`), the backward `srf_render_rays_backward` (csrc/backward.cu).  Differences
from autograd, all documented in include/scenerf_b200.h: `som_vars` is returned non-differentiable (its only consumer
logs it detached); feature-map gradients are accumulated with float atomics (like PyTorch's own CUDA grid_sample).
No CPU fallback: without the CUDA library this module raises."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from ._lib import MlpWeights, Outputs, Pyramid
from .renderer import B200Renderer, DICT_KEYS, SCALE_KEYS, _ptr, _stream_ptr

PARAM_KEYS = (["lin_in.weight", "lin_in.bias", "lin_out.weight", "lin_out.bias"]
              + [k % b for b in range(3) for k in ("lin_z.%d.weight", "lin_z.%d.bias", "blocks.%d.fc_0.weight",
                                                   "blocks.%d.fc_0.bias", "blocks.%d.fc_1.weight", "blocks.%d.fc_1.bias")])
NON_DIFFERENTIABLE = ("som_vars",)


def _weights_struct(tensors: Dict[str, torch.Tensor], d_out: int) -> MlpWeights:
    w = MlpWeights()
    w.d_out = d_out
    w.d_latent = int(tensors["lin_z.0.weight"].shape[1])
    w.lin_in_w, w.lin_in_b = tensors["lin_in.weight"].data_ptr(), tensors["lin_in.bias"].data_ptr()
    w.lin_out_w, w.lin_out_b = tensors["lin_out.weight"].data_ptr(), tensors["lin_out.bias"].data_ptr()
    for b in range(3):
        w.lin_z_w[b], w.lin_z_b[b] = tensors["lin_z.%d.weight" % b].data_ptr(), tensors["lin_z.%d.bias" % b].data_ptr()
        w.fc0_w[b], w.fc0_b[b] = tensors["blocks.%d.fc_0.weight" % b].data_ptr(), tensors["blocks.%d.fc_0.bias" % b].data_ptr()
        w.fc1_w[b], w.fc1_b[b] = tensors["blocks.%d.fc_1.weight" % b].data_ptr(), tensors["blocks.%d.fc_1.bias" % b].data_ptr()
    return w


def _check_param(t: torch.Tensor, device):
    if t.device != device or t.dtype != torch.float32 or not t.is_contiguous():
        raise ValueError("parameters / feature maps must be contiguous float32 tensors on %s" % device)


class RenderRaysFunction(torch.autograd.Function):
    """forward(renderer, cam_K, T, pixels, noise_u, noise_n, *maps(5), *main params(22), *gaussian params(22)) ->
    the 12 dict entries in DICT_KEYS order."""

    @staticmethod
    def forward(ctx, r: B200Renderer, cam_K, T, pix, noise_u, noise_n, *tensors):
        lib = r.lib
        maps, pm, pg = tensors[:5], tensors[5:27], tensors[27:49]
        for t in tensors:
            _check_param(t, r.device)
        main = dict(zip(PARAM_KEYS, pm))
        gauss = dict(zip(PARAM_KEYS, pg))
        w_main, w_gauss = _weights_struct(main, 4), _weights_struct(gauss, 2)
        cfg = r._config(cam_K, T)
        # no input needs a gradient (validation under torch.no_grad(), the per-step depth-eval call of scenerf.py:189-200):
        # nothing will read the activations -- do not store 24.4 KB per sample point
        wants_grad = any(ctx.needs_input_grad)
        if r.save_activations and wants_grad:
            cfg.flags |= _lib.FLAG_SAVE_ACTIVATIONS       # the backward reads the pre-activations instead of recomputing them
        if r.tf32_matmul:
            cfg.flags |= _lib.FLAG_SAVE_ACTIVATIONS | _lib.FLAG_TF32_MATMUL
        elif r.fp32tc_matmul:
            cfg.flags |= _lib.FLAG_SAVE_ACTIVATIONS | _lib.FLAG_FP32TC_MATMUL
        pyr = r._pack_pyramid(dict(zip(SCALE_KEYS, maps)))
        if pyr.format != _lib.PYR_FP32:
            raise RuntimeError("training needs a renderer built with precision='fp32'")
        R = int(pix.shape[0])
        G, S = cfg.n_gaussians, cfg.n_pts_uni + cfg.n_gaussians * cfg.n_pts_per_gaussian
        shapes = dict(depth=(R,), color=(R, 3), gaussian_means=(R, G), gaussian_stds=(R, G), weights_at_depth=(R,),
                      closest_pts_to_depths=(R,), loss_kl=(R,), alphas=(R, S), som_vars=(R, G), densities=(R, S),
                      weights=(R, S), depth_volumes=(R, S))
        ret = {k: torch.empty(shapes[k], dtype=torch.float32, device=r.device) for k in DICT_KEYS}
        som_means = torch.empty((R, G), dtype=torch.float32, device=r.device)
        out = Outputs()
        for k in DICT_KEYS:
            setattr(out, k, ret[k].data_ptr())
        out.som_means = som_means.data_ptr()
        if noise_u is None:
            r.seed += 1
            cfg.seed = r.seed
        nbytes = lib.srf_render_workspace_bytes(C.byref(cfg), R)
        ws = torch.empty(int(nbytes), dtype=torch.uint8, device=r.device)       # dedicated: the backward reads it
        if R:
            _lib.check(lib.srf_render_rays(C.byref(cfg), C.byref(pyr), C.byref(w_main), C.byref(w_gauss), _ptr(pix), R,
                                           _ptr(noise_u), _ptr(noise_n), C.byref(out), _ptr(ws), ws.numel(),
                                           _stream_ptr(r.device)))
        r.last_launches = lib.srf_last_launch_count()
        ctx.r, ctx.cfg, ctx.R, ctx.ws, ctx.noise_n, ctx.som_means = r, cfg, R, ws, noise_n, som_means
        ctx.cam_K, ctx.T = cam_K, T
        ctx.save_for_backward(*tensors, *[ret[k] for k in DICT_KEYS])
        outs = tuple(ret[k] for k in DICT_KEYS)
        ctx.mark_non_differentiable(*[ret[k] for k in NON_DIFFERENTIABLE])
        return outs

    @staticmethod
    def backward(ctx, *cots):
        r, lib, R = ctx.r, ctx.r.lib, ctx.R
        saved = ctx.saved_tensors
        tensors, fwd = saved[:49], dict(zip(DICT_KEYS, saved[49:]))
        maps, pm, pg = tensors[:5], tensors[5:27], tensors[27:49]
        w_main, w_gauss = _weights_struct(dict(zip(PARAM_KEYS, pm)), 4), _weights_struct(dict(zip(PARAM_KEYS, pg)), 2)
        # one zero-filled slab for the 44 parameter gradients (one memset instead of 44), views handed to autograd
        sizes = [t.numel() for t in pm] + [t.numel() for t in pg]
        offs = [0]
        for n in sizes:
            offs.append(offs[-1] + (n + 3) // 4 * 4)          # keep every tensor 16-byte aligned (float4 / TMA paths)
        slab = torch.zeros(offs[-1], dtype=torch.float32, device=r.device)
        views = [slab[offs[i]:offs[i] + sizes[i]].view(t.shape) for i, t in enumerate(list(pm) + list(pg))]
        g_main, g_gauss = views[:len(pm)], views[len(pm):]
        g_maps = [torch.zeros_like(t) for t in maps]
        if R:
            gw_main, gw_gauss = _weights_struct(dict(zip(PARAM_KEYS, g_main)), 4), _weights_struct(dict(zip(PARAM_KEYS, g_gauss)), 2)
            pyr = r._pack_pyramid(dict(zip(SCALE_KEYS, maps)))
            f_out, c_out = Outputs(), Outputs()
            keep = []
            for k, c in zip(DICT_KEYS, cots):
                setattr(f_out, k, fwd[k].data_ptr())
                if c is not None and k not in NON_DIFFERENTIABLE:
                    c = c.to(dtype=torch.float32).contiguous()
                    keep.append(c)
                    setattr(c_out, k, c.data_ptr())
            f_out.som_means = ctx.som_means.data_ptr()
            nbytes = lib.srf_render_backward_workspace_bytes(C.byref(ctx.cfg), R)
            bws = torch.empty(int(nbytes), dtype=torch.uint8, device=r.device)
            gp = (C.c_void_p * 5)(*[t.data_ptr() for t in g_maps])
            _lib.check(lib.srf_render_rays_backward(C.byref(ctx.cfg), C.byref(pyr), C.byref(w_main), C.byref(w_gauss), R,
                                                    _ptr(ctx.noise_n), C.byref(f_out), C.byref(c_out), _ptr(ctx.ws),
                                                    ctx.ws.numel(), C.byref(gw_main), C.byref(gw_gauss), gp, _ptr(bws),
                                                    bws.numel(), _stream_ptr(r.device)))
            r.last_backward_launches = lib.srf_last_launch_count()
        # gradients only where autograd asked for them (a frozen encoder gets None for its five maps)
        need = ctx.needs_input_grad[6:]
        grads = [g if need[i] else None for i, g in enumerate(list(g_maps) + list(g_main) + list(g_gauss))]
        return (None, None, None, None, None, None, *grads)


class TrainableRenderer:
    """`render_rays_batch` with the reference's signature whose outputs carry gradients to `mlp`, `mlp_gaussian`
    (any nn.Module / dict with the ResnetFC parameter names) and to the five maps of `x_rgb`."""

    def __init__(self, hp: dict, mlp, mlp_gaussian, device="cuda:0", rng: str = "torch", save_activations: bool = True,
                 matmul: str = "fp32"):
        if matmul not in ("fp32", "tf32", "fp32tc"):
            raise ValueError("matmul must be 'fp32' (strict SIMT), 'tf32' (wgmma tensor cores) or 'fp32tc' (split 3xTF32 wgmma, "
                             "float32-grade accuracy)")
        state = lambda m: dict(m.named_parameters()) if hasattr(m, "named_parameters") else dict(m)
        self.mlp, self.mlp_gaussian = mlp, mlp_gaussian
        self._state = state
        self.renderer = B200Renderer(hp, {k: v.detach() for k, v in state(mlp).items()},
                                     {k: v.detach() for k, v in state(mlp_gaussian).items()}, device=device, precision="fp32",
                                     rng=rng)
        # True: keep the ResnetFC pre-activations of the forward (24.4 KB per sample point) for the backward;
        # False: recompute them chunk by chunk in the backward (less memory, ~25 % more arithmetic)
        self.renderer.save_activations = bool(save_activations)
        # "tf32": the GEMMs of the training forward and of the backward run as wgmma tf32 (float32 storage, 10-bit
        # mantissa operands) -- several times faster, not bit-compatible with the strict mode (DESIGN.md 6.3);
        # "fp32tc": the same GEMMs on tensor cores as split 3xTF32 products, gradients within the strict mode's bounds
        self.renderer.tf32_matmul = matmul == "tf32"
        self.renderer.fp32tc_matmul = matmul == "fp32tc"

    def render_rays_batch(self, cam_K, T_source2infer, x_rgb, depth_window=100, T_cam2velo=None, sampled_pixels=None,
                          ray_batch_size=128, *, noise=None):
        if sampled_pixels is None:
            raise TypeError("sampled_pixels is required (the reference fails on None too: scenerf.py:419)")
        r = self.renderer
        pix = sampled_pixels.detach().to(device=r.device, dtype=torch.float32).contiguous()
        pm, pg = self._state(self.mlp), self._state(self.mlp_gaussian)
        tensors = [x_rgb[k] for k in SCALE_KEYS] + [pm[k] for k in PARAM_KEYS] + [pg[k] for k in PARAM_KEYS]
        R = int(pix.shape[0])
        cfg = r._config(cam_K, T_source2infer)
        chunks = []
        for s in range(0, max(R, 1), int(ray_batch_size)):          # scenerf.py:419-433: python loop over ray chunks
            e = min(R, s + int(ray_batch_size))
            if noise is not None:
                nu, nn_ = (noise[0][s:e].to(r.device, torch.float32).contiguous(),
                           noise[1][s:e].to(r.device, torch.float32).contiguous())
            elif r.rng == "torch":
                nu, nn_ = r._draw_noise_like_reference(e - s, e - s, cfg)
            else:
                nu = nn_ = None
            chunks.append(RenderRaysFunction.apply(r, cam_K, T_source2infer, pix[s:e].contiguous(), nu, nn_, *tensors))
        outs = chunks[0] if len(chunks) == 1 else tuple(torch.cat(c, 0) for c in zip(*chunks))
        return dict(zip(DICT_KEYS, outs))


def patch_for_training(model, rng: str = "torch", matmul: str = "fp32"):
    """Route `model.render_rays_batch` of a reference SceneRF module through the differentiable CUDA path: gradients
    reach model.mlp, model.mlp_gaussian and (through x_rgb) the image encoder.  Returns the TrainableRenderer."""
    base = B200Renderer.from_module(model, precision="fp32", rng=rng)
    t = TrainableRenderer(base.hp, model.mlp, model.mlp_gaussian, device=base.device, rng=rng, matmul=matmul)
    if t.renderer.hp["dataset"] == "kitti":
        def render_rays_batch(cam_K, T_source2infer, x_rgb, depth_window=100, T_cam2velo=None, sampled_pixels=None,
                              ray_batch_size=128):
            return t.render_rays_batch(cam_K, T_source2infer, x_rgb, depth_window, T_cam2velo, sampled_pixels, ray_batch_size)
    else:
        def render_rays_batch(cam_K, T_source2infer, x_rgb, sampled_pixels=None, ray_batch_size=128):
            return t.render_rays_batch(cam_K, T_source2infer, x_rgb, sampled_pixels=sampled_pixels, ray_batch_size=ray_batch_size)
    model.render_rays_batch = render_rays_batch
    model._b200_trainable = t
    return t
