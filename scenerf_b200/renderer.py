"""Host-side mirror of the reference's renderer interface on top of the C ABI.

`B200Renderer.render_rays_batch` has the argument meaning and the 12-key return dict of
`SceneRF.render_rays_batch` (/root/reference/scenerf/models/scenerf.py:392-471; BundleFusion twin
scenerf_bf.py:420-494), `B200Renderer.predict` those of `SceneRF.predict` (scenerf.py:505-547).  `patch(model)`
swaps the two methods of a live LightningModule for these, which is the whole integration (INTEGRATION.md).

PyTorch is plumbing here: device memory, the current stream and (for `rng="torch"`) the reference's own RNG calls.
All arithmetic of the path runs in libscenerf_b200.so; there is no CPU or eager-PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional

import torch

from . import _lib
from ._lib import Config, MlpWeights, Outputs, Pyramid

SCALE_KEYS = ("1_1", "1_2", "1_4", "1_8", "1_16")
DICT_KEYS = ("depth", "color", "gaussian_means", "gaussian_stds", "weights_at_depth", "closest_pts_to_depths",
             "loss_kl", "alphas", "som_vars", "densities", "weights", "depth_volumes")
MINIMAL_KEYS = ("depth", "color")
PRECISIONS = {"fp32": _lib.PREC_FP32, "fp16": _lib.PREC_FP16_TC, "fp32tc": _lib.PREC_FP32_TC}


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class _PackedMlp:
    """Keeps the 22 nn.Linear tensors of a ResnetFC alive (fp32, contiguous, on device) + the tensor-core pack."""

    def __init__(self, state: Dict[str, torch.Tensor], d_out: int, device, want_tc: bool, want_split: bool = False):
        lib = _lib.load()
        g = lambda k: state[k].detach().to(device=device, dtype=torch.float32).contiguous()
        self.tensors = {k: g(k) for k in state}
        w = MlpWeights()
        w.d_out = d_out
        w.d_latent = int(self.tensors["lin_z.0.weight"].shape[1])
        if tuple(self.tensors["lin_in.weight"].shape) != (512, 42) or self.tensors["lin_out.weight"].shape[0] != d_out:
            raise ValueError("unexpected ResnetFC shapes: lin_in %s lin_out %s" % (
                tuple(self.tensors["lin_in.weight"].shape), tuple(self.tensors["lin_out.weight"].shape)))
        w.lin_in_w, w.lin_in_b = self.tensors["lin_in.weight"].data_ptr(), self.tensors["lin_in.bias"].data_ptr()
        w.lin_out_w, w.lin_out_b = self.tensors["lin_out.weight"].data_ptr(), self.tensors["lin_out.bias"].data_ptr()
        for b in range(3):
            w.lin_z_w[b] = self.tensors["lin_z.%d.weight" % b].data_ptr()
            w.lin_z_b[b] = self.tensors["lin_z.%d.bias" % b].data_ptr()
            w.fc0_w[b] = self.tensors["blocks.%d.fc_0.weight" % b].data_ptr()
            w.fc0_b[b] = self.tensors["blocks.%d.fc_0.bias" % b].data_ptr()
            w.fc1_w[b] = self.tensors["blocks.%d.fc_1.weight" % b].data_ptr()
            w.fc1_b[b] = self.tensors["blocks.%d.fc_1.bias" % b].data_ptr()
        self.packed = None
        if want_tc:
            nbytes = lib.srf_tc_weights_bytes(d_out, w.d_latent)
            self.packed = torch.empty(nbytes, dtype=torch.uint8, device=device)
            _lib.check(lib.srf_pack_weights_tc(C.byref(w), _ptr(self.packed), nbytes, _stream_ptr(device)))
            w.tc_packed = self.packed.data_ptr()
        self.packed_split = None
        if want_split:
            nbytes = lib.srf_tc_split_weights_bytes(d_out, w.d_latent)
            self.packed_split = torch.empty(nbytes, dtype=torch.uint8, device=device)
            _lib.check(lib.srf_pack_weights_tc_split(C.byref(w), _ptr(self.packed_split), nbytes, _stream_ptr(device)))
            w.tc_split_packed = self.packed_split.data_ptr()
        self.struct = w


class B200Renderer:
    """Drop-in for the renderer half of SceneRF (scenerf.py:392-748) on one H100.

    hp: dict with the module attributes the path reads -- dataset ("kitti"|"bf"), n_pts_uni, n_gaussians,
        n_pts_per_gaussian, std, max_sample_depth, out_img_W, out_img_H, som_sigma, v_angle_min/max,
        h_angle_min/max (SphericalMapping incl. add_fov).
    mlp_state / mlp_gaussian_state: ResnetFC state dicts (resnetfc.py parameter names).
    precision: "fp32tc" tensor cores at float32-grade accuracy (fp16 hi/lo split operands, fp32 accumulate: the
         precision-matched mode for the reference's fp32 sgemm), "fp16" tensor cores with fp16 operands (fast mode),
         or "fp32" strict SIMT FMA.
    rng: "torch" reproduces the reference's two RNG calls (utils.py:84, 208-211) chunk by chunk so that seeded runs
         see identical noise; "philox" draws in-kernel (no noise tensors, fastest).
    """

    def __init__(self, hp: dict, mlp_state, mlp_gaussian_state, device="cuda:0", precision: str = "fp16",
                 rng: str = "philox", skip_zero_chunks: bool = False, pyramid_fp16: bool = True,
                 hidden_fp16: bool = True, preproject: bool = False):
        if precision not in PRECISIONS:
            raise ValueError("precision must be one of %s" % list(PRECISIONS))
        if rng not in ("torch", "philox"):
            raise ValueError("rng must be 'torch' or 'philox'")
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda" or not torch.cuda.is_available():
            raise RuntimeError("scenerf_b200 needs a CUDA device (no CPU fallback); got %s" % device)
        self.hp = dict(hp)
        self.precision = precision
        self.rng = rng
        self.skip_zero_chunks = skip_zero_chunks
        self.pyramid_fp16 = pyramid_fp16      # fp16 mode: store the packed pyramid as fp16 (half the gather bytes)
        self.hidden_fp16 = hidden_fp16        # fp16 mode: residual hidden state carried between blocks as fp16
        # tensor-core modes: once per image, tabulate lin_z[b](z) of the main network per integer sphere pixel
        # (srf_build_latent_table) and skip the three lin_z GEMM passes at render time -- exact in real arithmetic
        self.preproject = bool(preproject) and precision in ("fp16", "fp32tc")
        self._tab_buf = None
        self.last_pack_launches = 0
        want_tc, want_split = precision == "fp16", precision == "fp32tc"
        self.mlp = _PackedMlp(mlp_state, 4, self.device, want_tc, want_split)
        self.mlp_gaussian = _PackedMlp(mlp_gaussian_state, 2, self.device, want_tc, want_split)
        self._pyr_key = None
        self._pyr_held = None
        self._pyr_buf = None
        self._pyr = None
        self._ws = None
        self.seed = 0x5CE9E2F
        self.last_launches = 0
        self.last_backward_launches = 0
        self.save_activations = False
        self.tf32_matmul = False
        self.fp32tc_matmul = False

    # ------------------------------------------------------------------------------------------------------------
    @classmethod
    def from_module(cls, model, **kw):
        """Build from a live reference LightningModule (scenerf.py:22 / scenerf_bf.py:27)."""
        sm = model.spherical_mapping
        dataset = "bf" if type(model).__module__.endswith("scenerf_bf") else "kitti"
        hp = dict(dataset=dataset, n_pts_uni=model.n_pts_uni, n_gaussians=model.n_gaussians,
                  n_pts_per_gaussian=model.n_pts_per_gaussian, std=model.std,
                  max_sample_depth=model.max_sample_depth, out_img_W=model.out_img_W, out_img_H=model.out_img_H,
                  som_sigma=model.ray_som.som_sigma, v_angle_min=sm.v_angle_min, v_angle_max=sm.v_angle_max,
                  h_angle_min=sm.h_angle_min, h_angle_max=sm.h_angle_max)
        device = kw.pop("device", None) or next(model.mlp.parameters()).device
        return cls(hp, model.mlp.state_dict(), model.mlp_gaussian.state_dict(), device=device, **kw)

    # ------------------------------------------------------------------------------------------------------------
    def _pack_pyramid(self, x_rgb, cfg: Optional[Config] = None):
        if hasattr(x_rgb, "struct") and hasattr(x_rgb, "buf32"):
            return self._adopt_packed(x_rgb, cfg)
        ts = [x_rgb[k] for k in SCALE_KEYS]
        # The cached pack is reused only for the very same tensor OBJECTS, unmodified (same storage, same version
        # counter).  The renderer keeps references to the caller's tensors while the key is cached, so their storage
        # cannot be freed and re-allocated to another image at the same address (the ABA case of a key made of
        # data_ptr alone); writes that bypass the version counter (.data, raw pointers) need invalidate_pyramid().
        key = tuple((id(t), t.data_ptr(), tuple(t.shape), t.dtype, t._version) for t in ts)
        if key == self._pyr_key and all(a is b for a, b in zip(ts, self._pyr_held)):
            return self._pyr
        src = []
        for t in ts:
            if t.dim() != 3:
                raise ValueError("x_rgb maps must be unbatched CHW (scenerf.py:154-156), got %s" % (tuple(t.shape),))
            src.append(t.detach().to(device=self.device, dtype=torch.float32).contiguous())
        Cs = (C.c_int * 5)(*[t.shape[0] for t in src])
        Hs = (C.c_int * 5)(*[t.shape[1] for t in src])
        Ws = (C.c_int * 5)(*[t.shape[2] for t in src])
        fmt = _lib.PYR_FP16 if (self.precision == "fp16" and self.pyramid_fp16) else _lib.PYR_FP32
        nbytes = self.lib.srf_pyramid_bytes(Cs, Hs, Ws, fmt)
        if self._pyr_buf is None or self._pyr_buf.numel() < nbytes:
            self._pyr_buf = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        ptrs = (C.c_void_p * 5)(*[t.data_ptr() for t in src])
        pyr = Pyramid()
        _lib.check(self.lib.srf_pack_pyramid(ptrs, Cs, Hs, Ws, fmt, _ptr(self._pyr_buf), nbytes, C.byref(pyr),
                                             _stream_ptr(self.device)))
        if self.preproject:
            self._build_latent_table(pyr, fmt, src, Cs, Hs, Ws, cfg)
        self._pyr, self._pyr_key = pyr, key
        self._pyr_held = ts          # the caller's own tensors (pins their storage while the key is cached)
        self._pyr_src = src          # fp32 contiguous copies, if any: alive until the async pack has certainly run
        return pyr

    def _adopt_packed(self, packed, cfg):
        """x_rgb is a scenerf_b200.decoder.PackedPyramid: the producer already wrote the channels-last layout (fp32 and,
        optionally, fp16) -- no srf_pack_pyramid pass."""
        fmt = _lib.PYR_FP16 if (self.precision == "fp16" and self.pyramid_fp16 and packed.buf16 is not None) else _lib.PYR_FP32
        key = ("packed", id(packed), packed.version, fmt)
        if key == self._pyr_key and self._pyr_held is packed:
            return self._pyr
        pyr = packed.struct(fmt)
        if self.preproject:
            p32 = packed.struct(_lib.PYR_FP32)
            Cs = (C.c_int * 5)(*[s[0] for s in packed.shapes])
            Hs = (C.c_int * 5)(*[s[1] for s in packed.shapes])
            Ws = (C.c_int * 5)(*[s[2] for s in packed.shapes])
            self._build_latent_table(pyr, _lib.PYR_FP32, None, Cs, Hs, Ws, cfg, pyr32=p32)
        self._pyr, self._pyr_key, self._pyr_held, self._pyr_src = pyr, key, packed, None
        return pyr

    def _build_latent_table(self, pyr, fmt, src, Cs, Hs, Ws, cfg, pyr32=None):
        """srf_build_latent_table for the main network from an fp32 HWC pack of this image (a temporary one when the
        render pack is fp16); the table pointer rides in the srf_pyramid struct."""
        if cfg is None:
            cfg = self._config(torch.eye(3), None)
        dev = self.device
        keep = None
        if pyr32 is None:
            pyr32 = pyr
        if fmt != _lib.PYR_FP32:
            nb = self.lib.srf_pyramid_bytes(Cs, Hs, Ws, _lib.PYR_FP32)
            keep = torch.empty(nb, dtype=torch.uint8, device=dev)
            ptrs = (C.c_void_p * 5)(*[t.data_ptr() for t in src])
            pyr32 = Pyramid()
            _lib.check(self.lib.srf_pack_pyramid(ptrs, Cs, Hs, Ws, _lib.PYR_FP32, _ptr(keep), nb, C.byref(pyr32), _stream_ptr(dev)))
        tfmt = _lib.PYR_FP16 if self.precision == "fp16" else _lib.PYR_FP32
        nbytes = self.lib.srf_latent_table_bytes(C.byref(cfg), tfmt)
        if self._tab_buf is None or self._tab_buf.numel() < 2 * nbytes:
            self._tab_buf = None
            self._tab_buf = torch.empty(2 * nbytes, dtype=torch.uint8, device=dev)      # main network, then mlp_gaussian
        ws = torch.empty(self.lib.srf_latent_table_workspace_bytes(C.byref(pyr32)), dtype=torch.uint8, device=dev)
        self.last_pack_launches = 0
        for i, net in enumerate((self.mlp, self.mlp_gaussian)):
            tab = self._tab_buf[i * nbytes:(i + 1) * nbytes]
            _lib.check(self.lib.srf_build_latent_table(C.byref(cfg), C.byref(pyr32), C.byref(net.struct), tfmt, _ptr(tab),
                                                       nbytes, _ptr(ws), ws.numel(), _stream_ptr(dev)))
            self.last_pack_launches += self.lib.srf_last_launch_count()
        torch.cuda.current_stream(dev).synchronize()        # the temporaries (fp32 pack, GEMM workspace) die here
        pyr.latent_table = self._tab_buf.data_ptr()
        pyr.latent_table_gauss = self._tab_buf.data_ptr() + nbytes
        pyr.latent_table_format = tfmt

    def invalidate_pyramid(self):
        """Forget the cached feature-pyramid pack (call after writing into x_rgb through .data / raw pointers)."""
        self._pyr_key = None
        self._pyr_held = None
        self._pyr_src = None

    def _config(self, cam_K: torch.Tensor, T: Optional[torch.Tensor]) -> Config:
        hp = self.hp
        cfg = Config()
        cfg.dataset = 0 if hp["dataset"] == "kitti" else 1
        n_uni = int(hp["n_pts_uni"])
        if n_uni <= 0:
            # scenerf_bf.py:623-626,650-661: with n_pts_uni <= 0 the reference renders the gaussian samples only (a
            # stand-in n_pts_uni=2 merely provides the view direction).  That sample set is not built here; refuse
            # loudly (the KITTI class cannot run with it either: torch.linspace(steps=0) -> empty cat at utils.py:86)
            raise ValueError("n_pts_uni=%d: the gaussian-only sampling branch of scenerf_bf.py:650-661 is not supported"
                             % n_uni)
        cfg.n_pts_uni = n_uni
        cfg.n_gaussians = int(hp["n_gaussians"])
        cfg.n_pts_per_gaussian = int(hp["n_pts_per_gaussian"])
        cfg.max_sample_depth = float(hp["max_sample_depth"])
        cfg.base_std = float(hp["std"])
        cfg.som_sigma = float(hp["som_sigma"])
        cfg.sphere_W, cfg.sphere_H = int(hp["out_img_W"]), int(hp["out_img_H"])
        cfg.d_latent = int(self.mlp.struct.d_latent)
        cfg.v_angle_min, cfg.v_angle_max = float(hp["v_angle_min"]), float(hp["v_angle_max"])
        cfg.h_angle_min, cfg.h_angle_max = float(hp["h_angle_min"]), float(hp["h_angle_max"])
        K = cam_K.detach().to(torch.float32)
        inv_K = torch.inverse(K)                         # same op as scenerf.py:401 -> bit-equal inverse
        cfg.K = (C.c_float * 9)(*K.reshape(-1).tolist())
        cfg.inv_K = (C.c_float * 9)(*inv_K.reshape(-1).tolist())
        if T is None:
            T = torch.eye(4)
        cfg.T = (C.c_float * 16)(*T.detach().to(torch.float32).reshape(-1).tolist())
        cfg.precision = PRECISIONS[self.precision]
        cfg.seed = self.seed
        cfg.flags = (_lib.FLAG_SKIP_ZERO_CHUNKS if self.skip_zero_chunks else 0) | \
                    (_lib.FLAG_HIDDEN_FP16 if (self.hidden_fp16 and self.precision == "fp16") else 0)
        return cfg

    def _workspace(self, nbytes: int) -> torch.Tensor:
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = torch.empty(int(nbytes), dtype=torch.uint8, device=self.device)
        return self._ws

    def _draw_noise_like_reference(self, R: int, ray_batch_size: int, cfg: Config):
        """The reference draws, per ray chunk, torch.rand_like on an expanded (R_c,U,1) device tensor (utils.py:78-84)
        and then torch.normal on the CPU (utils.py:208-211).  Same calls, same order -> same streams."""
        U, GP = cfg.n_pts_uni, cfg.n_gaussians * cfg.n_pts_per_gaussian
        us, ns = [], []
        for s in range(0, R, ray_batch_size):
            rc = min(ray_batch_size, R - s)
            lin = torch.linspace(0.2, cfg.max_sample_depth, steps=U, device=self.device).reshape(1, U, 1).expand(rc, -1, -1)
            us.append(torch.rand_like(lin).reshape(rc, U))
            ns.append(torch.normal(mean=torch.zeros(rc, GP), std=torch.ones(rc, GP)).to(self.device))
        return torch.cat(us, 0).contiguous(), torch.cat(ns, 0).contiguous()

    # ------------------------------------------------------------------------------------------------------------
    def render_rays_batch(self, cam_K, T_source2infer, x_rgb, depth_window=100, T_cam2velo=None,
                          sampled_pixels=None, ray_batch_size=128, *, noise=None, outputs="all", debug=False,
                          ray_offset=0, seed=None):
        """scenerf.py:392-471.  `depth_window` and `T_cam2velo` are accepted and unused, exactly like the reference.
        noise: optional (noise_u (R,U), noise_n (R,G*P)) tensors overriding the RNG (parity tests).
        outputs: "all" -> the reference's 12-key dict; "minimal" -> depth and color only (what inference reads).
        ray_offset / seed (rng="philox" only): the rays are rays [ray_offset, ray_offset+R) of a larger frame rendered
        with Philox seed `seed` -- a frame split over several calls or GPUs draws the noise of the single call."""
        if sampled_pixels is None:
            raise TypeError("sampled_pixels is required (the reference fails on None too: scenerf.py:419)")
        pix = sampled_pixels.detach().to(device=self.device, dtype=torch.float32).contiguous()
        if pix.dim() != 2 or pix.shape[1] != 2:
            raise ValueError("sampled_pixels must be (R,2), got %s" % (tuple(pix.shape),))
        R = int(pix.shape[0])
        cfg = self._config(cam_K, T_source2infer)
        pyr = self._pack_pyramid(x_rgb, cfg)
        G, S = cfg.n_gaussians, cfg.n_pts_uni + cfg.n_gaussians * cfg.n_pts_per_gaussian
        keys = DICT_KEYS if outputs == "all" else MINIMAL_KEYS
        shapes = dict(depth=(R,), color=(R, 3), gaussian_means=(R, G), gaussian_stds=(R, G), weights_at_depth=(R,),
                      closest_pts_to_depths=(R,), loss_kl=(R,), alphas=(R, S), som_vars=(R, G), densities=(R, S),
                      weights=(R, S), depth_volumes=(R, S))
        ret = {k: torch.empty(shapes[k], dtype=torch.float32, device=self.device) for k in keys}
        out = Outputs()
        for k in keys:
            setattr(out, k, ret[k].data_ptr())
        if debug:
            ret["som_means"] = torch.empty((R, G), dtype=torch.float32, device=self.device)
            ret["dbg_sphere_main"] = torch.empty((R * S, 2), dtype=torch.int32, device=self.device)
            ret["dbg_sphere_gauss"] = torch.empty((R * G, 2), dtype=torch.int32, device=self.device)
            for k in ("som_means", "dbg_sphere_main", "dbg_sphere_gauss"):
                setattr(out, k, ret[k].data_ptr())
        if R == 0:
            return ret
        nu = nn_ = None
        if noise is not None:
            nu = noise[0].detach().to(device=self.device, dtype=torch.float32).contiguous()
            nn_ = noise[1].detach().to(device=self.device, dtype=torch.float32).contiguous()
            if tuple(nu.shape) != (R, cfg.n_pts_uni) or tuple(nn_.shape) != (R, G * cfg.n_pts_per_gaussian):
                raise ValueError("noise shapes %s %s" % (tuple(nu.shape), tuple(nn_.shape)))
        elif self.rng == "torch":
            nu, nn_ = self._draw_noise_like_reference(R, int(ray_batch_size), cfg)
        elif seed is not None:
            cfg.seed = int(seed)
        else:
            self.seed += 1
            cfg.seed = self.seed
        cfg.ray_offset = int(ray_offset)
        nbytes = self.lib.srf_render_workspace_bytes(C.byref(cfg), R)
        ws = self._workspace(nbytes)
        _lib.check(self.lib.srf_render_rays(C.byref(cfg), C.byref(pyr), C.byref(self.mlp.struct),
                                            C.byref(self.mlp_gaussian.struct), _ptr(pix), R, _ptr(nu), _ptr(nn_),
                                            C.byref(out), _ptr(ws), ws.numel(), _stream_ptr(self.device)))
        self.last_launches = self.lib.srf_last_launch_count()
        return ret

    # ------------------------------------------------------------------------------------------------------------
    def predict(self, mlp, cam_pts, x_rgb, cam_K, T_cam2velo=None, viewdir=None, output_type="density", *,
                debug=False):
        """scenerf.py:505-547.  `mlp` selects the network: the string "mlp"/"mlp_gaussian", or one of this
        renderer's packed networks, or the nn.Module the renderer was built from (matched by d_out)."""
        if viewdir is None:
            raise TypeError("viewdir is required (scenerf.py:508)")
        net = self._select(mlp)
        pts = cam_pts.detach().to(device=self.device, dtype=torch.float32).contiguous()
        saved = tuple(pts.shape)
        if pts.dim() != 3 or saved[2] != 3:
            raise ValueError("cam_pts must be (n_cols, n_per, 3), got %s" % (saved,))
        vd = viewdir.detach().to(device=self.device, dtype=torch.float32).contiguous()
        n_cols, n_per = saved[0], saved[1]
        cfg = self._config(cam_K, None)
        pyr = self._pack_pyramid(x_rgb, cfg)
        n = n_cols * n_per
        d_out = net.struct.d_out
        raw = torch.empty((n, d_out), dtype=torch.float32, device=self.device)
        dens = col = None
        if output_type == "density":
            if d_out != 4:
                raise ValueError("output_type='density' needs the d_out=4 network")
            dens = torch.empty((n_cols, n_per), dtype=torch.float32, device=self.device)
            col = torch.empty((n_cols, n_per, 3), dtype=torch.float32, device=self.device)
        dbg = torch.empty((n, 2), dtype=torch.int32, device=self.device) if debug else None
        if n:
            nbytes = self.lib.srf_predict_workspace_bytes(C.byref(cfg), n)
            ws = self._workspace(nbytes)
            _lib.check(self.lib.srf_predict(C.byref(cfg), C.byref(pyr), C.byref(net.struct), _ptr(pts), _ptr(vd),
                                            n_cols, n_per, _ptr(raw), _ptr(dens), _ptr(col), _ptr(dbg), _ptr(ws),
                                            ws.numel(), _stream_ptr(self.device)))
            self.last_launches = self.lib.srf_last_launch_count()
        if output_type == "density":
            return (dens, col, dbg) if debug else (dens, col)
        res = raw.reshape(n_cols, n_per, d_out)
        return (res, dbg) if debug else res

    def render_rays_batch_host(self, cam_K, T_source2infer, x_rgb, sampled_pixels_host, out_host=None):
        """Same call with HOST buffers (include/scenerf_b200.h: srf_render_rays_host): `sampled_pixels_host` is a CPU
        tensor (pinned for full-speed copies); the rays go host->device, are rendered, and depth (R) + color (R,3)
        come back into CPU tensors, all on the current stream, which is synchronised on return."""
        pix = sampled_pixels_host
        if pix.device.type != "cpu" or pix.dtype != torch.float32 or not pix.is_contiguous():
            raise ValueError("sampled_pixels_host must be a contiguous float32 CPU tensor")
        R = int(pix.shape[0])
        cfg = self._config(cam_K, T_source2infer)
        pyr = self._pack_pyramid(x_rgb, cfg)
        if out_host is None:
            out_host = {"depth": torch.empty((R,), dtype=torch.float32).pin_memory(),
                        "color": torch.empty((R, 3), dtype=torch.float32).pin_memory()}
        out = Outputs()
        out.depth, out.color = out_host["depth"].data_ptr(), out_host["color"].data_ptr()
        self.seed += 1
        cfg.seed = self.seed
        nbytes = self.lib.srf_render_host_workspace_bytes(C.byref(cfg), R)
        ws = self._workspace(nbytes)
        _lib.check(self.lib.srf_render_rays_host(C.byref(cfg), C.byref(pyr), C.byref(self.mlp.struct),
                                                 C.byref(self.mlp_gaussian.struct), C.c_void_p(pix.data_ptr()), R,
                                                 C.byref(out), _ptr(ws), ws.numel(), _stream_ptr(self.device)))
        self.last_launches = self.lib.srf_last_launch_count()
        return out_host

    def set_profiling(self, on: bool):
        self.lib.srf_set_profiling(1 if on else 0)

    def last_mlp_ms(self):
        """(mlp_gaussian pass ms, main mlp pass ms) of the most recent render call, from CUDA events."""
        g, m = C.c_float(-1.0), C.c_float(-1.0)
        _lib.check(self.lib.srf_last_mlp_ms(C.byref(g), C.byref(m)))
        return g.value, m.value

    def debug_tc_layer(self, mlp, cam_pts, x_rgb, cam_K, viewdir, layer: int, out: Optional[torch.Tensor] = None):
        """Diagnostic: raw fp32 accumulator after `layer` of the tensor-core tile program (include/scenerf_b200.h:
        srf_debug_tc_layer), the same pass `predict` runs (latent-table variant included).  Tiles hold 64 points in
        both modes.  fp16: (ceil(n/64)*64, 512), point i at row i.  fp32tc: (ceil(n/32)*64, 512), point i at row
        64 (i//32) + i%32, in units of the weight scale 2^s.  Rows the kernel does not write keep the contents of
        `out` (a float32 tensor of that shape on the renderer's device; zeros when omitted)."""
        net = self._select(mlp)
        if net.packed is None and net.packed_split is None:
            raise RuntimeError("renderer was not built with precision='fp16' / 'fp32tc'")
        pts = cam_pts.detach().to(device=self.device, dtype=torch.float32).contiguous()
        vd = viewdir.detach().to(device=self.device, dtype=torch.float32).contiguous()
        n_cols, n_per = pts.shape[0], pts.shape[1]
        cfg = self._config(cam_K, None)
        pyr = self._pack_pyramid(x_rgb, cfg)
        n = n_cols * n_per
        rows = (n + 31) // 32 * 64 if self.precision == "fp32tc" else (n + 63) // 64 * 64
        if out is None:
            acc = torch.zeros((rows, 512), dtype=torch.float32, device=self.device)
        else:
            if out.dtype != torch.float32 or tuple(out.shape) != (rows, 512) or out.device != self.device or not out.is_contiguous():
                raise ValueError("out must be a contiguous float32 (%d, 512) tensor on %s" % (rows, self.device))
            acc = out
        ws = self._workspace(self.lib.srf_predict_workspace_bytes(C.byref(cfg), n))
        _lib.check(self.lib.srf_debug_tc_layer(C.byref(cfg), C.byref(pyr), C.byref(net.struct), _ptr(pts), _ptr(vd),
                                               n_cols, n_per, int(layer), _ptr(acc), _ptr(ws), ws.numel(),
                                               _stream_ptr(self.device)))
        return acc

    def _select(self, mlp):
        if mlp in ("mlp", None) or mlp is self.mlp:
            return self.mlp
        if mlp in ("mlp_gaussian",) or mlp is self.mlp_gaussian:
            return self.mlp_gaussian
        d_out = getattr(mlp, "d_out", None)
        if d_out == 4:
            return self.mlp
        if d_out == 2:
            return self.mlp_gaussian
        raise ValueError("cannot map %r to mlp / mlp_gaussian" % (mlp,))


def patch(model, **kw):
    """Replace `model.render_rays_batch` / `model.predict` of a reference SceneRF module by the CUDA path.
    Call again after loading new weights.  Returns the renderer."""
    r = B200Renderer.from_module(model, **kw)
    if r.hp["dataset"] == "kitti":
        def render_rays_batch(cam_K, T_source2infer, x_rgb, depth_window=100, T_cam2velo=None, sampled_pixels=None,
                              ray_batch_size=128):
            return r.render_rays_batch(cam_K, T_source2infer, x_rgb, depth_window, T_cam2velo, sampled_pixels,
                                       ray_batch_size)

        def predict(mlp, cam_pts, x_rgb, cam_K, T_cam2velo, viewdir, output_type="density"):
            return r.predict(mlp, cam_pts, x_rgb, cam_K, T_cam2velo, viewdir, output_type)
    else:
        def render_rays_batch(cam_K, T_source2infer, x_rgb, sampled_pixels=None, ray_batch_size=128):
            return r.render_rays_batch(cam_K, T_source2infer, x_rgb, sampled_pixels=sampled_pixels,
                                       ray_batch_size=ray_batch_size)

        def predict(mlp, cam_pts, x_rgb, cam_K, viewdir, output_type="density"):
            return r.predict(mlp, cam_pts, x_rgb, cam_K, None, viewdir, output_type)
    model.render_rays_batch = render_rays_batch
    model.predict = predict
    model._b200_renderer = r
    return r
