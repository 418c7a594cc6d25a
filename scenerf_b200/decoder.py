"""Producer tail of the feature pyramid on the device: the convolutional part of `DecoderSphere.forward`
(/root/reference/scenerf/models/unet2d_sphere.py:167-206) -- six `get_sphere_feature` resamplings (csrc/sphere_feature.cu) and the
five `UpSampleBN` stacks (:37-57: bilinear align_corners upsample + concat, Conv2d 3x3, three dilated `BasicBlock`s with eval-mode
BatchNorm, LeakyReLU and residual add) as wgmma tf32 implicit GEMMs on channels-last maps (csrc/conv_tf32.cu).

The last convolution of every level writes its [H][W][C] output straight into one contiguous buffer laid out exactly like
`srf_pack_pyramid`'s result (fp32 and, optionally, fp16): `PackedPyramid` is handed to `B200Renderer.render_rays_batch` /
`predict` as `x_rgb` and no CHW -> HWC pass runs.  `.as_x_rgb()` gives the reference's dict of CHW tensors (views) for callers
that still want it.  Inference only (BatchNorm in eval mode, no backward).  The EfficientNet encoder and the 1x1 `conv2` on the
1/32 map (:79-81,176) stay PyTorch's: they are outside the hot path's producer tail (DESIGN.md section 8).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict

import torch

from . import _lib
from .sphere_feature import get_sphere_feature
from .synth import SCALE_KEYS

LEVELS = (16, 8, 4, 2, 1)
BN_EPS = 1e-5
LRELU_SLOPE = 0.01


def _ceil4(n: int) -> int:
    return (n + 3) // 4 * 4


class PackedPyramid:
    """The five maps of x_rgb, channels-last, in the layout of srf_pack_pyramid (scale order 1_1 .. 1_16, 256-byte aligned)."""

    def __init__(self, shapes, device, want_fp16: bool):
        self.shapes = list(shapes)                       # [(C, H, W)] for 1_1, 1_2, 1_4, 1_8, 1_16
        self.device = device
        al = lambda b: (b + 255) // 256 * 256
        self.offs32, self.offs16 = [], []
        o32 = o16 = 0
        for c, h, w in self.shapes:
            self.offs32.append(o32)
            self.offs16.append(o16)
            o32 += al(c * h * w * 4)
            o16 += al(c * h * w * 2)
        self.buf32 = torch.empty(o32, dtype=torch.uint8, device=device)
        self.buf16 = torch.empty(o16, dtype=torch.uint8, device=device) if want_fp16 else None
        self.version = 0

    def view32(self, i):
        c, h, w = self.shapes[i]
        return self.buf32[self.offs32[i]:self.offs32[i] + c * h * w * 4].view(torch.float32).view(h, w, c)

    def view16(self, i):
        c, h, w = self.shapes[i]
        return self.buf16[self.offs16[i]:self.offs16[i] + c * h * w * 2].view(torch.float16).view(h, w, c)

    def as_x_rgb(self) -> Dict[str, torch.Tensor]:
        """The reference's dict "1_1".."1_16" of (C,H,W) tensors (non-contiguous views of the channels-last buffer)."""
        return {k: self.view32(i).permute(2, 0, 1) for i, k in enumerate(SCALE_KEYS)}

    def struct(self, fmt: int) -> _lib.Pyramid:
        p = _lib.Pyramid()
        for i, (c, h, w) in enumerate(self.shapes):
            if fmt == _lib.PYR_FP16:
                if self.buf16 is None:
                    raise RuntimeError("this PackedPyramid was produced without the fp16 copy (SphereDecoderB200(emit_fp16=True))")
                p.hwc[i] = self.buf16.data_ptr() + self.offs16[i]
            else:
                p.hwc[i] = self.buf32.data_ptr() + self.offs32[i]
            p.C[i], p.H[i], p.W[i] = c, h, w
        p.format = fmt
        return p


class SphereDecoderB200:
    """state: DecoderSphere.state_dict() (or the dict of scenerf_b200.synth.make_decoder_params) -- weights are folded
    (conv bias + eval BatchNorm -> per-channel scale/shift) and repacked [tap][Cout][Cin] once."""

    def __init__(self, state: Dict[str, torch.Tensor], out_img_W: int, out_img_H: int, device="cuda:0", emit_fp16: bool = True):
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("scenerf_b200.decoder is the device path (no CPU fallback)")
        self.out_img_W, self.out_img_H = int(out_img_W), int(out_img_H)
        self.emit_fp16 = bool(emit_fp16)
        g = lambda k: state[k].detach().to(device=self.device, dtype=torch.float32)
        self.conv2_w, self.conv2_b = g("conv2.weight").contiguous(), g("conv2.bias").contiguous()
        self.levels = {}
        for s in LEVELS:
            pre = "up%d._net." % s
            convs = [self._pack(g(pre + "0.weight"), g(pre + "0.bias"), None, state, 1, 1.0)]
            for blk, dil in ((1, 1), (2, 2), (3, 3)):
                for cb in (1, 2):
                    name = pre + "%d.conv_block%d" % (blk, cb)
                    convs.append(self._pack(g(name + ".0.weight"), g(name + ".0.bias"), name + ".1", state, dil,
                                            LRELU_SLOPE))      # conv_block2's LeakyReLU comes after the residual add: same slope
            self.levels[s] = convs
        self.launches = 0

    def _pack(self, w, b, bn, state, dil, slope):
        cout, cin = int(w.shape[0]), int(w.shape[1])
        ld = _ceil4(cin)
        w9 = torch.zeros((9, cout, ld), dtype=torch.float32, device=self.device)
        w9[:, :, :cin] = w.permute(2, 3, 0, 1).reshape(9, cout, cin)             # [ky][kx][co][ci] -> tap-major, K contiguous
        # round to the nearest tf32 value once: the tensor core then truncates nothing (csrc/conv_tf32.cu)
        w9 = ((w9.contiguous().view(torch.int32) + 0x1000) & -8192).view(torch.float32)
        if bn is None:
            scale, shift = torch.ones(cout, device=self.device), b.clone()
        else:
            g = lambda k: state[bn + k].detach().to(device=self.device, dtype=torch.float32)
            scale = g(".weight") / torch.sqrt(g(".running_var") + BN_EPS)
            shift = (b - g(".running_mean")) * scale + g(".bias")
        return dict(w9=w9.contiguous(), scale=scale.contiguous(), shift=shift.contiguous(), cin=cin, ld=ld, cout=cout, dil=dil, slope=slope)

    def _conv(self, x, H, W, cv, residual, out32, out16=None, round_out=True):
        st = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        _lib.check(self.lib.srf_conv3x3_hwc(x.data_ptr(), H, W, cv["ld"], cv["w9"].data_ptr(), cv["cout"], cv["dil"],
                                            cv["scale"].data_ptr(), cv["shift"].data_ptr(),
                                            residual.data_ptr() if residual is not None else None, cv["cout"], float(cv["slope"]),
                                            1 if round_out else 0, out32.data_ptr() if out32 is not None else None, cv["cout"],
                                            out16.data_ptr() if out16 is not None else None, cv["cout"], st))
        self.launches += 1

    def _up(self, x_hwc, skip_hwc, s, out32, out16):
        """One UpSampleBN (unet2d_sphere.py:37-57) on channels-last maps; the last conv writes into the packed pyramid."""
        H, W, Cs = skip_hwc.shape
        h, w, Cx = x_hwc.shape
        convs = self.levels[s]
        cat = torch.empty((H, W, convs[0]["ld"]), dtype=torch.float32, device=self.device)
        st = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        _lib.check(self.lib.srf_upsample_concat_hwc(x_hwc.data_ptr(), h, w, Cx, Cx, skip_hwc.data_ptr(), Cs, Cs, H, W, cat.data_ptr(),
                                                    convs[0]["ld"], st))
        self.launches += 1
        co = convs[0]["cout"]
        y = torch.empty((H, W, co), dtype=torch.float32, device=self.device)
        self._conv(cat, H, W, convs[0], None, y)
        for blk in range(3):
            c1, c2 = convs[1 + 2 * blk], convs[2 + 2 * blk]
            t = torch.empty_like(y)
            self._conv(y, H, W, c1, None, t)
            last = blk == 2
            z = out32 if last else torch.empty_like(y)
            self._conv(t, H, W, c2, y, z, out16 if last else None, round_out=not last)   # BN(conv) + residual, then LeakyReLU; the pyramid map itself is not rounded
            y = z
        return y

    @torch.no_grad()
    def forward(self, features, pix, pix_sphere) -> PackedPyramid:
        """features: the encoder's list (indices 0,4,5,6,8,11 are read, unet2d_sphere.py:168-175), maps (1,C,h,w)."""
        f = {1: features[0], 2: features[4], 4: features[5], 8: features[6], 16: features[8], 32: features[11]}
        f = {s: t.detach().to(device=self.device, dtype=torch.float32) for s, t in f.items()}
        if any(t.shape[0] != 1 for t in f.values()):
            raise ValueError("one image per call (the reference renders per image: scenerf.py:154-156)")
        self.launches = 0
        x32 = torch.nn.functional.conv2d(f[32], self.conv2_w, self.conv2_b, stride=1, padding=1)     # 1x1, padding 1 (:79-81)
        sph = {32: get_sphere_feature(x32, pix, pix_sphere, 32, self.out_img_W, self.out_img_H, channels_last=True)[0]}
        for s in LEVELS:
            sph[s] = get_sphere_feature(f[s].contiguous(), pix, pix_sphere, s, self.out_img_W, self.out_img_H, channels_last=True)[0]
        shapes = [(self.levels[s][0]["cout"], sph[s].shape[0], sph[s].shape[1]) for s in (1, 2, 4, 8, 16)]
        pyr = PackedPyramid(shapes, self.device, self.emit_fp16)
        x = sph[32]
        for s in LEVELS:
            i = (1, 2, 4, 8, 16).index(s)
            x = self._up(x, sph[s], s, pyr.view32(i), pyr.view16(i) if self.emit_fp16 else None)
        return pyr

    __call__ = forward
