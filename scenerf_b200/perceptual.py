"""LPIPS-VGG on the device (csrc/color_metrics.cu, DESIGN.md 6.8): the perceptual distance of
scripts/evaluation/eval_color.py:22-26 (`lpips.LPIPS(net="vgg")`, lpips 0.1, version "0.1", spatial=False).

The VGG16 convolutions run on the decoder's wgmma tf32 implicit-GEMM kernel (srf_conv3x3_hwc's kernel), with every
operand rounded to the nearest tf32 value -- the regime of the reference's own GPU run (cuDNN's default
allow_tf32=True).  Weights are not shipped: the caller passes `lpips.LPIPS(net="vgg").state_dict()`."""
from __future__ import annotations

import ctypes as C
import re
from typing import Dict, Tuple

import torch

from . import _lib

# torchvision vgg16().features indices of the 13 convolutions, and the lpips slice each one sits in (slice1 = [0,4),
# slice2 = [4,9), slice3 = [9,16), slice4 = [16,23), slice5 = [23,30))
VGG_CONVS = (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28)
_SLICE_STARTS = (0, 4, 9, 16, 23)
TAP_CHANNELS = (64, 128, 256, 512, 512)
DEFAULT_SHIFT = (-.030, -.088, -.188)
DEFAULT_SCALE = (.458, .448, .450)
_CIN0 = 32          # conv1_1's input as stored: RGB + 29 zero channels (one 32-wide k-block of the kernel)


def _slice_of(idx: int) -> int:
    return max(k for k, s in enumerate(_SLICE_STARTS) if idx >= s) + 1


def _round_tf32(t: torch.Tensor) -> torch.Tensor:
    """Nearest tf32 value (ties away from zero), as the kernels round their own outputs."""
    return ((t.contiguous().view(torch.int32) + 0x1000) & -8192).view(torch.float32)


def parse_state_dict(sd: Dict[str, torch.Tensor]):
    """lpips.LPIPS(net="vgg").state_dict() -> (convs [(weight, bias)] x 13, lins [(C,)] x 5, shift (3,), scale (3,)).
    lin keys may carry the dropout index (`lin{k}.model.1.weight`, use_dropout=True, lpips' default) or not
    (`lin{k}.model.0.weight`).  scaling_layer.* is optional (lpips' constants otherwise).  A missing tensor raises KeyError."""
    convs = []
    for idx in VGG_CONVS:
        pre = "net.slice%d.%d." % (_slice_of(idx), idx)
        if pre + "weight" not in sd or pre + "bias" not in sd:
            raise KeyError("LPIPS state dict has no %sweight / %sbias" % (pre, pre))
        convs.append((sd[pre + "weight"], sd[pre + "bias"]))
    lins = []
    for k, c in enumerate(TAP_CHANNELS):
        keys = [key for key in sd if re.fullmatch(r"lin%d\.model\.[01]\.weight" % k, key)]
        if len(keys) != 1:
            raise KeyError("LPIPS state dict needs exactly one lin%d.model.{0,1}.weight, found %s" % (k, keys))
        w = sd[keys[0]]
        if w.numel() != c:
            raise ValueError("%s has %d values, expected %d" % (keys[0], w.numel(), c))
        lins.append(w.reshape(c))
    for i, (w, b) in enumerate(convs):
        cin = 3 if i == 0 else convs[i - 1][0].shape[0]
        if tuple(w.shape[1:]) != (cin, 3, 3) or b.numel() != w.shape[0]:
            raise ValueError("conv %d (features[%d]) has shape %s" % (i, VGG_CONVS[i], tuple(w.shape)))
    shift = sd.get("scaling_layer.shift", torch.tensor(DEFAULT_SHIFT)).reshape(3)
    scale = sd.get("scaling_layer.scale", torch.tensor(DEFAULT_SCALE)).reshape(3)
    return convs, lins, shift, scale


class LPIPSVGG:
    """LPIPSVGG(state_dict, device)(img0, img1) -> device float32 scalar, the reference's lpips_func(img0, img1) for two
    (H,W,3) float32 images in [0,1] (compute_lpips maps them to [-1,1] itself).  Weights are repacked channels-last and
    rounded to tf32 once; a workspace is kept per image shape.  Calls never synchronise."""

    def __init__(self, state_dict: Dict[str, torch.Tensor], device="cuda:0"):
        self.lib = _lib.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("scenerf_b200.perceptual is the device path (no CPU fallback)")
        convs, lins, shift, scale = parse_state_dict(state_dict)
        f32 = lambda t: t.detach().to(device=self.device, dtype=torch.float32)
        self._w9, self._bias = [], []
        for i, (w, b) in enumerate(convs):
            w = f32(w)
            cout, cin = int(w.shape[0]), int(w.shape[1])
            w9 = torch.zeros((9, cout, _CIN0 if i == 0 else cin), dtype=torch.float32, device=self.device)
            w9[:, :, :cin] = w.permute(2, 3, 0, 1).reshape(9, cout, cin)
            self._w9.append(_round_tf32(w9))
            self._bias.append(f32(b).contiguous())
        self._lin = [f32(l).contiguous() for l in lins]
        self._w9_p = (C.c_void_p * 13)(*[t.data_ptr() for t in self._w9])
        self._bias_p = (C.c_void_p * 13)(*[t.data_ptr() for t in self._bias])
        self._lin_p = (C.c_void_p * 5)(*[t.data_ptr() for t in self._lin])
        self._shift = (C.c_float * 3)(*[float(v) for v in shift.detach().cpu().float()])
        self._scale = (C.c_float * 3)(*[float(v) for v in scale.detach().cpu().float()])
        self._ws: Dict[Tuple[int, int], torch.Tensor] = {}
        self.launches = 0

    def workspace(self, h: int, w: int) -> torch.Tensor:
        """The workspace of one image shape (allocated on first use and kept)."""
        key = (int(h), int(w))
        if key not in self._ws:
            n = int(self.lib.srf_lpips_workspace_bytes(*key))
            if n == 0:
                raise ValueError("LPIPS-VGG needs both image sides in [16, 8192], got %dx%d" % key)
            self._ws[key] = torch.empty(n, dtype=torch.uint8, device=self.device)
        return self._ws[key]

    def __call__(self, img0: torch.Tensor, img1: torch.Tensor) -> torch.Tensor:
        a, b = _image(img0, self.device), _image(img1, self.device)
        if a.shape != b.shape:
            raise ValueError("image shapes differ: %s vs %s" % (tuple(a.shape), tuple(b.shape)))
        h, w = int(a.shape[0]), int(a.shape[1])
        ws = self.workspace(h, w)
        out = torch.empty((), dtype=torch.float32, device=self.device)
        st = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        _lib.check(self.lib.srf_lpips_vgg(a.data_ptr(), b.data_ptr(), h, w, self._w9_p, self._bias_p, self._lin_p, self._shift,
                                          self._scale, ws.data_ptr(), ws.numel(), out.data_ptr(), st))
        self.launches = self.lib.srf_last_launch_count()
        return out


def _image(img, device) -> torch.Tensor:
    """An (H,W,3) image as a contiguous float32 tensor on `device`."""
    t = torch.as_tensor(img)
    if t.dim() != 3 or t.shape[2] != 3:
        raise ValueError("expected an (H,W,3) image, got shape %s" % (tuple(t.shape),))
    return t.to(device=device, dtype=torch.float32).contiguous()
