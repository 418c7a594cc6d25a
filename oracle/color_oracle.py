"""Restatement of the reference's novel-view colour evaluation (scripts/evaluation/eval_color.py, eval_color_bf.py) for the
tests of csrc/color_metrics.cu and scenerf_b200.evaluation.ColorErrorBuckets (DESIGN.md 6.8).

The reference scores with scikit-image 0.18.1 (peak_signal_noise_ratio, structural_similarity) and lpips 0.1
(LPIPS(net="vgg")), pinned in its requirements.txt.  Neither package is a dependency here, so this file restates their
documented algorithms; it does not call them:
  * PSNR: 10*log10(data_range**2 / mse), mse = mean((a - b)**2, dtype=float64) with the difference and square in the
    inputs' float32 (skimage's _as_floats keeps float32).
  * SSIM: per channel in float64, scipy.ndimage.uniform_filter(size=7) (the filter skimage 0.18.1 calls, mode 'reflect')
    of x, y, x*x, y*y, x*y, sample covariance (49/48), C1 = (0.01)**2, C2 = (0.03)**2, mean of S[3:-3, 3:-3], then the mean
    over channels; a side below 7 raises ValueError.
  * LPIPS-VGG (version "0.1"): scaling layer, torchvision VGG16 features[0:30] taps after ReLU 3/8/15/22/29, unit
    normalisation over channels (eps 1e-10), squared difference, 1x1 lin (no bias), spatial mean, sum over the 5 taps.
    Computed in float64; tf32=True rounds every convolution operand to the nearest tf32 value first, which is what the
    GPU path does and explains its difference from the float64 value.
  * print_metrics of both scripts (KITTI integer keys printed "{:08d}", BundleFusion string keys printed as they are)."""
from __future__ import annotations

import math

import numpy as np
import scipy.ndimage
import torch

TAPS = (3, 8, 15, 22, 29)
TAP_CHANNELS = (64, 128, 256, 512, 512)
SHIFT = (-.030, -.088, -.188)
SCALE = (.458, .448, .450)


def psnr(image_true, image_test, data_range=1):
    a, b = np.asarray(image_true), np.asarray(image_test)
    err = np.mean((a - b) ** 2, dtype=np.float64)
    with np.errstate(divide="ignore"):
        return 10 * np.log10((data_range ** 2) / err)


def _ssim_channel(X, Y, data_range, win_size=7, K1=0.01, K2=0.03):
    if np.any((np.asarray(X.shape) - win_size) < 0):
        raise ValueError("win_size exceeds image extent.  If the input is a multichannel (color) image, set multichannel=True.")
    X, Y = X.astype(np.float64), Y.astype(np.float64)
    ndim = X.ndim
    NP = win_size ** ndim
    cov_norm = NP / (NP - 1)
    f = lambda z: scipy.ndimage.uniform_filter(z, size=win_size)
    ux, uy = f(X), f(Y)
    uxx, uyy, uxy = f(X * X), f(Y * Y), f(X * Y)
    vx = cov_norm * (uxx - ux * ux)
    vy = cov_norm * (uyy - uy * uy)
    vxy = cov_norm * (uxy - ux * uy)
    R = data_range
    C1 = (K1 * R) ** 2
    C2 = (K2 * R) ** 2
    A1, A2, B1, B2 = (2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2)
    S = (A1 * A2) / (B1 * B2)
    pad = (win_size - 1) // 2
    return S[pad:-pad, pad:-pad].mean()


def ssim(X, Y, data_range=1):
    """structural_similarity(X, Y, multichannel=True, data_range=data_range) of (H,W,C) images."""
    X, Y = np.asarray(X), np.asarray(Y)
    if X.shape != Y.shape:
        raise ValueError("Input images must have the same dimensions.")
    m = np.empty(X.shape[-1])
    for ch in range(X.shape[-1]):
        m[ch] = _ssim_channel(X[..., ch], Y[..., ch], data_range)
    return m.mean()


# --- LPIPS-VGG ---------------------------------------------------------------------------------------------------
def _r32(t: torch.Tensor) -> torch.Tensor:
    """Nearest tf32 value (ties away from zero) of a float64 tensor, through float32."""
    return ((t.float().contiguous().view(torch.int32) + 0x1000) & -8192).view(torch.float32).double()


class LPIPSOracle:
    """lpips.LPIPS(net="vgg") of a state dict in float64 (scenerf_b200.perceptual.parse_state_dict reads the keys)."""

    def __init__(self, state_dict, device="cpu"):
        import torchvision
        from scenerf_b200.perceptual import VGG_CONVS, parse_state_dict
        convs, lins, shift, scale = parse_state_dict(state_dict)
        self.device = torch.device(device)
        self.features = torchvision.models.vgg16(weights=None).features[:30].double().eval().to(self.device)
        with torch.no_grad():
            for idx, (w, b) in zip(VGG_CONVS, convs):
                self.features[idx].weight.copy_(w.double())
                self.features[idx].bias.copy_(b.double())
        self.lins = [l.double().reshape(1, -1, 1, 1).to(self.device) for l in lins]
        self.shift = shift.double().reshape(1, 3, 1, 1).to(self.device)
        self.scale = scale.double().reshape(1, 3, 1, 1).to(self.device)

    def _taps(self, x, tf32):
        out = []
        for i, m in enumerate(self.features):
            if tf32 and isinstance(m, torch.nn.Conv2d):
                x = torch.nn.functional.conv2d(_r32(x), _r32(m.weight), m.bias, padding=1)
            else:
                x = m(x)
            if i in TAPS:
                out.append(x)
        return out

    @torch.no_grad()
    def __call__(self, img0, img1, tf32=False) -> float:
        """img0, img1: (H,W,3) arrays in [0,1] (the compute_lpips inputs before its (x-0.5)*2)."""
        t = lambda a: torch.as_tensor(np.asarray(a, dtype=np.float64)).to(self.device).permute(2, 0, 1)[None]
        x0 = ((t(img0) - 0.5) * 2 - self.shift) / self.scale
        x1 = ((t(img1) - 0.5) * 2 - self.shift) / self.scale
        v = 0.0
        for f0, f1, lin in zip(self._taps(x0, tf32), self._taps(x1, tf32), self.lins):
            n0 = f0 / (f0.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            n1 = f1 / (f1.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            v += float(((n0 - n1) ** 2 * lin).sum(1).mean())
        return v


def random_lpips_state_dict(seed, dropout_index=True, with_scaling=True):
    """A state dict in lpips.LPIPS(net="vgg")'s key layout with seeded random weights: Kaiming-initialised VGG16 (torchvision's
    own init) with N(0, 0.05) biases, non-negative lins (lpips clamps its lins to >= 0 in training)."""
    import torchvision
    from scenerf_b200.perceptual import TAP_CHANNELS as CH, VGG_CONVS, _slice_of
    torch.manual_seed(seed)
    feat = torchvision.models.vgg16(weights=None).features
    sd = {}
    for idx in VGG_CONVS:
        torch.nn.init.normal_(feat[idx].bias, 0, 0.05)
        sd["net.slice%d.%d.weight" % (_slice_of(idx), idx)] = feat[idx].weight.detach().clone()
        sd["net.slice%d.%d.bias" % (_slice_of(idx), idx)] = feat[idx].bias.detach().clone()
    for k, c in enumerate(CH):
        sd["lin%d.model.%d.weight" % (k, 1 if dropout_index else 0)] = (torch.rand(c) / c * 4).reshape(1, c, 1, 1)
    if with_scaling:
        sd["scaling_layer.shift"] = torch.tensor(SHIFT).reshape(1, 3, 1, 1)
        sd["scaling_layer.scale"] = torch.tensor(SCALE).reshape(1, 3, 1, 1)
    return sd


# --- buckets and print_metrics -------------------------------------------------------------------------------------
def bucket_key(dataset, source_distance_str):
    """eval_color.py:80,103 (KITTI: ceil of the file name's distance) / eval_color_bf.py:80,103 (the string itself)."""
    return math.ceil(float(source_distance_str)) if dataset == "kitti" else source_distance_str


def print_metrics(dataset, psnr_accum, ssim_accum, lpips_accum, cnt_accum):
    """eval_color.py:33-60 / eval_color_bf.py:33-60, the printed lines joined."""
    lines = ["|distance |psnr |ssim   |lpips     |n_frames|"]
    total_psnr = 0
    total_ssim = 0
    total_lpips = 0
    total_frame = 0
    key = "|{:08d}|" if dataset == "kitti" else "|{}|"
    for distance in sorted(psnr_accum):
        total_psnr += psnr_accum[distance]
        total_ssim += ssim_accum[distance]
        total_lpips += lpips_accum[distance]
        total_frame += cnt_accum[distance]
        lines.append((key + "{:02.6f}|{:.6f}|{:.6f}|{:.6f}|").format(
            distance, psnr_accum[distance] / cnt_accum[distance], ssim_accum[distance] / cnt_accum[distance],
            lpips_accum[distance] / cnt_accum[distance], cnt_accum[distance]))
    lines.append("|{}|{:02.6f}|{:.6f}|{:.6f}|{:.6f}|".format(
        "All     ", total_psnr / total_frame, total_ssim / total_frame, total_lpips / total_frame, total_frame))
    return "\n".join(lines) + "\n"
