"""Evaluation metrics on the device (csrc/metrics.cu, DESIGN.md 6.7): the numbers the reference computes on the host
after a reconstruction or a novel-depth render, from the volumes and depths this package already keeps in HBM.

Reference (file:line):
  scenerf/loss/sscMetrics.py:361-529                           SSCMetrics (add_batch / get_stats / reset)
  scenerf/scripts/evaluation/eval_sr.py:11-17,79-87            tsdf2occ (KITTI) and the per-frame scoring
  scenerf/scripts/evaluation/eval_sc_bf.py:117-123,203-210     tsdf2occ (BundleFusion)
  scenerf/scripts/reconstruction/generate_sc_gt_bf.py:280-309  the BundleFusion completion target
  scenerf/loss/depth_metrics.py                                compute_depth_errors
  scenerf/scripts/evaluation/save_depth_metrics.py:98-183      ceil(distance) buckets and print_metrics
Counts are integers from one kernel pass, so every statistic equals the reference's to the last bit.  Nothing here
synchronises the stream except where a host value is returned (get_stats, compute_depth_errors, table, the empty-target
check of score_reconstruction_kitti)."""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import numpy as np
import torch

from . import _lib

EVAL_U8, EVAL_I32, EVAL_I64, EVAL_F32, EVAL_F64 = 0, 1, 2, 3, 4
_PRED_DTYPES = {torch.uint8: EVAL_U8, torch.int32: EVAL_I32, torch.int64: EVAL_I64, torch.float32: EVAL_F32,
                torch.float64: EVAL_F64}
MAX_CLASSES = 64


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _device(device=None):
    return torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())


def _tensor(x, device):
    """numpy array or tensor -> contiguous tensor on `device` (device tensors are used in place)."""
    return torch.as_tensor(x).to(device=device).contiguous()


def _volume(vol, device=None):
    """A TSDFVolume (its device tsdf) or an (X,Y,Z) array / tensor -> float32 contiguous device tensor."""
    t = vol._tsdf if hasattr(vol, "_tsdf") else torch.as_tensor(vol)
    if t.dim() != 3:
        raise ValueError("expected an (X,Y,Z) volume, got shape %s" % (tuple(t.shape),))
    dev = t.device if t.is_cuda else _device(device)
    return t.to(device=dev, dtype=torch.float32).contiguous()


def _dims(shape):
    return (C.c_int * 3)(*[int(s) for s in shape])


def _labels(y_true, device):
    """Target labels as uint8.  Other integer / bool / integral float labels are accepted when they lie in [0, 255]."""
    t = _tensor(y_true, device)
    if t.dtype == torch.uint8:
        return t
    if t.dtype == torch.bool:
        return t.to(torch.uint8)
    tf = t.to(torch.float64)
    if t.numel() and not bool(((tf >= 0) & (tf <= 255) & (tf == torch.floor(tf))).all()):
        raise ValueError("target labels must be integers in [0, 255]")
    return t.to(torch.uint8)


def _mask(m, numel, device):
    """A mask as uint8 0/1.  The reference selects voxels where `(y_true != 255) & mask == 1`: a bool mask counts where it
    is True, an integer mask where its lowest bit is set."""
    t = _tensor(m, device).reshape(-1)
    if t.numel() != numel:
        raise ValueError("mask has %d elements, the volume %d" % (t.numel(), numel))
    if t.dtype == torch.bool:
        return t.to(torch.uint8)
    if t.is_floating_point():
        raise TypeError("masks must be bool or integer arrays (the reference combines them with `&`)")
    return (t & 1).to(torch.uint8)


def _pred(y_pred, device):
    t = _tensor(y_pred, device)
    if t.dtype == torch.bool:
        t = t.to(torch.uint8)
    elif t.dtype in (torch.int8, torch.int16):
        t = t.to(torch.int32)
    elif t.dtype in (torch.float16, torch.bfloat16):
        t = t.to(torch.float32)
    elif t.dtype not in _PRED_DTYPES:
        t = t.to(torch.int64)
    return t


def _confusion(shape, n_classes, device, *, tsdf=None, th=None, axis=0, pred=None, target=None, mask=None, per_z=False,
               occ=None):
    """One srf_eval_confusion pass.  Returns (hist int64 (Zh, 2, C+1, C+2), max_z int32 (1,)) on the device."""
    lib = _lib.load()
    dims = _dims(shape)
    n = int(_lib.load().srf_eval_hist_len(dims, int(n_classes), 1 if per_z else 0))
    if n == 0:
        raise ValueError("n_classes=%d outside [1, %d]" % (n_classes, MAX_CLASSES))
    hist = torch.empty(n, dtype=torch.int64, device=device)
    max_z = torch.empty(1, dtype=torch.int32, device=device)
    p = lambda t: None if t is None else t.data_ptr()
    _lib.check(lib.srf_eval_confusion(p(tsdf), p(pred), _PRED_DTYPES[pred.dtype] if pred is not None else 0, p(target), p(mask),
                                      dims, int(n_classes), int(axis), p(th), 1 if per_z else 0, hist.data_ptr(),
                                      max_z.data_ptr(), p(occ), _stream(device)))
    return hist.reshape(-1, 2, n_classes + 1, n_classes + 2), max_z


def _crop_z(hist, max_z):
    """eval_sr.py:84 occ[:, :, max_z:] = 0 on per-z histograms: every slice from max_z up moves to pred bucket 0."""
    h = hist.clone()
    top = h[max_z:]
    top[..., 0] = top.sum(-1)
    top[..., 1:] = 0
    return h.sum(0)


# --- tsdf2occ -------------------------------------------------------------------------------------------------------
def th_table_kitti(n, th=0.25, max_th=6.0):
    """eval_sr.py:13-15 (there n = 256, the x extent): float64 with the reference's expression and clamps."""
    t = (0.1 + np.arange(n) * 0.2) * th
    t[t < 0.2] = 0.2
    t[t > max_th] = max_th
    return t


def th_table_bf(n, min_th, th=0.25, max_th=0.2, voxel_size=0.04):
    """eval_sc_bf.py:119-121 (there n = 96, the z extent)."""
    t = voxel_size + np.arange(n) * voxel_size * th
    t[t < min_th] = min_th
    t[t > max_th] = max_th
    return t


def _occupancy(vol, table, axis, device=None):
    t = _volume(vol, device)
    th = torch.from_numpy(np.ascontiguousarray(table, dtype=np.float64)).to(t.device)
    occ = torch.empty(t.shape, dtype=torch.uint8, device=t.device)
    _confusion(t.shape, 2, t.device, tsdf=t, th=th, axis=axis, occ=occ)
    return occ


def tsdf2occ_kitti(vol, th=0.25, max_th=6.0, device=None):
    """eval_sr.py:11-17: occupancy (X,Y,Z) uint8 0/1 on the device; the threshold grows along x."""
    t = _volume(vol, device)
    return _occupancy(t, th_table_kitti(t.shape[0], th, max_th), 0)


def tsdf2occ_bf(vol, min_th, th=0.25, max_th=0.2, voxel_size=0.04, device=None):
    """eval_sc_bf.py:117-123: occupancy (X,Y,Z) uint8 0/1 on the device; the threshold grows along z."""
    t = _volume(vol, device)
    return _occupancy(t, th_table_bf(t.shape[2], min_th, th, max_th, voxel_size), 2)


# --- SSCMetrics -----------------------------------------------------------------------------------------------------
class SSCMetrics:
    """loss/sscMetrics.py:361-529 as a device accumulator: add_batch runs one kernel pass (two when both nonempty and
    nonsurface are given) and adds integer histograms on the device; get_stats reads them back.  Inputs are numpy
    arrays or tensors of any shape (the reference's reshape to (shape[0], -1) only orders its loop).  y_true holds
    labels in [0, 255], 255 = not evaluated; labels >= n_classes count as occupied for completion, as in the reference."""

    def __init__(self, n_classes, device=None):
        if not 1 <= int(n_classes) <= MAX_CLASSES:
            raise ValueError("n_classes=%d outside [1, %d]" % (n_classes, MAX_CLASSES))
        self.n_classes = int(n_classes)
        self.device = _device(device)
        self.reset()

    def reset(self):
        shape = (self.n_classes + 1, self.n_classes + 2)
        self._comp = torch.zeros(shape, dtype=torch.int64, device=self.device)   # completion (nonempty & nonsurface)
        self._sem = torch.zeros(shape, dtype=torch.int64, device=self.device)    # semantic (nonempty)

    def _add_hist(self, comp, sem):
        self._comp += comp
        self._sem += sem

    def add_batch(self, y_pred, y_true, nonempty=None, nonsurface=None):
        target = _labels(y_true, self.device).reshape(-1)
        pred = _pred(y_pred, self.device).reshape(-1)
        if pred.numel() != target.numel():
            raise ValueError("y_pred has %d elements, y_true %d" % (pred.numel(), target.numel()))
        n = target.numel()
        shape = (1, 1, n)
        ne = _mask(nonempty, n, self.device) if nonempty is not None else None
        ns = _mask(nonsurface, n, self.device) if nonsurface is not None else None
        comp_mask = ne if ns is None else (ns if ne is None else ne & ns)
        h, _ = _confusion(shape, self.n_classes, self.device, pred=pred, target=target, mask=comp_mask)
        h = h[0]
        comp = h[1] if comp_mask is not None else h[0]
        if ns is None:
            sem = comp
        elif ne is None:
            sem = h[0]
        else:
            sem = _confusion(shape, self.n_classes, self.device, pred=pred, target=target, mask=ne)[0][0][1]
        self._add_hist(comp, sem)

    def counts(self):
        """(completion_tp, completion_fp, completion_fn, tps, fps, fns) as the reference accumulates them: Python ints
        and float64 arrays."""
        C_ = self.n_classes
        comp = self._comp.cpu().numpy()
        sem = self._sem.cpu().numpy()
        pos_t, pos_p = slice(1, C_ + 1), slice(1, C_ + 1)        # label > 0 ; pred bucket 1..C-1 or "other > 0"
        tp = int(comp[pos_t, pos_p].sum())
        fp = int(comp[0, pos_p].sum())
        fn = int(comp[pos_t, 0].sum() + comp[pos_t, C_ + 1].sum())
        d = np.diag(sem[:C_, :C_])
        tps = d.astype(np.float64)
        fps = (sem[:, :C_].sum(0) - d).astype(np.float64)
        fns = (sem[:C_, :].sum(1) - d).astype(np.float64)
        return tp, fp, fn, tps, fps, fns

    def get_stats(self):
        tp, fp, fn, tps, fps, fns = self.counts()
        if tp != 0:
            precision = tp / (tp + fp)
            recall = tp / (tp + fn)
            iou = tp / (tp + fp + fn)
        else:
            precision, recall, iou = 0, 0, 0
        iou_ssc = tps / (tps + fps + fns + 1e-5)
        return {"precision": precision, "recall": recall, "iou": iou, "iou_ssc": iou_ssc, "iou_ssc_mean": np.mean(iou_ssc[1:])}

    def all_reduce(self, rank: int = 0, world: int = 1, group=None):
        """Sum the counts of all ranks (rank order); afterwards every rank holds the total."""
        if world > 1:
            both = dist_sum(torch.stack([self._comp, self._sem]), rank, world, group)
            self._comp, self._sem = both[0].clone(), both[1].clone()
        return self


def score_reconstruction_kitti(vol, target_1_1, fov_mask, metric: SSCMetrics, fov_metric: SSCMetrics, th=0.25, max_th=6.0,
                               return_occ=False):
    """eval_sr.py:79-87 in one kernel pass: occupancy of `vol` (TSDFVolume or (X,Y,Z) tsdf), crop at the top labelled
    z slice, metric.add_batch(occ, target) and fov_metric.add_batch(occ, target, fov_mask).  Raises ValueError when the
    target has no label other than 0 and 255 (the reference's .max() of an empty array).  return_occ: also return the
    cropped occupancy (uint8, on the device)."""
    if metric.n_classes != fov_metric.n_classes:
        raise ValueError("metric and fov_metric have different n_classes")
    t = _volume(vol, metric.device)
    target = _labels(target_1_1, t.device)
    if target.numel() != t.numel():
        raise ValueError("target has %d elements, the volume %d" % (target.numel(), t.numel()))
    fov = _mask(fov_mask, t.numel(), t.device)
    th_t = torch.from_numpy(th_table_kitti(t.shape[0], th, max_th)).to(t.device)
    occ = torch.empty(t.shape, dtype=torch.uint8, device=t.device) if return_occ else None
    hist, max_z = _confusion(t.shape, metric.n_classes, t.device, tsdf=t, th=th_t, axis=0, target=target, mask=fov,
                             per_z=True, occ=occ)
    mz = int(max_z.item())
    if mz < 0:
        raise ValueError("target has no occupied voxel (zero-size array to reduction operation maximum)")
    h = _crop_z(hist, mz)
    metric._add_hist(h[0], h[0])
    fov_metric._add_hist(h[1], h[1])
    if return_occ:
        occ[:, :, mz:] = 0
        return occ


# --- BundleFusion completion target ----------------------------------------------------------------------------------
BF_VOXEL_SIZE = 0.04
BF_VOL_BNDS = np.array([[-2.4, 2.4], [-2.4, 2.4], [0.0, 3.84]])     # generate_sc_gt_bf.py:280-286
BF_IMG = (480, 640)


def completion_target_bf(vol, voxel_size=BF_VOXEL_SIZE, device=None):
    """generate_sc_gt_bf.py:307-309: uint8 (X,Y,Z) on the device, 255 unknown / 0 free / 1 surface."""
    t = _volume(vol, device)
    out = torch.empty(t.shape, dtype=torch.uint8, device=t.device)
    _lib.check(_lib.load().srf_eval_sc_label(t.data_ptr(), _dims(t.shape), float(voxel_size), out.data_ptr(), _stream(t.device)))
    return out


def resize_bilinear(img, out_h, out_w, device=None):
    """F.interpolate(img[None, None], size=(out_h, out_w), mode="bilinear", align_corners=False) of one (H,W) image, with
    the arithmetic of ATen's CPU kernel (csrc/image_ops.cu)."""
    src = torch.as_tensor(img)
    dev = src.device if src.is_cuda else _device(device)
    src = src.to(device=dev, dtype=torch.float32).contiguous()
    if src.dim() != 2:
        raise ValueError("expected an (H,W) image, got shape %s" % (tuple(src.shape),))
    out = torch.empty((int(out_h), int(out_w)), dtype=torch.float32, device=dev)
    _lib.check(_lib.load().srf_resize_bilinear(src.data_ptr(), int(src.shape[0]), int(src.shape[1]), out.data_ptr(), int(out_h),
                                               int(out_w), _stream(dev)))
    return out


def fuse_completion_target_bf(source_depths, img_sources, cam_K, T_source2infers, voxel_size=BF_VOXEL_SIZE,
                              vol_bnds=BF_VOL_BNDS, img_size=BF_IMG, device=None):
    """generate_sc_gt_bf.py:280-309 for one frame, on the device: each source depth resized to 480x640, integrated with
    its colour (img_sources (N,3,H,W) in [0,1], times 255) into a TSDFVolume, then labelled.  Returns (volume, occ)."""
    from .tsdf import TSDFVolume
    dev = _device(device)
    vol = TSDFVolume(np.asarray(vol_bnds, dtype=np.float64), voxel_size=voxel_size, trunc_margin=10, device=dev)
    cam_K = np.asarray(torch.as_tensor(cam_K).detach().cpu().numpy())
    for depth, img, T in zip(source_depths, img_sources, T_source2infers):
        d = resize_bilinear(depth, img_size[0], img_size[1], device=dev)
        rgb = torch.as_tensor(img).to(device=dev, dtype=torch.float32).permute(1, 2, 0) * 255
        vol.integrate(rgb, d, cam_K, np.asarray(torch.as_tensor(T).detach().cpu().numpy()), obs_weight=1.)
    return vol, completion_target_bf(vol, voxel_size)


# --- depth metrics --------------------------------------------------------------------------------------------------
DEPTH_METRICS = ("abs_rel", "sq_rel", "rmse", "rmse_log", "a1", "a2", "a3")


def _depth_call(gt, pred, buckets, slot, frame, device):
    lib = _lib.load()
    g = torch.as_tensor(gt)
    dev = g.device if g.is_cuda else _device(device)
    g = g.to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
    p = torch.as_tensor(pred).to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
    if g.numel() != p.numel():
        raise ValueError("gt has %d elements, pred %d" % (g.numel(), p.numel()))
    ws_bytes = int(lib.srf_depth_errors_workspace_bytes())
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    _lib.check(lib.srf_depth_errors(g.data_ptr(), p.data_ptr(), int(g.numel()), ws.data_ptr(), ws_bytes,
                                    None if buckets is None else buckets.data_ptr(), int(slot),
                                    None if frame is None else frame.data_ptr(), _stream(dev)))


def compute_depth_errors(gt, pred, device=None):
    """loss/depth_metrics.py for one (gt, pred) pair: (abs_rel, sq_rel, rmse, rmse_log) as numpy float32 and (a1, a2, a3)
    as numpy float64, like the reference.  pred is clamped to [1e-3, 80] in the computation only (the reference clamps
    its argument in place).  Synchronises to return host values; DepthErrorBuckets.add does not."""
    dev = torch.as_tensor(gt).device if torch.as_tensor(gt).is_cuda else _device(device)
    frame = torch.empty(7, dtype=torch.float64, device=dev)
    _depth_call(gt, pred, None, 0, frame, dev)
    v = frame.cpu().numpy()
    return tuple(np.float32(x) for x in v[:4]) + tuple(np.float64(x) for x in v[4:])


class DepthErrorBuckets:
    """save_depth_metrics.py:98-131: per-frame depth errors summed by k = ceil(source_distance), with a frame count per
    k, held on the device (row k = 7 float64 sums + the count).  add() launches two kernels and never synchronises."""

    def __init__(self, device=None, max_distance: int = 16):
        self.device = _device(device)
        self.rows = torch.zeros((max(int(max_distance), 0) + 1, 8), dtype=torch.float64, device=self.device)

    def _grow(self, k):
        if k >= self.rows.shape[0]:
            more = torch.zeros((k + 1 - self.rows.shape[0], 8), dtype=torch.float64, device=self.device)
            self.rows = torch.cat([self.rows, more])

    def add(self, gt, pred, source_distance):
        k = math.ceil(float(source_distance))
        if k < 0:
            raise ValueError("source_distance %r < 0" % (source_distance,))
        self._grow(k)
        _depth_call(gt, pred, self.rows, k, None, self.device)

    def merge(self, other: "DepthErrorBuckets"):
        """Add another set of buckets (agg_depth_metrics.py:59-65)."""
        self._grow(other.rows.shape[0] - 1)
        self.rows[:other.rows.shape[0]] += other.rows.to(self.device)
        return self

    def as_dicts(self):
        """(agg_depth_errors {k: float64 (7,)}, n_frames {k: int}) in the reference's format."""
        rows = self.rows.cpu().numpy()
        ks = [k for k in range(rows.shape[0]) if rows[k, 7] > 0]
        return {k: rows[k, :7].copy() for k in ks}, {k: int(rows[k, 7]) for k in ks}

    def table(self):
        """print_metrics (save_depth_metrics.py:149-183) as text, one line per print."""
        agg, n_frames = self.as_dicts()
        lines = ["|distance|abs_rel |sq_rel  |rmse     |rmse_log|a1      |a2      |a3      |n_frames|"]
        total, total_frame = None, 0
        for distance in sorted(agg):
            total = np.copy(agg[distance]) if total is None else total + agg[distance]
            e, n = agg[distance], n_frames[distance]
            lines.append("|{:08d}|{:02.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:08d}|".format(
                distance, *[e[i] / n for i in range(7)], n))
            total_frame += n
        if total is None:
            raise ValueError("no frame added")
        lines.append("|{}|{:02.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:08d}|".format(
            "All     ", *[total[i] / total_frame for i in range(7)], total_frame))
        return "\n".join(lines) + "\n"

    def all_reduce(self, rank: int = 0, world: int = 1, group=None):
        """Sum the buckets of all ranks in rank order; afterwards every rank holds the same rows bit for bit."""
        if world > 1:
            import torch.distributed as dist
            n = torch.tensor([self.rows.shape[0]], dtype=torch.int64, device=self.device)
            sizes = [torch.empty_like(n) for _ in range(world)]
            dist.all_gather(sizes, n, group=group)
            self._grow(int(max(int(s.item()) for s in sizes)) - 1)
            self.rows = dist_sum(self.rows, rank, world, group).clone()
        return self


def dist_sum(t: torch.Tensor, rank: int = 0, world: int = 1, group=None) -> torch.Tensor:
    """All-gather `t` from every rank and sum the copies in rank order, so that every rank gets the same result bit for
    bit (an all-reduce may sum floating-point values in a rank-dependent order)."""
    if world <= 1:
        return t
    import torch.distributed as dist
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t.contiguous(), group=group)
    out = parts[0].clone()
    for p in parts[1:]:
        out += p
    return out
