"""numpy restatement of the reference's evaluation arithmetic, in its operation order (reference file:line cited), for the
tests of scenerf_b200.evaluation (csrc/metrics.cu, DESIGN.md 6.7).  It restates, it does not import: the goldens of
tests/golden/make_eval_golden.py are made by the reference's own code, and tests/test_eval.py checks this file
against them on the CPU and the CUDA path against both on the GPU."""
from __future__ import annotations

import numpy as np
import torch

from oracle.tsdf_oracle import TSDFVolumeOracle


# --- tsdf2occ ----------------------------------------------------------------------------------------------------
def th_table_kitti(n, th=0.25, max_th=6.0):
    """eval_sr.py:13-15 (n = 256 there): float64, clamped below at 0.2 and above at max_th."""
    t = (0.1 + np.arange(n) * 0.2) * th
    t[t < 0.2] = 0.2
    t[t > max_th] = max_th
    return t


def th_table_bf(n, min_th, th=0.25, max_th=0.2, voxel_size=0.04):
    """eval_sc_bf.py:119-121 (n = 96 there)."""
    t = voxel_size + np.arange(n) * voxel_size * th
    t[t < min_th] = min_th
    t[t > max_th] = max_th
    return t


def tsdf2occ(tsdf, table, axis):
    """eval_sr.py:16 / eval_sc_bf.py:122 with the table along `axis` (0 for KITTI, 2 for BundleFusion); float64 0/1."""
    shape = [1, 1, 1]
    shape[axis] = len(table)
    occ = np.zeros(tsdf.shape)
    occ[(np.abs(tsdf) < table.reshape(shape)) & (np.abs(tsdf) != 255)] = 1
    return occ


def kitti_max_z(target):
    """eval_sr.py:79-81."""
    t = np.copy(target)
    t[target == 255] = 0
    return t.nonzero()[2].max()


# --- SSCMetrics (loss/sscMetrics.py:361-529) ---------------------------------------------------------------------
class SSCMetricsOracle:
    def __init__(self, n_classes):
        self.n_classes = n_classes
        self.reset()

    def reset(self):
        self.completion_tp = self.completion_fp = self.completion_fn = 0
        self.tps = np.zeros(self.n_classes)
        self.fps = np.zeros(self.n_classes)
        self.fns = np.zeros(self.n_classes)

    def add_batch(self, y_pred, y_true, nonempty=None, nonsurface=None):
        """:391-413.  The 3-D volume is flattened whole: the reference's per-x loop only changes the summation order of
        integer counts."""
        y_pred, y_true = np.asarray(y_pred).reshape(-1), np.asarray(y_true).reshape(-1)
        mask = y_true != 255
        if nonempty is not None:
            mask = mask & np.asarray(nonempty).reshape(-1)
        if nonsurface is not None:
            mask = mask & np.asarray(nonsurface).reshape(-1)
        sel = mask == 1                                               # :478-480
        bt, bp = y_true[sel] > 0, y_pred[sel] > 0                    # :462-471 (255 never selected)
        self.completion_tp += int(np.sum(bt & bp))
        self.completion_fp += int(np.sum(~bt & bp))
        self.completion_fn += int(np.sum(bt & ~bp))
        mask = y_true != 255
        if nonempty is not None:
            mask = mask & np.asarray(nonempty).reshape(-1)
        sel = mask == 1                                               # :513-519
        yt, yp = y_true[sel], y_pred[sel]
        for j in range(self.n_classes):                              # :520-527
            self.tps[j] += int(np.sum((yt == j) & (yp == j)))
            self.fps[j] += int(np.sum((yt != j) & (yp == j)))
            self.fns[j] += int(np.sum((yt == j) & (yp != j)))

    def get_stats(self):
        """:415-432."""
        if self.completion_tp != 0:
            precision = self.completion_tp / (self.completion_tp + self.completion_fp)
            recall = self.completion_tp / (self.completion_tp + self.completion_fn)
            iou = self.completion_tp / (self.completion_tp + self.completion_fp + self.completion_fn)
        else:
            precision, recall, iou = 0, 0, 0
        iou_ssc = self.tps / (self.tps + self.fps + self.fns + 1e-5)
        return {"precision": precision, "recall": recall, "iou": iou, "iou_ssc": iou_ssc, "iou_ssc_mean": np.mean(iou_ssc[1:])}


def score_reconstruction_kitti(tsdf, target, fov_mask, metric, fov_metric, th=0.25, max_th=6.0):
    """eval_sr.py:79-87."""
    max_z = kitti_max_z(target)
    occ = tsdf2occ(tsdf, th_table_kitti(tsdf.shape[0], th, max_th), 0)
    occ[:, :, max_z:] = 0
    metric.add_batch(occ, target)
    fov_metric.add_batch(occ, target, fov_mask)
    return occ


# --- BundleFusion completion target (generate_sc_gt_bf.py:288-309) -------------------------------------------------
def sc_label(tsdf_grid, voxel_size):
    """:307-309; numpy compares the float32 grid with the Python float in float32."""
    occ = np.zeros_like(tsdf_grid) + 255
    occ[(tsdf_grid > voxel_size) & (tsdf_grid != 255)] = 0
    occ[(abs(tsdf_grid) < voxel_size) & (tsdf_grid != 255)] = 1
    return occ.astype(np.uint8)


def _fma(a, b, c):
    """float32 fma(a, b, c): the float32 product is exact in float64 (rounding the float64 sum once more can differ from a
    true fma only on a float64 tie, far rarer than any test here needs)."""
    return (np.float64(a) * np.float64(b) + np.float64(c)).astype(np.float32)


def resize_bilinear(img, out_h, out_w):
    """F.interpolate(size=(out_h, out_w), mode="bilinear", align_corners=False) of one float32 CPU image as ATen's CPU
    kernel computes it (csrc/image_ops.cu resize_bilinear_kernel): src = fma(float(in/out), dst+0.5, -0.5) clamped at 0,
    weights in float32, lerp(a, wa, b, wb) = fma(a, wa, b*wb), the two x lerps then the y lerp."""
    img = np.asarray(img, dtype=np.float32)
    in_h, in_w = img.shape

    def taps(n_out, n_in):
        scale = np.float32(n_in) / np.float32(n_out)
        src = _fma(scale, np.arange(n_out, dtype=np.float32) + np.float32(0.5), np.float32(-0.5))
        src = np.maximum(src, np.float32(0))
        i0 = np.minimum(src.astype(np.int64), n_in - 1)
        i1 = i0 + (i0 < n_in - 1)
        w1 = np.clip(src - i0.astype(np.float32), np.float32(0), np.float32(1))
        return i0, i1, np.float32(1) - w1, w1

    def lerp(a, wa, b, wb):
        return _fma(a, wa, b * wb)

    x0, x1, wx0, wx1 = taps(out_w, in_w)
    y0, y1, wy0, wy1 = taps(out_h, in_h)
    r0 = lerp(img[y0][:, x0], wx0, img[y0][:, x1], wx1)
    r1 = lerp(img[y1][:, x0], wx0, img[y1][:, x1], wx1)
    return lerp(r0, wy0[:, None], r1, wy1[:, None])


BF_VOXEL_SIZE = 0.04
BF_VOL_BNDS = np.array([[-2.4, 2.4], [-2.4, 2.4], [0.0, 3.84]])      # :280-286
BF_IMG = (480, 640)


def fuse_completion_target_bf(source_depths, img_sources, cam_K, T_source2infers):
    """:288-309 for one frame: resize each source depth to 480x640, integrate (fusion.TSDFVolume, CPU path), label.
    img_sources (N,3,480,640) float in [0,1].  Returns (tsdf_grid float32, occ uint8)."""
    vol = TSDFVolumeOracle(BF_VOL_BNDS.copy(), voxel_size=BF_VOXEL_SIZE, trunc_margin=10)
    for depth, img, T in zip(source_depths, img_sources, T_source2infers):
        d = resize_bilinear(depth, *BF_IMG)
        rgb = np.transpose(np.asarray(img, dtype=np.float32), (1, 2, 0)) * 255
        vol.integrate(rgb, d, cam_K, T, obs_weight=1.)
    tsdf_grid, _ = vol.get_volume()
    return tsdf_grid, sc_label(tsdf_grid, BF_VOXEL_SIZE)


def resize_bilinear_torch(img, out_h, out_w):
    """The reference's own call (:296-297), for comparison with resize_bilinear."""
    t = torch.from_numpy(np.asarray(img, dtype=np.float32)).unsqueeze(0).unsqueeze(0)
    return torch.nn.functional.interpolate(t, size=(out_h, out_w), mode="bilinear", align_corners=False).squeeze().numpy()


# --- depth metrics (loss/depth_metrics.py, save_depth_metrics.py:98-183) -----------------------------------------
def compute_depth_errors(gt, pred, min_depth=1e-3, max_depth=80):
    """depth_metrics.py:3-24 on float32 arrays (pred is copied, not clamped in place)."""
    gt = np.asarray(gt, dtype=np.float32)
    pred = np.array(pred, dtype=np.float32)
    pred[pred < min_depth] = min_depth
    pred[pred > max_depth] = max_depth
    thresh = np.maximum((gt / pred), (pred / gt))
    a1 = (thresh < 1.25).mean()
    a2 = (thresh < 1.25 ** 2).mean()
    a3 = (thresh < 1.25 ** 3).mean()
    rmse = np.sqrt(((gt - pred) ** 2).mean())
    rmse_log = np.sqrt(((np.log(gt) - np.log(pred)) ** 2).mean())
    abs_rel = np.mean(np.abs(gt - pred) / gt)
    sq_rel = np.mean(((gt - pred) ** 2) / gt)
    return abs_rel, sq_rel, rmse, rmse_log, a1, a2, a3


def bucket_add(agg, n_frames, depth_errors, source_distance):
    """save_depth_metrics.py:27,124-131: the frame's 7-tuple as a float64 row, summed per ceil(distance)."""
    import math
    row = np.array([depth_errors]).sum(0)
    k = math.ceil(source_distance)
    if k not in agg:
        agg[k] = row
        n_frames[k] = 1
    else:
        agg[k] += row
        n_frames[k] += 1


def metrics_table(agg_depth_errors, n_frames):
    """save_depth_metrics.py:149-183 print_metrics, returned as text (one line per print)."""
    lines = ["|distance|abs_rel |sq_rel  |rmse     |rmse_log|a1      |a2      |a3      |n_frames|"]
    total, total_frame = None, 0
    for distance in sorted(agg_depth_errors):
        total = np.copy(agg_depth_errors[distance]) if total is None else total + agg_depth_errors[distance]
        e, n = agg_depth_errors[distance], n_frames[distance]
        lines.append("|{:08d}|{:02.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:08d}|".format(
            distance, e[0] / n, e[1] / n, e[2] / n, e[3] / n, e[4] / n, e[5] / n, e[6] / n, n))
        total_frame += n
    lines.append("|{}|{:02.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:.6f}|{:08d}|".format(
        "All     ", *[total[i] / total_frame for i in range(7)], total_frame))
    return "\n".join(lines) + "\n"
