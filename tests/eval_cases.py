"""Hash-generated inputs of the evaluation golden (tests/golden/make_eval_golden.py) and tests (tests/test_eval.py),
with the adversarial values that decide every comparison: float32 tsdf values on both sides of every distinct
threshold, +-255, |tsdf| == float32(voxel_size) and its neighbours, 255s and labels >= n_classes in the targets, a target
whose top labelled slice is the last one, preds at and beyond the depth clamps and gt/pred ratios of exactly 1.25,
1.5625 and 1.953125."""
import numpy as np

from scenerf_b200 import synth

KITTI_SHAPE = (256, 256, 32)
BF_SHAPE = (120, 120, 96)


def _ulp_neighbours(values):
    """float32 values next to each float64 threshold: the float32 nearest it and one ulp either side."""
    v = np.asarray(values, dtype=np.float64).astype(np.float32)
    return np.stack([np.nextafter(v, np.float32(-np.inf)), v, np.nextafter(v, np.float32(np.inf))], axis=1)


def tsdf_volume(shape, seed, table, axis):
    """tsdf in [-3, 3) with 10 % unobserved (255) and a few -255; along `axis`, index i carries the float32 neighbours
    of table[i] (both signs) on its first rows."""
    n = int(np.prod(shape))
    t = (synth.hash_uniform(seed, n) * np.float32(3.0)).reshape(shape)
    u = synth.hash_unit(seed + 1, n).reshape(shape)
    t[u < 0.10] = 255.0
    t[u > 0.995] = -255.0
    vals = _ulp_neighbours(table)                              # (len, 3)
    vals = np.concatenate([vals, -vals], axis=1)              # (len, 6)
    m = np.moveaxis(t, axis, 0)                               # view: m[i] is the slab at index i along `axis`
    for i in range(m.shape[0]):
        flat = m[i].reshape(-1)
        flat[:6] = vals[i]
        flat[6:8] = (255.0, -255.0)
        m[i] = flat.reshape(m[i].shape)
    return t


def labels(shape, seed, top_z=None):
    """uint8 labels: 0 (60 %), 1 (22 %), 255 (10 %), 2..5 (8 %); nothing but 0 above z = top_z when given."""
    n = int(np.prod(shape))
    u = synth.hash_unit(seed, n).reshape(shape)
    y = np.zeros(shape, dtype=np.uint8)
    y[u >= 0.60] = 1
    y[u >= 0.82] = 255
    y[u >= 0.92] = (2 + (u[u >= 0.92] * 1000).astype(np.int64) % 4).astype(np.uint8)
    if top_z is not None:
        y[:, :, top_z + 1:][y[:, :, top_z + 1:] != 255] = 0
    return y


def fov_mask(shape, seed):
    return synth.hash_unit(seed, int(np.prod(shape))).reshape(shape) < 0.6


def semantic_pred(shape, seed):
    """float64 predictions with class values, an out-of-range class, a negative and a fraction."""
    choices = np.array([0, 1, 2, 3, 5, -1, 0.5, 0, 0, 1], dtype=np.float64)
    idx = (synth.hash_unit(seed, int(np.prod(shape))) * len(choices)).astype(np.int64) % len(choices)
    return choices[idx].reshape(shape)


def sc_label_tsdf():
    """(8, 8, 6) float32 grid around +-float32(0.04) and +-0.04, plus +-255 and random values."""
    vs = np.float32(0.04)
    special = [vs, np.nextafter(vs, np.float32(1)), np.nextafter(vs, np.float32(-1)), np.float32(np.float64(0.04)),
               0.0, 255.0, -255.0, 1.0, 0.5, 0.03, 0.05]
    special = np.array(special + [-v for v in special], dtype=np.float32)
    t = synth.hash_uniform(91, 8 * 8 * 6).astype(np.float32) * np.float32(0.1)
    t[:special.size] = special
    return t.reshape(8, 8, 6)


# --- BundleFusion completion target: one frame of three sources -------------------------------------------------------
BF_SRC = (120, 160)


def bf_batch():
    """(source_depths (3, 120, 160) float32, img_sources (3, 3, 480, 640) float32 in [0,1], cam_K (3,3) float32,
    T_source2infers (3, 4, 4) float64)."""
    H, W = BF_SRC
    depths, imgs, poses = [], [], []
    for i, (yaw, tz) in enumerate(((0.0, 0.0), (8.0, -0.3), (-6.0, 0.2))):
        d = (1.2 + 2.0 * synth.hash_unit(120 + i, H * W).reshape(H, W) + np.linspace(0, 0.6, W)[None, :]).astype(np.float32)
        d[synth.hash_unit(130 + i, H * W).reshape(H, W) < 0.05] = 0.0
        depths.append(d)
        imgs.append(synth.hash_unit(140 + i, 3 * 480 * 640).reshape(3, 480, 640))
        poses.append(synth.yaw_translate(yaw, tz).astype(np.float64))
    return np.stack(depths), np.stack(imgs).astype(np.float32), synth.BF_K.copy(), np.stack(poses)


# --- depth errors ---------------------------------------------------------------------------------------------------
DEPTH_DISTANCES = (0.3, 0.9, 1.0, 1.2, 2.5, 3.7, 0.0)


def depth_pair(i, n=20000):
    """gt in [1, 60], pred = gt times a factor in [0.5, 2) with exact-ratio, clamp and zero cases on the first rows."""
    gt = (1.0 + 59.0 * synth.hash_unit(200 + i, n)).astype(np.float32)
    pred = (gt * (0.5 + 1.5 * synth.hash_unit(210 + i, n))).astype(np.float32)
    g = [5.0, 4.0, 6.25, 4.0, 7.8125, 4.0, 2.0, 2.0, 2.0, 2.0, 2.0, 50.0, 50.0, 50.0, 50.0]
    p = [4.0, 5.0, 4.0, 6.25, 4.0, 7.8125, 0.0, 1e-4, 1e-3, -1.0, np.float32(1e-3), 80.0, 81.0, 1000.0, np.nextafter(np.float32(80), np.float32(100))]
    gt[:len(g)] = g
    pred[:len(p)] = np.asarray(p, dtype=np.float32)
    return gt, pred
