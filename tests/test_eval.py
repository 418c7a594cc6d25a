"""Evaluation metrics (csrc/metrics.cu, scenerf_b200/evaluation.py, DESIGN.md 6.7).  CPU: the numpy oracle against the
golden made by the reference's own SSCMetrics, tsdf2occ, generate_sc_gt_bf.main, compute_depth_errors and print_metrics
(tests/golden/make_eval_golden.py), and argument validation of the C entries.  GPU: the CUDA path against both."""
import ctypes as C
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import eval_cases as EC
from cases import load_golden
from oracle import eval_oracle as O
from scenerf_b200 import _lib


@pytest.fixture(scope="module")
def g():
    return load_golden("eval_metrics")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def kitti_inputs():
    tsdf = EC.tsdf_volume(EC.KITTI_SHAPE, 300, O.th_table_kitti(256), 0)
    targets = [EC.labels(EC.KITTI_SHAPE, 301, top_z=20), EC.labels(EC.KITTI_SHAPE, 302)]
    return tsdf, targets, EC.fov_mask(EC.KITTI_SHAPE, 303)


def bf_inputs():
    vs = 0.04
    return EC.tsdf_volume(EC.BF_SHAPE, 310, O.th_table_bf(96, vs, 0.1, vs * 10, vs), 2), EC.labels(EC.BF_SHAPE, 311)


SEM_SHAPE = (24, 20, 12)


def sem_inputs():
    s = SEM_SHAPE
    return EC.semantic_pred(s, 320), EC.labels(s, 321), EC.fov_mask(s, 322), EC.fov_mask(s, 323)


SEM_CASES = (("sem", False, False), ("sem_ne", True, False), ("sem_ns", False, True), ("sem_ne_ns", True, True))


def assert_metric(m, g, prefix):
    """Counts equal, stats equal to the last bit and of the reference's types."""
    assert m.completion_tp == g[prefix + "_ctp"] and m.completion_fp == g[prefix + "_cfp"] and m.completion_fn == g[prefix + "_cfn"]
    for k in ("tps", "fps", "fns"):
        assert np.array_equal(getattr(m, k), g["%s_%s" % (prefix, k)]), (prefix, k)
    s = m.get_stats()
    for k in ("precision", "recall", "iou", "iou_ssc_mean"):
        assert type(s[k]).__name__ == str(g["%s_%s_type" % (prefix, k)]), (prefix, k, type(s[k]))
        assert np.float64(s[k]).tobytes() == g["%s_%s" % (prefix, k)].tobytes(), (prefix, k)
    assert s["iou_ssc"].dtype == np.float64 and s["iou_ssc"].tobytes() == g[prefix + "_iou_ssc"].tobytes()


class _Counts:
    """The accumulator fields of a device SSCMetrics, for assert_metric."""

    def __init__(self, m):
        self.completion_tp, self.completion_fp, self.completion_fn, self.tps, self.fps, self.fns = m.counts()
        self._m = m

    def get_stats(self):
        return self._m.get_stats()


# --- CPU: the oracle against the reference's goldens -------------------------------------------------------------------
def test_oracle_kitti_scores_match_reference(g):
    tsdf, targets, fov = kitti_inputs()
    m, fm = O.SSCMetricsOracle(2), O.SSCMetricsOracle(2)
    for i, t in enumerate(targets):
        assert sha(O.tsdf2occ(tsdf, O.th_table_kitti(256), 0).astype(np.uint8)) == g["kitti_occ_sha%d" % i]
        assert O.kitti_max_z(t) == g["kitti_max_z%d" % i]
        occ = O.score_reconstruction_kitti(tsdf, t, fov, m, fm)
        assert sha(occ.astype(np.uint8)) == g["kitti_cropped_occ_sha%d" % i]
    assert g["kitti_max_z1"] == EC.KITTI_SHAPE[2] - 1            # the second target's top labelled slice is the last one
    assert_metric(m, g, "kitti")
    assert_metric(fm, g, "kitti_fov")


def test_oracle_bf_and_semantic_scores_match_reference(g):
    tsdf, target = bf_inputs()
    occ = O.tsdf2occ(tsdf, O.th_table_bf(96, 0.04, 0.1, 0.4, 0.04), 2)
    assert sha(occ.astype(np.uint8)) == g["bf_occ_sha"]
    m = O.SSCMetricsOracle(2)
    m.add_batch(occ, target)
    assert_metric(m, g, "bf")
    pred, target, ne, ns = sem_inputs()
    for tag, use_ne, use_ns in SEM_CASES:
        m = O.SSCMetricsOracle(4)
        m.add_batch(pred, target, ne if use_ne else None, ns if use_ns else None)
        assert_metric(m, g, tag)
    m = O.SSCMetricsOracle(4)
    m.add_batch(np.zeros(SEM_SHAPE), target)
    assert_metric(m, g, "empty_pred")


def test_oracle_completion_target_matches_reference(g):
    assert np.array_equal(O.sc_label(EC.sc_label_tsdf(), 0.04), g["sc_label_adv"])
    tsdf, occ = O.fuse_completion_target_bf(*EC.bf_batch())
    assert tsdf.shape == tuple(g["bf_fused_tsdf_shape"])
    assert sha(tsdf) == g["bf_fused_tsdf_sha"]
    assert np.array_equal(occ, g["bf_sc_occ"])


def test_oracle_resize_matches_torch_cpu():
    d = EC.bf_batch()[0]
    for img in (d[0], d[1][:37, :53]):
        assert np.array_equal(O.resize_bilinear(img, 480, 640), O.resize_bilinear_torch(img, 480, 640))


def test_oracle_depth_errors_and_table_match_reference(g):
    agg, n_frames = {}, {}
    for i, dist in enumerate(EC.DEPTH_DISTANCES):
        e = O.compute_depth_errors(*EC.depth_pair(i))
        assert [type(v).__name__ for v in e] == list(g["depth_types%d" % i])
        assert np.array_equal(np.array(e, dtype=np.float64), g["depth_frames"][i])
        O.bucket_add(agg, n_frames, e, dist)
    assert list(sorted(agg)) == list(g["depth_bucket_keys"])
    assert np.array_equal(np.stack([agg[k] for k in sorted(agg)]), g["depth_bucket_rows"])
    assert O.metrics_table(agg, n_frames) == str(g["depth_table"])


# --- CPU: argument validation of the C entries (no device needed: every check runs before a launch) ---------------------
def test_eval_abi_validation():
    lib = _lib.load()
    dims = (C.c_int * 3)(256, 256, 32)
    fake = C.c_void_p(0x1000)
    assert lib.srf_eval_hist_len(dims, 2, 1) == 32 * 2 * 3 * 4
    assert lib.srf_eval_hist_len(dims, 2, 0) == 2 * 3 * 4
    assert lib.srf_eval_hist_len(dims, 0, 0) == 0 and lib.srf_eval_hist_len(dims, 65, 0) == 0
    args = lambda **kw: [kw.get(k, v) for k, v in (
        ("tsdf", fake), ("pred", None), ("dtype", 0), ("target", fake), ("mask", None), ("dims", dims), ("C", 2), ("axis", 0),
        ("th", fake), ("per_z", 1), ("hist", fake), ("max_z", fake), ("occ", None), ("stream", None))]
    for bad in (dict(dims=(C.c_int * 3)(0, 256, 32)), dict(C=0), dict(C=65), dict(hist=None), dict(max_z=None),
                dict(target=None), dict(tsdf=None), dict(th=None), dict(axis=3), dict(pred=fake, dtype=7),
                dict(C=64, dims=(C.c_int * 3)(8, 8, 64))):
        assert lib.srf_eval_confusion(*args(**bad)) == 1, bad
    assert b"srf_eval_confusion" in lib.srf_last_error()
    assert lib.srf_eval_sc_label(None, dims, 0.04, fake, None) == 1
    assert lib.srf_eval_sc_label(fake, (C.c_int * 3)(1, 0, 1), 0.04, fake, None) == 1
    assert lib.srf_resize_bilinear(fake, 0, 10, fake, 480, 640, None) == 1
    assert lib.srf_resize_bilinear(fake, 10, 10, None, 480, 640, None) == 1
    ws = lib.srf_depth_errors_workspace_bytes()
    assert ws > 0
    assert lib.srf_depth_errors(fake, fake, 0, fake, ws, fake, 0, None, None) == 1
    assert lib.srf_depth_errors(fake, fake, 10, fake, ws, None, 0, None, None) == 1
    assert lib.srf_depth_errors(fake, fake, 10, fake, ws, fake, -1, None, None) == 1
    assert lib.srf_depth_errors(fake, fake, 10, fake, ws - 1, fake, 0, None, None) == 2


# --- GPU ------------------------------------------------------------------------------------------------------------
def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("on_device", [False, True])
def test_gpu_kitti_scores_equal_reference(g, on_device):
    from scenerf_b200 import evaluation as E
    tsdf, targets, fov = kitti_inputs()
    conv = _dev if on_device else (lambda x: x)
    assert sha(E.tsdf2occ_kitti(conv(tsdf)).cpu().numpy()) == g["kitti_occ_sha0"]
    m, fm = E.SSCMetrics(2), E.SSCMetrics(2)
    om, ofm = O.SSCMetricsOracle(2), O.SSCMetricsOracle(2)
    for i, t in enumerate(targets):
        occ = E.score_reconstruction_kitti(conv(tsdf), conv(t), conv(fov), m, fm, return_occ=True)
        assert sha(occ.cpu().numpy()) == g["kitti_cropped_occ_sha%d" % i]
        O.score_reconstruction_kitti(tsdf, t, fov, om, ofm)
    assert_metric(_Counts(m), g, "kitti")
    assert_metric(_Counts(fm), g, "kitti_fov")
    assert m.counts()[:3] == (om.completion_tp, om.completion_fp, om.completion_fn)
    # the same frames through add_batch with the oracle's cropped occupancy (float64, numpy or device)
    m2, fm2 = E.SSCMetrics(2), E.SSCMetrics(2)
    for t in targets:
        occ = O.tsdf2occ(tsdf, O.th_table_kitti(256), 0)
        occ[:, :, O.kitti_max_z(t):] = 0
        m2.add_batch(conv(occ), conv(t))
        fm2.add_batch(conv(occ), conv(t), conv(fov))
    assert_metric(_Counts(m2), g, "kitti")
    assert_metric(_Counts(fm2), g, "kitti_fov")


@pytest.mark.gpu
@pytest.mark.parametrize("on_device", [False, True])
def test_gpu_bf_and_semantic_scores_equal_reference(g, on_device):
    from scenerf_b200 import evaluation as E
    conv = _dev if on_device else (lambda x: x)
    tsdf, target = bf_inputs()
    occ = E.tsdf2occ_bf(conv(tsdf), 0.04, th=0.1, max_th=0.4, voxel_size=0.04)
    assert sha(occ.cpu().numpy()) == g["bf_occ_sha"]
    m = E.SSCMetrics(2)
    m.add_batch(occ if on_device else occ.cpu().numpy(), conv(target))
    assert_metric(_Counts(m), g, "bf")
    fov = EC.fov_mask(EC.BF_SHAPE, 312)                   # with a mask: against the oracle
    m, om = E.SSCMetrics(2), O.SSCMetricsOracle(2)
    m.add_batch(occ, conv(target), conv(fov))
    om.add_batch(occ.cpu().numpy().astype(np.float64), target, fov)
    assert m.counts()[:3] == (om.completion_tp, om.completion_fp, om.completion_fn)
    assert np.array_equal(m.counts()[3], om.tps) and np.array_equal(m.counts()[5], om.fns)
    pred, target, ne, ns = sem_inputs()
    for tag, use_ne, use_ns in SEM_CASES:
        m = E.SSCMetrics(4)
        m.add_batch(conv(pred), conv(target), conv(ne) if use_ne else None, conv(ns) if use_ns else None)
        assert_metric(_Counts(m), g, tag)
    m = E.SSCMetrics(4)
    m.add_batch(conv(np.zeros(SEM_SHAPE)), conv(target))
    assert_metric(_Counts(m), g, "empty_pred")
    m.reset()
    assert m.get_stats()["iou"] == 0 and type(m.get_stats()["iou"]) is int


@pytest.mark.gpu
def test_gpu_empty_target_raises():
    from scenerf_b200 import evaluation as E
    tsdf, _, fov = kitti_inputs()
    t = np.zeros(EC.KITTI_SHAPE, dtype=np.uint8)
    t[:, :, 3] = 255
    with pytest.raises(ValueError):
        E.score_reconstruction_kitti(tsdf, t, fov, E.SSCMetrics(2), E.SSCMetrics(2))
    with pytest.raises(ValueError):
        O.kitti_max_z(t)


@pytest.mark.gpu
def test_gpu_completion_target_equals_reference(g):
    from scenerf_b200 import evaluation as E
    assert np.array_equal(E.completion_target_bf(EC.sc_label_tsdf(), 0.04).cpu().numpy(), g["sc_label_adv"])
    depths, imgs, K, poses = EC.bf_batch()
    for img in (depths[0], depths[1][:37, :53]):
        assert np.array_equal(E.resize_bilinear(img, 480, 640).cpu().numpy(), O.resize_bilinear_torch(img, 480, 640))
    vol, occ = E.fuse_completion_target_bf(depths, imgs, K, poses)
    tsdf, _ = vol.get_volume()
    assert sha(tsdf) == g["bf_fused_tsdf_sha"]
    assert np.array_equal(occ.cpu().numpy(), g["bf_sc_occ"])


@pytest.mark.gpu
def test_gpu_depth_errors_and_buckets(g):
    from scenerf_b200 import evaluation as E
    b, half = E.DepthErrorBuckets(max_distance=2), [E.DepthErrorBuckets(), E.DepthErrorBuckets()]
    frames, agg, n_frames = [], {}, {}
    for i, dist in enumerate(EC.DEPTH_DISTANCES):
        gt, pred = EC.depth_pair(i)
        e = E.compute_depth_errors(_dev(gt), _dev(pred))
        ref = g["depth_frames"][i]
        assert [type(v).__name__ for v in e] == list(g["depth_types%d" % i])
        assert np.array_equal(np.array(e[4:]), ref[4:])                           # a1..a3 exact
        assert np.allclose(np.array(e[:4], dtype=np.float64), ref[:4], rtol=1e-6, atol=0)
        frames.append(e)
        O.bucket_add(agg, n_frames, e, dist)
        b.add(_dev(gt), _dev(pred), dist)
        half[i % 2].add(gt, pred, dist)
    rows_agg, rows_n = b.as_dicts()
    assert sorted(rows_agg) == list(g["depth_bucket_keys"]) and [rows_n[k] for k in sorted(rows_n)] == list(g["depth_bucket_frames"])
    for k in agg:                              # the device buckets add the device frames exactly as the reference's loop
        assert rows_agg[k].tobytes() == agg[k].tobytes() and rows_n[k] == n_frames[k]
    assert np.allclose(np.stack([rows_agg[k] for k in sorted(rows_agg)]), g["depth_bucket_rows"], rtol=1e-6, atol=0)
    assert b.table() == O.metrics_table(agg, n_frames)
    # against the reference's printout: same layout, every printed number within one unit of its last place (the
    # reference's float32 pairwise means and the device's float64 sums can round the 6th decimal differently)
    got, want = b.table().splitlines(), str(g["depth_table"]).splitlines()
    assert len(got) == len(want) and got[0] == want[0]
    for lg, lw in zip(got[1:], want[1:]):
        fg, fw = lg.split("|"), lw.split("|")
        assert len(fg) == len(fw) and fg[1] == fw[1] and fg[-2] == fw[-2]
        assert all(abs(float(a) - float(c)) <= 1.5e-6 for a, c in zip(fg[2:-2], fw[2:-2])), (lg, lw)
    merged = half[0].merge(half[1]).as_dicts()
    for k in agg:
        assert np.allclose(merged[0][k], agg[k], rtol=1e-12) and merged[1][k] == n_frames[k]


@pytest.mark.gpu
def test_gpu_score_of_sweep_reconstruction_equals_oracle():
    import torch
    from scenerf_b200 import evaluation as E, sweep
    from cases import load_golden as lg
    from test_sweep import _renderer, N_POSES
    sg = lg("sweep_kitti")
    cfg, r, x_rgb = _renderer("fp32")
    sw = sweep.NovelDepthSweep(r, torch.from_numpy(cfg.K).cuda(), x_rgb, img_size=(244, 74), scale=4)
    poses = sweep.sample_rel_poses(step=1.0, angle=10, max_distance=1.1)
    noises = [(torch.from_numpy(sg["noise_u%d" % i]), torch.from_numpy(sg["noise_n%d" % i])) for i in range(N_POSES)]
    vol = sw.reconstruct(poses, sg["T_velo2cam"], sg["vol_bnds"], noises=noises)
    tsdf, _ = vol.get_volume()
    target, fov = EC.labels(tsdf.shape, 330), EC.fov_mask(tsdf.shape, 331)
    m, fm, om, ofm = E.SSCMetrics(2), E.SSCMetrics(2), O.SSCMetricsOracle(2), O.SSCMetricsOracle(2)
    E.score_reconstruction_kitti(vol, target, fov, m, fm)
    O.score_reconstruction_kitti(tsdf, target, fov, om, ofm)
    for dev_m, orc in ((m, om), (fm, ofm)):
        tp, fp, fn, tps, fps, fns = dev_m.counts()
        assert (tp, fp, fn) == (orc.completion_tp, orc.completion_fp, orc.completion_fn)
        assert np.array_equal(tps, orc.tps) and np.array_equal(fps, orc.fps) and np.array_equal(fns, orc.fns)
        assert dev_m.get_stats()["iou"] == orc.get_stats()["iou"]


@pytest.mark.gpu
def test_gpu_two_ranks_get_identical_stats():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29743", os.path.join(here, "_eval_dist_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "EVAL_DIST_OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
