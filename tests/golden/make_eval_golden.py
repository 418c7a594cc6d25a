"""Golden vectors of the evaluation metrics (tests/golden/eval_metrics.npz), made by running the reference's own code on
the hash-generated inputs of tests/eval_cases.py:
  * SSCMetrics (loss/sscMetrics.py) and compute_depth_errors (loss/depth_metrics.py), imported directly;
  * tsdf2occ of scripts/evaluation/eval_sr.py and eval_sc_bf.py, imported with their dataset modules and imageio stubbed,
    and eval_sr.py's per-frame body (:79-87) restated around them;
  * generate_sc_gt_bf.main on one synthetic batch through a stubbed BundlefusionDM, with the reference's CPU
    fusion.TSDFVolume; the pickle it writes is read back.  A second run with a TSDFVolume stand-in whose get_volume
    returns an adversarial grid pins the labelling comparisons;
  * print_metrics of save_depth_metrics.py, with the per-source bucketing of its main loop (:122-131) restated.

Runs only where the reference tree exists (like make_goldens.py, which puts it on sys.path):
    python tests/golden/make_eval_golden.py"""
import contextlib
import hashlib
import io
import math
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_goldens  # noqa: E402  (puts the repository and the reference tree on sys.path)
import eval_cases as EC  # noqa: E402


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def import_reference():
    _stub("imageio", imread=None)
    _stub("scenerf.data.semantic_kitti.kitti_dm", KittiDataModule=None)
    _stub("scenerf.data.bundlefusion.bundlefusion_dm", BundlefusionDM=None)
    _stub("scenerf.models.scenerf", SceneRF=None)
    sk = _stub("skimage")
    sk.measure = _stub("skimage.measure")
    # get_mesh's result is discarded by generate_sc_gt_bf.py:304: an empty mesh keeps the run short
    sk.measure.marching_cubes_lewiner = lambda vol, level=0: (np.zeros((0, 3)), np.zeros((0, 3), dtype=np.int64),
                                                                np.zeros((0, 3)), np.zeros(0))
    from scenerf.loss.sscMetrics import SSCMetrics
    from scenerf.loss.depth_metrics import compute_depth_errors
    import scenerf.scripts.evaluation.eval_sr as eval_sr
    import scenerf.scripts.evaluation.eval_sc_bf as eval_sc_bf
    import scenerf.scripts.evaluation.save_depth_metrics as save_dm
    import scenerf.scripts.reconstruction.generate_sc_gt_bf as gen_bf
    import scenerf.data.utils.fusion as fusion
    fusion.measure = sk.measure
    return SSCMetrics, compute_depth_errors, eval_sr, eval_sc_bf, save_dm, gen_bf


def counts(m, prefix, out):
    out[prefix + "_ctp"], out[prefix + "_cfp"], out[prefix + "_cfn"] = m.completion_tp, m.completion_fp, m.completion_fn
    out[prefix + "_tps"], out[prefix + "_fps"], out[prefix + "_fns"] = m.tps, m.fps, m.fns
    s = m.get_stats()
    for k in ("precision", "recall", "iou", "iou_ssc_mean"):
        out["%s_%s" % (prefix, k)] = np.float64(s[k])
        out["%s_%s_type" % (prefix, k)] = type(s[k]).__name__
    out[prefix + "_iou_ssc"] = s["iou_ssc"]


def run_gen_bf(gen_bf, batch, tsdf_cls=None):
    depths, imgs, K, poses = batch
    b = {"cam_K_depth": torch.from_numpy(K)[None], "frame_id": ["000000"], "sequence": ["seq"],
         "infer_depths": torch.zeros(1, 1), "source_depths": [list(depths)],
         "img_sources": [[torch.from_numpy(i) for i in imgs]], "T_source2infers": [torch.from_numpy(poses)]}

    class DM:
        def __init__(self, **kw):
            pass

        def setup(self):
            pass

        def val_dataloader(self, shuffle=False):
            return [b]

    gen_bf.BundlefusionDM = DM
    saved = gen_bf.fusion.TSDFVolume
    if tsdf_cls is not None:
        gen_bf.fusion.TSDFVolume = tsdf_cls
    try:
        with tempfile.TemporaryDirectory() as d, contextlib.redirect_stdout(io.StringIO()):
            gen_bf.main.callback(root="", bs=1, n_gpus=1, n_workers_per_gpu=0, recon_save_dir=d)
            with open(os.path.join(d, "sc_gt", "seq", "000000.pkl"), "rb") as f:
                return pickle.load(f)
    finally:
        gen_bf.fusion.TSDFVolume = saved


def make():
    SSCMetrics, compute_depth_errors, eval_sr, eval_sc_bf, save_dm, gen_bf = import_reference()
    from scenerf_b200.evaluation import th_table_kitti, th_table_bf
    out = {}
    # KITTI: two frames of eval_sr.py:79-87 into the same pair of metrics
    tsdf = EC.tsdf_volume(EC.KITTI_SHAPE, 300, th_table_kitti(256), 0)
    targets = [EC.labels(EC.KITTI_SHAPE, 301, top_z=20), EC.labels(EC.KITTI_SHAPE, 302)]     # second: top slice = 31
    fov = EC.fov_mask(EC.KITTI_SHAPE, 303)
    metric, fov_metric = SSCMetrics(2), SSCMetrics(2)
    for i, target_1_1 in enumerate(targets):
        t = np.copy(target_1_1)
        t[target_1_1 == 255] = 0
        max_z = t.nonzero()[2].max()
        occ = eval_sr.tsdf2occ(tsdf, 0.25, 6.0)
        out["kitti_occ_sha%d" % i] = sha(occ.astype(np.uint8))
        occ[:, :, max_z:] = 0
        out["kitti_max_z%d" % i] = max_z
        out["kitti_cropped_occ_sha%d" % i] = sha(occ.astype(np.uint8))
        metric.add_batch(occ, target_1_1)
        fov_metric.add_batch(occ, target_1_1, fov)
    counts(metric, "kitti", out)
    counts(fov_metric, "kitti_fov", out)
    # BundleFusion: eval_sc_bf.py:203-210
    vs = 0.04
    tsdf_bf = EC.tsdf_volume(EC.BF_SHAPE, 310, th_table_bf(96, vs, 0.1, vs * 10, vs), 2)
    target_bf = EC.labels(EC.BF_SHAPE, 311)
    occ = eval_sc_bf.tsdf2occ(tsdf_bf, th=0.1, min_th=vs, max_th=vs * 10, voxel_size=vs)
    out["bf_occ_sha"] = sha(occ.astype(np.uint8))
    m = SSCMetrics(2)
    m.add_batch(occ, target_bf)
    counts(m, "bf", out)
    # SSCMetrics with semantic predictions, nonempty and nonsurface masks, 4 classes
    shp = (24, 20, 12)
    pred, target = EC.semantic_pred(shp, 320), EC.labels(shp, 321)
    ne, ns = EC.fov_mask(shp, 322), EC.fov_mask(shp, 323)
    for tag, kw in (("sem", {}), ("sem_ne", {"nonempty": ne}), ("sem_ns", {"nonsurface": ns}),
                    ("sem_ne_ns", {"nonempty": ne, "nonsurface": ns})):
        m = SSCMetrics(4)
        m.add_batch(pred, target, **kw)
        counts(m, tag, out)
    m = SSCMetrics(4)                                           # all-empty prediction: integer zeros from get_stats
    m.add_batch(np.zeros(shp), target)
    counts(m, "empty_pred", out)
    # completion target: the reference's fusion + labelling, then its labelling on the adversarial grid
    batch = EC.bf_batch()
    data = run_gen_bf(gen_bf, batch)
    out["bf_fused_tsdf_sha"], out["bf_sc_occ"] = sha(data["tsdf_grid"]), data["occ"]
    out["bf_fused_tsdf_shape"] = np.array(data["tsdf_grid"].shape)
    adv = EC.sc_label_tsdf()

    class FixedVolume:
        def __init__(self, *a, **k):
            pass

        def integrate(self, *a, **k):
            pass

        def get_mesh(self):
            return None, None, None, None

        def get_volume(self):
            return adv.copy(), None

    out["sc_label_adv"] = run_gen_bf(gen_bf, batch, FixedVolume)["occ"]
    # depth errors: per frame, bucketed by ceil(source distance), printed
    frames, agg, n_frames = [], {}, {}
    for i, dist in enumerate(EC.DEPTH_DISTANCES):
        gt, pred = EC.depth_pair(i)
        e = compute_depth_errors(gt=gt.copy(), pred=pred.copy())
        out["depth_types%d" % i] = np.array([type(v).__name__ for v in e])
        frames.append(np.array(e, dtype=np.float64))
        row = np.array([e]).sum(0)
        k = math.ceil(dist)
        if k not in agg:
            agg[k], n_frames[k] = row, 1
        else:
            agg[k] += row
            n_frames[k] += 1
    out["depth_frames"] = np.stack(frames)
    out["depth_bucket_keys"] = np.array(sorted(agg))
    out["depth_bucket_rows"] = np.stack([agg[k] for k in sorted(agg)])
    out["depth_bucket_frames"] = np.array([n_frames[k] for k in sorted(agg)])
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        save_dm.print_metrics(agg, n_frames)
    out["depth_table"] = np.array(buf.getvalue())
    return out


if __name__ == "__main__":
    g = make()
    path = os.path.join(HERE, "eval_metrics.npz")
    np.savez_compressed(path, **g)
    print("%-32s %8.1f KB  keys=%d" % ("eval_metrics", os.path.getsize(path) / 1024.0, len(g)))
