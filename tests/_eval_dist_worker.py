"""torchrun worker of tests/test_eval.py::test_gpu_two_ranks_get_identical_stats: every rank scores its own frames,
the counts and depth buckets are summed across ranks in rank order, and every rank must hold the same totals bit for bit,
equal to one process scoring all the frames."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import eval_cases as EC                                 # noqa: E402
from scenerf_b200 import evaluation as E                # noqa: E402

SHAPE = (64, 48, 32)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    table = E.th_table_kitti(SHAPE[0])
    frames = [(EC.tsdf_volume(SHAPE, 400 + i, table, 0), EC.labels(SHAPE, 410 + i), EC.fov_mask(SHAPE, 420 + i)) for i in range(4)]
    depth = [EC.depth_pair(i, 5000) for i in range(4)]

    def score(idx):
        m, fm, b = E.SSCMetrics(2, device=dev), E.SSCMetrics(2, device=dev), E.DepthErrorBuckets(device=dev)
        for i in idx:
            E.score_reconstruction_kitti(frames[i][0], frames[i][1], frames[i][2], m, fm)
            b.add(depth[i][0], depth[i][1], EC.DEPTH_DISTANCES[i])
        return m, fm, b

    m, fm, b = score(range(rank, 4, world))
    m.all_reduce(rank, world)
    fm.all_reduce(rank, world)
    b.all_reduce(rank, world)
    mine = np.concatenate([np.array(m.counts()[:3] + fm.counts()[:3], dtype=np.float64), m.counts()[3], fm.counts()[5],
                           b.rows.cpu().numpy().ravel()])
    single_m, single_fm, _ = score(range(4))
    ok = m.counts()[:3] == single_m.counts()[:3] and fm.counts()[:3] == single_fm.counts()[:3]
    t = torch.from_numpy(mine).to(dev)
    parts = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(parts, t)
    ok = ok and all(torch.equal(parts[0], p) for p in parts)
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("EVAL_DIST_OK" if int(flag.item()) == 1 else "EVAL_DIST_MISMATCH", "world", world)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
