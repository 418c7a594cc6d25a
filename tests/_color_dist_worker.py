"""torchrun worker of tests/test_color_eval.py::test_gpu_two_ranks_get_identical_rows: every rank scores its own pairs into
ColorErrorBuckets, the buckets are summed across ranks in rank order, and every rank must hold the same rows bit for bit,
equal (to float64 rounding of the reordered sums) to one process scoring all the pairs."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import color_oracle as O                   # noqa: E402
from scenerf_b200 import evaluation as E               # noqa: E402
from scenerf_b200.perceptual import LPIPSVGG           # noqa: E402
from test_color_eval import color_eval_pairs           # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    net = LPIPSVGG(O.random_lpips_state_dict(7), dev)
    ok = True
    for dataset in ("kitti", "bf"):
        pairs = color_eval_pairs(dataset)

        def score(idx):
            b = E.ColorErrorBuckets(dataset, device=dev)
            for i in idx:
                img, gt = torch.from_numpy(pairs[i][0]).to(dev), torch.from_numpy(pairs[i][1]).to(dev)
                b.add(img, gt, pairs[i][2], lpips=net(img, gt))
            return b

        b = score(range(rank, len(pairs), world)).all_reduce(rank, world)
        single = score(range(len(pairs)))
        mine = b.rows.cpu().numpy()
        ref = np.stack([single.rows[single.keys[k]].cpu().numpy() for k in b.keys])
        finite = np.isfinite(ref)
        ok = ok and sorted(b.keys) == sorted(single.keys) and np.array_equal(np.isfinite(mine), finite)
        ok = ok and np.allclose(mine[finite], ref[finite], rtol=1e-12, atol=0) and np.array_equal(mine[~finite], ref[~finite])
        ok = ok and b.table() == single.table()
        t = b.rows.reshape(-1).contiguous()
        parts = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(parts, t)
        ok = ok and all(p.cpu().numpy().tobytes() == parts[0].cpu().numpy().tobytes() for p in parts)
    flag = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("COLOR_DIST_OK" if int(flag.item()) == 1 else "COLOR_DIST_MISMATCH", "world", world)
    dist.destroy_process_group()
    sys.exit(0 if int(flag.item()) == 1 else 1)


if __name__ == "__main__":
    main()
