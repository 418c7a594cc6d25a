"""GPU, multi-process: the NCCL paths of scenerf_b200.dist on real hardware (needs >= 2 GPUs; skipped on a 1-GPU machine --
run with `python -m pytest tests/test_gpu_nccl.py -m gpu` where two or more GPUs are visible)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu


def test_ray_sharded_frame_equals_single_gpu_bit_for_bit():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs 2 GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    world = 4 if n >= 4 else 2
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", "29741", os.path.join(here, "_shard_dist_worker.py")]
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    print(p.stdout[-3000:])
    assert p.returncode == 0 and "SHARD_DIST_OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
