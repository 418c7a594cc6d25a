"""The float32 training path over several chunks of points: the 150-ray case of test_backward.py's edge sizes with
SRF_TRAIN_CHUNK=1024, i.e. a 9600-point main pass in 9 full chunks and a 384-point tail.  Covers what a single-chunk pass
cannot: the per-chunk scale flags of the saved activations, parameter gradients accumulated over chunks, and chunk tails
in the backward.  The chunk size is read once per process, so each case runs in a subprocess (_train_chunk_worker.py)."""
import os
import subprocess
import sys

import pytest


@pytest.mark.gpu
@pytest.mark.parametrize("matmul", ["fp32", "tf32"])
def test_cuda_backward_multi_chunk(matmul):
    """Against the float64 oracle with the bounds of test_cuda_backward_edge_sizes; fp32 also checks that recomputing the
    forward in the backward gives the same gradients as reading the saved activations, bit for bit."""
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_train_chunk_worker.py")
    cmd = [sys.executable, *(["-s"] if sys.flags.no_user_site else []), worker, matmul]
    p = subprocess.run(cmd, env=dict(os.environ, SRF_TRAIN_CHUNK="1024"), capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and "TRAIN_CHUNK_OK" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
    print(p.stdout.strip())
