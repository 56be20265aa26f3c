"""Pair sharding over GPUs through the C-ABI NCCL communicator (needs >= 2 GPUs:
`python -m pytest tests/test_multi_gpu.py -m gpu`).  The host-side sharding logic
is covered on CPU with gloo (tests/test_dist_gloo.py)."""
import ctypes
import os
import subprocess
import sys

import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpu_count():
    try:
        cuda = ctypes.CDLL("libcuda.so.1")
        n = ctypes.c_int(0)
        return n.value if (cuda.cuInit(0) == 0 and cuda.cuDeviceGetCount(ctypes.byref(n)) == 0) else 0
    except OSError:
        return 0


@pytest.mark.skipif(_gpu_count() < 2, reason="needs two GPUs")
def test_pair_sharding_two_ranks_matches_single_gpu():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29541", os.path.join(ROOT, "tests", "multi_gpu_worker.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=800)
    assert r.returncode == 0 and "MULTI_GPU_OK" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
