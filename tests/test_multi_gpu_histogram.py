"""The sharded histogram_quantile over the library's own NCCL path on real GPUs (needs >= 2 visible devices; skipped
on a single-GPU box): launches tests/multi_gpu_histogram_check.py under torchrun, one rank per GPU, and reads its verdict
line.  A small exchange cap makes the shuffle run in several batches."""
import os
import subprocess
import sys

import pytest

from tests.ranks import free_port

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("cap", [None, 64 << 10])
def test_sharded_histogram_quantile_over_the_library_communicator(cap):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least two GPUs")
    world = 2 if n < 4 else 4
    env = dict(os.environ)
    if cap:
        env["B2P_TOPK_EXCHANGE_BYTES"] = str(cap)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
                        os.path.join(ROOT, "tests", "multi_gpu_histogram_check.py")], capture_output=True, text=True,
                       timeout=900, env=env)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "MULTI_GPU_HISTOGRAM_CHECK" in r.stdout and "ok=True" in r.stdout, r.stdout[-2000:]
