"""The sharded plan nodes over the library's NCCL communicator on real GPUs (needs >= 2 visible devices; skipped on a
single-GPU box): launches tests/multi_gpu_plan_check.py under torchrun, one rank per GPU."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_plan_nodes_over_the_library_communicator():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least two GPUs")
    world = 2 if n < 4 else 4
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tests", "multi_gpu_plan_check.py")], capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "MULTI_GPU_PLAN_CHECK" in r.stdout and "ok=True" in r.stdout, r.stdout[-2000:]
