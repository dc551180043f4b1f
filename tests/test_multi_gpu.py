"""The library's own NCCL path on real GPUs (needs >= 2 visible devices; skipped on a single-GPU box): launches each
tests/multi_gpu_*_check.py under torchrun, one rank per GPU, and reads its verdict line."""
import os
import subprocess
import sys

import pytest

from tests.ranks import free_port

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("script, tag", [
    ("multi_gpu_check.py", "MULTI_GPU_CHECK"),                              # sum by, min / max / stddev / stdvar merges
    ("multi_gpu_topk_check.py", "MULTI_GPU_TOPK_CHECK"),
    ("multi_gpu_quantile_check.py", "MULTI_GPU_QUANTILE_CHECK"),
    ("multi_gpu_count_values_check.py", "MULTI_GPU_COUNT_VALUES_CHECK"),
    ("multi_gpu_sort_check.py", "MULTI_GPU_SORT_CHECK"),
    ("multi_gpu_plan_check.py", "MULTI_GPU_PLAN_CHECK"),
])
def test_sharded_operators_over_the_library_communicator(script, tag):
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs at least two GPUs")
    world = 2 if n < 4 else 4
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
                        "--master-addr", "127.0.0.1", "--master-port", str(free_port()),
                        os.path.join(ROOT, "tests", script)], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert tag in r.stdout and "ok=True" in r.stdout, r.stdout[-2000:]
