"""Multi-GPU numeric check of the data path's only collective (VERDICT "What's weak" 5): on a box with >= 2 GPUs, the NCCL
all-reduced gradient buffer of a sharded view batch equals the single-rank sum of the same views (tests/dist_nccl_check.py,
one process per GPU under torch.distributed.run).  Skipped on a single-GPU box; the host-side logic has its own world-size-2
gloo test on CPU (tests/test_dist_gloo.py).  `python -m pytest tests/test_gpu_dist.py -m gpu -s` on a
multi-GPU machine runs it."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("nvls", ["0", "1"], ids=["nccl", "own_nvls_kernel_if_available"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_nccl_all_reduce_equals_single_rank_sum(cuda, world, nvls):
    import torch
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs, this box has {torch.cuda.device_count()}")
    port = 29500 + world + (20 if nvls == "1" else 0)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tests", "dist_nccl_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=ROOT, env={**os.environ, "LGS_NVLS": nvls})
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("NCCL_CHECK ")]
    assert r.returncode == 0 and lines, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    out = json.loads(lines[-1][len("NCCL_CHECK "):])
    print(json.dumps(out))
    assert out["ok"] and out["world"] == world
