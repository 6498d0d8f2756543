"""-m gpu, needs >= 2 GPUs (skipped on a single-GPU box): FusedSparseAdam's data-parallel step with real NCCL --
scripts/check_sparse_ddp.py under torch.distributed.run: bit-identical replicas, and a single-process step on the whole
batch as the reference, both judged against fp64."""
import os
import subprocess
import sys

import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs on one box")
def test_sparse_data_parallel_step_with_nccl():
    n = min(torch.cuda.device_count(), 4)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
                        "--master-addr", "127.0.0.1", "--master-port", "29537",
                        os.path.join(ROOT, "scripts", "check_sparse_ddp.py")],
                       capture_output=True, text=True, timeout=900)
    sys.stdout.write(r.stdout[-4000:]); sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0
    assert r.stdout.count("PASS") == n
