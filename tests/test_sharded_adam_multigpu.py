"""-m gpu, needs >= 2 GPUs (skipped on the single-GPU test box; run with `gpurun --gpus 2`): ShardedFlatAdam with the fused
reduction + Adam + broadcast kernel (nvls / p2p transports) and the NCCL fallback against torch.optim.Adam on the
rank-averaged gradients -- scripts/check_sharded_adam.py under torchrun.  Prints which transports ran; fails when p2p
did not run although every pair of GPUs reports peer access (an unavailable nvls is reported, not failed)."""
import itertools
import json
import os
import subprocess
import sys

import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs on one box")
def test_sharded_adam_transports_match_torch_adam():
    n = min(torch.cuda.device_count(), 4)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={n}",
                        "--master-addr", "127.0.0.1", "--master-port", "29533", os.path.join(ROOT, "scripts", "check_sharded_adam.py")],
                       capture_output=True, text=True, timeout=900)
    sys.stdout.write(r.stdout[-4000:]); sys.stderr.write(r.stderr[-2000:])
    assert r.returncode == 0
    assert r.stdout.count("PASS") == n
    lines = [json.loads(x[len("TRANSPORT "):]) for x in r.stdout.splitlines() if x.startswith("TRANSPORT ")]
    assert len(lines) == 5 * n, f"expected 5 TRANSPORT lines per rank, got {len(lines)}"
    for x in lines:
        if x["rank"] == 0:
            label = x["case"] + (" + early region" if x["early"] else "")
            print(f"[{label}] " + (f"ran as {x['transport']}" if x["ran"] else f"did not run: {x['reason']}"))
    assert all(x["ran"] for x in lines if x["case"] == "nccl")
    if all(torch.cuda.can_device_access_peer(a, b) for a, b in itertools.permutations(range(n), 2)):
        missing = [x for x in lines if x["case"] == "p2p" and not x["ran"]]
        assert not missing, f"p2p did not run although every pair of the {n} GPUs has peer access: {missing[0]['reason']}"
