"""The sharded classic-Paxos fallback across GPUs: one process per GPU under torchrun, receivers and acceptors sharded by
ring-0 range, a split vote with no fast quorum recovered by rapid_px_phase{1,2}b_from_acceptor_shards over NCCL.  Needs >= 2
GPUs; on a 1-GPU machine it is skipped.  See tests/nccl_fallback_worker.py for what every rank checks (the same cval, trigger
index and decision on every rank as a single-handle round over all acceptors)."""
import os
import socket
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _gpus():
    import torch
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


@pytest.mark.parametrize("world", [2, 4])
def test_sharded_classic_round_matches_single_handle(world):
    have = _gpus()
    if have < world:
        pytest.skip("needs %d GPUs (this box has %d)" % (world, have))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), os.path.join(ROOT, "tests", "nccl_fallback_worker.py"), "20000"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert r.returncode == 0, (r.stdout[-3000:] + "\n" + r.stderr[-6000:])
    assert "nccl fallback worker ok" in r.stdout
