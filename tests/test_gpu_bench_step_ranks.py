"""The DeepFM step bench.py --gpus N times, at two and three ranks (tests/mgpu_bench_step_check.py through torchrun):
every step of its feeds on the owner-computes exchange checked against the oracle's dedup, the rows the step
started from, the float64 tower reference and the oracle's Adam of every rank's push; the dense parameters, which
the ranks push lock-free, against the interleavings of the ranks' updates."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world,port", [(2, 29571), (3, 29572)])
def test_bench_step_matches_references_at_n_ranks_via_torchrun(world, port):
    """One rank per GPU when the box has enough of them, otherwise every rank as a process on cuda:0
    (B200_SHARED_GPU=1: CUDA IPC between the processes, gloo for the host plumbing)."""
    env = dict(os.environ)
    if torch.cuda.device_count() < world:
        env["B200_SHARED_GPU"] = "1"
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                          "--master-addr", "127.0.0.1", "--master-port", str(port),
                          os.path.join(ROOT, "tests", "mgpu_bench_step_check.py")],
                         capture_output=True, text=True, timeout=1800, env=env)
    assert out.returncode == 0 and "mgpu_bench_step_check ok: world=%d" % world in out.stdout, (
        out.stdout[-3000:] + out.stderr[-6000:])
    print(out.stdout[-4000:])
