"""The owner-computes exchange on the Keras optimizers at two and three ranks (tests/mgpu_xchg_keras_check.py
through torchrun): ordinary and paired tables, rows that several ranks push in one step, bit for bit against the
Keras oracle."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world,port", [(2, 29561), (3, 29562)])
def test_exchange_keras_optimizers_match_oracle_via_torchrun(world, port):
    """One rank per GPU when the box has enough of them, otherwise every rank as a process on cuda:0."""
    env = dict(os.environ)
    if torch.cuda.device_count() < world:
        env["B200_SHARED_GPU"] = "1"
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                          "--master-addr", "127.0.0.1", "--master-port", str(port),
                          os.path.join(ROOT, "tests", "mgpu_xchg_keras_check.py")],
                         capture_output=True, text=True, timeout=1800, env=env)
    assert out.returncode == 0 and "mgpu_xchg_keras_check ok: world=%d" % world in out.stdout, (
        out.stdout[-3000:] + out.stderr[-6000:])
