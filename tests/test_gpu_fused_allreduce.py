"""DistributedOptimizer(fused=True) against the torch optimizer it wraps at two and three ranks
(tests/mgpu_fused_allreduce_check.py through torchrun): every step of SGD, momentum, Nesterov, Adam and AMSGrad
within the fp32 bound of oracle/torch_optim_oracle.py, at the layout edges of the flat bucket, in every gradient
scaling mode, under lr schedules and in-place parameter edits; and the refusals."""
import os
import subprocess
import sys

import pytest
import torch
import torch.distributed as dist

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("world,port", [(2, 29555), (3, 29556)])
def test_fused_allreduce_matches_torch_optimizer_via_torchrun(world, port):
    """One rank per GPU when the box has enough of them, otherwise every rank as a process on cuda:0
    (B200_SHARED_GPU=1: CUDA IPC between the processes, gloo for the host plumbing)."""
    env = dict(os.environ)
    if torch.cuda.device_count() < world:
        env["B200_SHARED_GPU"] = "1"
    out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                          "--master-addr", "127.0.0.1", "--master-port", str(port),
                          os.path.join(ROOT, "tests", "mgpu_fused_allreduce_check.py")],
                         capture_output=True, text=True, timeout=1800, env=env)
    assert out.returncode == 0 and "mgpu_fused_allreduce_check ok: world=%d" % world in out.stdout, (
        out.stdout[-8000:] + out.stderr[-4000:])


def test_fused_refuses_a_one_rank_group(tmp_path):
    """fused=True needs world_size > 1 (there is nothing to reduce); other truthy values fall back silently."""
    from elasticdl_b200.elasticai_api.pytorch.optimizer import DistributedOptimizer

    dist.init_process_group("gloo", store=dist.FileStore(str(tmp_path / "store"), 1), rank=0, world_size=1)
    try:
        p = torch.nn.Parameter(torch.randn(8, device="cuda"))
        with pytest.raises(ValueError):
            DistributedOptimizer(torch.optim.SGD([p], lr=0.1), fused=True)
        opt = DistributedOptimizer(torch.optim.SGD([p], lr=0.1), fused=1)
        assert opt._ps is None
    finally:
        dist.destroy_process_group()
