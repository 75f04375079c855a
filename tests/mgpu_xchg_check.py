"""Owner-computes exchange (csrc/ps_exchange.cuh) set-up (torchrun, one rank per GPU).  Checks: xchg_create
refuses hashed, dense and raw tables and too many groups, and a refused create leaves the valid one possible; a
DeepFM engine with too many groups takes the direct path; no wait timed out.  The exchange's data paths -- pull,
push, created rows, out-of-range ids, every optimizer, paired tables -- are checked bit for bit against the oracle
by tests/mgpu_xchg_paths_check.py, and the DeepFM step bench.py times on it, step by step, by
tests/mgpu_bench_step_check.py."""
import ctypes
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticdl_b200 import _lib  # noqa: E402
from elasticdl_b200._lib import check  # noqa: E402
from elasticdl_b200.ps import PSGroup  # noqa: E402

ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    # B200_SHARED_GPU=1: every rank is a process on cuda:0 (the shards are still separate allocations mapped
    # across PROCESSES with CUDA IPC, the kernels of the ranks time-slice the one device) and the host-side
    # plumbing runs over gloo -- NCCL refuses two ranks on one device.  Lets a 1-GPU box run this check.
    shared = os.environ.get("B200_SHARED_GPU") == "1"
    local = 0 if shared else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    group = PSGroup(world, *ADAM, device=local, local_shards=[rank])
    rows = [7, 3000, 400000]
    G, B, D = len(rows), 4096, 8
    deep = [group.register_table("d%d" % g, D, "zero", r) for g, r in enumerate(rows)]
    wide = [group.register_table("w%d" % g, 1, "zero", r) for g, r in enumerate(rows)]
    hashed_id = group.register_table("hashed", D, "zero", expected_rows=64)
    dense_id = group.register_dense("dense", (16, D), 0)
    raw_id = check(group.lib.b200ps_raw_register(group._h, b"raw", 64))
    group.commit()

    def create(dt, wt):
        return group.lib.b200ps_xchg_create(group._h, len(dt), B, (ctypes.c_int32 * len(dt))(*dt),
                                            (ctypes.c_int32 * len(wt))(*wt))

    # the exchange serves direct-indexed striped tables only, and at most MAX_SEGS / 2 pairs; a refused
    # create leaves no exchange behind, so the valid one below still succeeds
    kx = _lib.MAX_SEGS // 2 + 1
    for dt, wt in (([hashed_id] + deep[1:], wide), ([dense_id] + deep[1:], wide), (deep, [raw_id] + wide[1:]),
                   ((deep * kx)[:kx], (wide * kx)[:kx])):
        assert create(dt, wt) == _lib.EINVAL, (dt, wt, group.lib.b200ps_last_error())
    group.xchg_create(G, B, deep, wide)
    group.check()
    dist.barrier()
    # ---- more id groups than the exchange moves: the engine takes the direct path ------------------
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    g3 = PSGroup(world, *ADAM, device=local, local_shards=[rank])
    assert DeepFMPSEngine(g3, 64, group_rows=[16] * kx).exchange == "direct"
    dist.barrier()
    if rank == 0:
        print("mgpu_xchg_check ok: world=%d exchange created" % world)
    g3.close()
    group.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
