"""Learning-rate schedules evaluated by k_push_begin on the owner-computes exchange (torchrun, one rank per GPU;
B200_SHARED_GPU=1 puts every rank on cuda:0 as its own process).

Each rank installs the same schedule on its own view and pushes through b200ps_xchg_push; the owner of a row applies
the lr, Adam alpha and FTRL l2 the SOURCE rank's k_push_begin computed (they travel in the exchange header).  Every
rank begins its push after every rank's previous push ended (the pull before it ends with a barrier), so every rank
reads the shard versions n_pushes * world and evaluates the schedule at x = n_pushes * world - 1, clamped at 0.
The rows -- params and every optimizer slot, of rows one rank pushes and of rows every rank pushes -- equal, bit for
bit, the oracle applying the ranks' pushes in rank order with that x's float32 lr: a one-process run of the same
pushes.  The request's learning_rate, a different value, is ignored.  The schedules change the lr at every push
(ExponentialDecay, InverseTimeDecay) or cross boundaries (PiecewiseConstantDecay)."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticdl_b200 import callbacks as cb  # noqa: E402
from elasticdl_b200._lib import check  # noqa: E402
from oracle import lr_schedule_oracle as orc  # noqa: E402
from tests import mgpu_xchg_paths_check as X  # noqa: E402

CAPS = (1, 3001, 5003)
B = 4096
ROUNDS = ("collide", "disjoint", "collide", "collide", "disjoint", "collide")
CASES = (  # (optimizer of tests/test_gpu_parity.OPTS, device schedule, float64 oracle of x)
    ("sgd", cb.ExponentialDecay(0.2, 1, 0.8), lambda x: orc.exponential(x, 0.2, 1, 0.8)),
    ("adam", cb.InverseTimeDecay(0.002, 2, 0.5), lambda x: orc.inverse_time(x, 0.002, 2, 0.5)),
    ("ftrl_shrink", cb.PiecewiseConstantDecay([2, 6], [0.1, 0.03, 0.01]),
     lambda x: orc.piecewise_constant(x, [2, 6], [0.1, 0.03, 0.01])),
)


def counts(p, g, rnd, world):
    return (1, 1400 - 7 * p, 2300 + 11 * p)[g]


class ScheduledExchange(X.Exchange):
    def push_scheduled(self, lists, rnd, ref, what):
        """X.Exchange.push with push_begin's learning_rate at 0.777 (ignored under the schedule) and the oracle fed
        the schedule's float32 value at x = pushes * world - 1."""
        v = self.pushes * self.world
        assert [s[0] for s in self.group.snapshot()] == [v] * self.world, self.tag("versions before the push")
        lr = float(np.float32(ref(orc.schedule_argument([v]))))
        grads = [[None] * self.G for _ in range(self.world)]
        for p in range(self.world):
            for g in range(self.G):
                rs = np.random.RandomState((rnd * 16 + p) * 64 + g + 7)
                n = len(lists[p][g])
                grads[p][g] = (rs.randn(n, 8).astype(X.F), rs.randn(n, 1).astype(X.F))
        gd, gw = np.zeros((self.G * self.B, 8), X.F), np.zeros((self.G * self.B, 1), X.F)
        for g in range(self.G):
            n = len(lists[self.rank][g])
            gd[g * self.B:g * self.B + n], gw[g * self.B:g * self.B + n] = grads[self.rank][g]
        self.gs_d.copy_(torch.from_numpy(gd))
        self.gs_w.copy_(torch.from_numpy(gw))
        for r in range(self.world):  # push_begin in rank order: shard steps (Adam's alpha) are deterministic
            if r == self.rank:
                self.group.push_begin(0.777, [0] * self.world)
            torch.cuda.synchronize()
            dist.barrier()
        check(self._push())
        self.group.push_end(sync=True)
        self.group.check()
        dist.barrier()
        for p in range(self.world):
            named = []
            for g, (a, b) in enumerate(self.names):
                named += [(a, lists[p][g], grads[p][g][0]), (b, lists[p][g], grads[p][g][1])]
            X.oracle_push(self.servers, named, lr)
        self.pushes += 1
        self.check_state(what + " (lr %r)" % lr)


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    shared = os.environ.get("B200_SHARED_GPU") == "1"
    local = 0 if shared else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    for opt, sched, ref in CASES:
        x = ScheduledExchange(opt, CAPS, B, False, world, rank, local, dev)
        x.group.set_lr_schedule(sched)
        for rnd, kind in enumerate(ROUNDS):
            lists = (X.disjoint_lists(x.caps, rnd, world) if kind == "disjoint"
                     else X.collide_lists(x.caps, counts, rnd, world))
            x.pull(lists[rank])
            x.check_pull(lists, "%s round %d %s pull" % (opt, rnd, kind))
            x.push_scheduled(lists, rnd, ref, "%s round %d %s push" % (opt, rnd, kind))
        x.close()
    if rank == 0:
        print("mgpu_lr_schedule_check ok: world=%d, %d schedules x %d pushes" % (world, len(CASES), len(ROUNDS)))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
