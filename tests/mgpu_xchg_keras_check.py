"""The owner-computes exchange (csrc/ps_exchange.cuh) on the Keras optimizers (RMSprop and its three variants,
Adadelta, Adamax, Nadam), bit for bit against oracle/keras_optim_oracle.py, at any world size (torchrun, one rank per
GPU; B200_SHARED_GPU=1 puts every rank on cuda:0 as its own process).

It runs tests/mgpu_xchg_paths_check.py's Exchange -- pulls, pushes of rank-disjoint rows, of rows every rank pushes
and of each rank's own rows, a decoy pull, an explicit lr -- over ordinary tables and over paired records, with the
Keras optimizer table in place of tests/test_gpu_parity.OPTS and the Keras oracle shards in place of the Go ones.
k_x_apply<OPT> applies the per-push words the pusher's k_push_begin wrote for the owner shard (Nadam's folded
scalars included), so every shard's step and every slot are checked after every push.  The largest group is 40009
rows with up to 20003 live ids, enough for several blocks per grid; the grid loops are checked by the Go optimizers'
run of the same class."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import keras_optim_oracle as K  # noqa: E402
from oracle import ps_oracle as O  # noqa: E402
from tests import mgpu_xchg_paths_check as X  # noqa: E402
from tests.test_gpu_keras_optimizers import KERAS_OPTS  # noqa: E402


class _KerasOracle:
    """ps_oracle with OracleServer swapped for the Keras oracle shard (everything else is ps_oracle's)."""

    @staticmethod
    def OracleServer(ps_id, opt_type, opt_args, num_ps=1):
        return K.KerasOracleServer(ps_id, opt_type, opt_args, num_ps=num_ps)

    def __getattr__(self, name):
        return getattr(O, name)


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
    # this process only: the Exchange helper reads its optimizer table, oracle module and batch size from its module
    X.OPTS, X.O, X.B = KERAS_OPTS, _KerasOracle(), 20_003
    caps = (1, 3001, 40_009, 5003)
    for opt in KERAS_OPTS:
        for paired in (False, True):
            x = X.Exchange(opt, caps, X.B, paired, world, rank, local, dev)
            assert x.n_slots == len(K.KINDS[opt][1]), x.tag("slots")
            x.run_rounds(X.main_counts, X.ROUNDS)
            x.close()
    if rank == 0:
        print("mgpu_xchg_keras_check ok: world=%d, %d optimizer configurations x (plain, paired)" % (world, len(KERAS_OPTS)))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
