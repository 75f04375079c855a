"""The owner-computes exchange's data paths (csrc/ps_exchange.cuh) against the oracle, bit for bit, at any world
size (torchrun, one rank per GPU; B200_SHARED_GPU=1 puts every rank on cuda:0 as its own process).

For every optimizer configuration of tests/test_gpu_parity.OPTS, once over ordinary tables and once over paired
records (b200ps_table_register_pair), a fresh group exchanges G = 4 (deep, wide) pairs of 1 row (every rank asks
for id 0, only shard 0 owns it), 3001 rows (not a multiple of N) and 400009 rows (up to B = 200003 live ids: the
post, serve, unscatter and apply grids loop), and a group that is empty on one rank per round:
* xchg_pull equals pull_rows and the oracle, deep and wide; bet rows past a group's n_unique keep their sentinel;
* after the exchange pulls, the created rows of every table on every shard equal the oracle's (the union of the
  ids every rank pulled), read before any direct pull creates rows;
* xchg_push on rank-disjoint rows (routing), then on rows every rank pushes -- the hottest first, the 1-row
  table's id 0 -- and rows of each rank's own: params and every optimizer slot equal the oracle applying the
  ranks' pushes in rank order;
* a push updates the rows of the pull just before it, and a push without a pull returns B200PS_ESTATE;
* an id >= rows * N, and 2**32 + 5 (which must not alias row 5), come back as zero rows and make the REQUESTING
  rank's check() raise B200PS_ERANGE, no other rank's; the exchange then serves a valid pull.
A create that mixes paired and ordinary tables is refused, and one run at G = MAX_SEGS / 2 with a small B checks the
largest per-group prefix of k_x_post.  No case lets a rank skip a step: the exchange's timeouts stay untested."""
import ctypes
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticdl_b200 import _lib  # noqa: E402
from elasticdl_b200._lib import check  # noqa: E402
from elasticdl_b200.ps import PSGroup  # noqa: E402
from oracle import ps_oracle as O  # noqa: E402
from tests.test_gpu_parity import OPTS  # noqa: E402

F = np.float32
SENTINEL = -7.0
PAD_ID = 1 << 40  # uniq entries past n_unique: outside every table, so reading one would raise ERANGE
CAPS = (1, 3001, 400_009, 5003)
B = 200_003  # not a multiple of 4 or 256; the 400009-row group reaches exactly B live ids
ROUNDS = (("disjoint", 0.0), ("collide", 0.0), ("collide", 0.05), ("decoy", 0.0), ("collide", 0.0))


def main_counts(p, g, rnd, world):
    """Live ids of rank p in group g: exactly B in the big group on one rank, none in the last group on another."""
    if g == 0:
        return 1
    if g == 1:
        return 2999 - 2 * p
    if g == 2:
        return B if p == rnd % world else B - 1000 * (p + 1) - 17
    return 0 if p == (rnd + 1) % world else 1237 + p


def oracle_rows(servers, name, ids, slot=0):
    """Params (slot 0) or optimizer slot `slot` of `ids` from the oracle shards (id % N); creates missing rows, as a
    pull from the PS does."""
    n = len(servers)
    out = np.empty((len(ids), servers[0].tables[name].dim), dtype=F)
    for s in servers:
        m = ids % n == s.id
        t = s.tables[name] if slot == 0 else s.opt.table_slots[s.opt.slot_names[slot - 1]][name]
        out[m] = t.get(ids[m])
    return out


def oracle_push(servers, named, lr):
    """OraclePSClient.push_gradients for lists of unique ids [(name, ids, grads)], routed with vector masks: every
    shard takes one push, an empty one too (ps_client.py:190-287)."""
    n = len(servers)
    for s in servers:
        sparse = {}
        for name, ids, g in named:
            m = ids % n == s.id
            if m.any():
                sparse[name] = (ids[m], g[m])
        ok, _ = s.push_gradients({}, sparse, lr, 0)
        assert ok


def collide_lists(caps, counts, rnd, world):
    """lists[p][g]: the same head on every rank (0, 5, cap - 1, then a shared random prefix: the hot ids of a zipf
    batch, first in first-occurrence order), then ids of rank p's own draw (which may meet other ranks' draws)."""
    lists = [[None] * len(caps) for _ in range(world)]
    for g, c in enumerate(caps):
        head = np.array(list(dict.fromkeys(i for i in (0, 5, c - 1) if i < c)), dtype=np.int64)
        rest = np.random.RandomState(1000 * rnd + g).permutation(c).astype(np.int64)
        perm = np.concatenate([head, rest[~np.isin(rest, head)]])
        n = [counts(p, g, rnd, world) for p in range(world)]
        shared = [min(k, k // 2 + 1) for k in n]
        for p in range(world):
            own = np.random.RandomState((rnd * 16 + p) * 64 + g).permutation(perm[max(shared):])[:n[p] - shared[p]]
            lists[p][g] = np.concatenate([perm[:shared[p]], own]).astype(np.int64)
    return lists


def disjoint_lists(caps, rnd, world):
    """lists[p][g]: id = q*N*N + p*N + owner, so no two ranks push the same row."""
    lists = [[None] * len(caps) for _ in range(world)]
    for g, c in enumerate(caps):
        k = min(1500, max(c // (world * world), 1))
        q = np.random.RandomState(5 * rnd + g).permutation(max(c // (world * world), 1))[:k] * world * world
        for p in range(world):
            ids = q + p * world + np.random.RandomState(1000 * rnd + 64 * p + g).randint(0, world, size=k)
            lists[p][g] = ids[ids < c].astype(np.int64)
    return lists


class Exchange:
    """One PSGroup whose exchange moves G (deep, wide) table pairs, and the oracle shards that mirror it."""

    def __init__(self, opt, caps, batch, paired, world, rank, local, dev):
        ot, oa = OPTS[opt]
        self.opt, self.paired = opt, paired
        self.world, self.rank, self.dev = world, rank, dev
        self.caps, self.B, self.G = list(caps), batch, len(caps)
        self.group = grp = PSGroup(world, ot, oa, device=local, local_shards=[rank])
        self.names = [("d%d" % g, "w%d" % g) for g in range(self.G)]
        if paired:
            tids = [grp.register_pair(a, b, c) for (a, b), c in zip(self.names, caps)]
            deep, wide = [t[0] for t in tids], [t[1] for t in tids]
            plain_d, plain_w = grp.register_table("xd", 8, "zero", 16), grp.register_table("xw", 1, "zero", 16)
        else:
            deep = [grp.register_table(a, 8, "zero", c) for (a, _), c in zip(self.names, caps)]
            wide = [grp.register_table(b, 1, "zero", c) for (_, b), c in zip(self.names, caps)]
        grp.commit()
        self.lib, self.h = grp.lib, grp._h
        if paired:  # a paired record's sections are 12 floats, an ordinary record's are not: one layout per family
            for dt, wt in (([plain_d] + deep[1:], wide), (deep, [plain_w] + wide[1:])):
                rc = self.lib.b200ps_xchg_create(self.h, self.G, batch, (ctypes.c_int32 * self.G)(*dt),
                                                 (ctypes.c_int32 * self.G)(*wt))
                assert rc == _lib.EINVAL, (rc, self.lib.b200ps_last_error())
        grp.xchg_create(self.G, batch, deep, wide)
        self.servers = [O.OracleServer(i, ot, oa, num_ps=world) for i in range(world)]
        for s in self.servers:
            s.push_embedding_table_infos([O.EmbeddingTableInfo(n, d, "zero", 1) for a, b in self.names
                                          for n, d in ((a, 8), (b, 1))])
        self.n_slots = len(self.servers[0].opt.slot_names)
        f32 = dict(dtype=torch.float32, device=dev)
        self.uniq = torch.empty(self.G * batch, dtype=torch.int64, device=dev)
        self.n_dev = torch.empty(self.G, dtype=torch.int32, device=dev)
        self.bet_d, self.bet_w = torch.empty((self.G * batch, 8), **f32), torch.empty((self.G * batch, 1), **f32)
        self.gs_d, self.gs_w = torch.zeros((self.G * batch, 8), **f32), torch.zeros((self.G * batch, 1), **f32)
        self.pushes = 0
        assert self._push() == _lib.ESTATE  # no pull yet

    def tag(self, what):
        return "%s %s world=%d rank=%d: %s" % (self.opt, "paired" if self.paired else "plain", self.world,
                                                self.rank, what)

    def _push(self):
        return self.lib.b200ps_xchg_push(self.h, self.gs_d.data_ptr(), self.gs_w.data_ptr(), self.group._stream())

    def rows(self, bet, g, n):
        return bet[g * self.B:g * self.B + n].cpu().numpy()

    # ---------------------------------------------------------------- pull
    def pull(self, mine):
        """xchg_pull of this rank's lists; bet is filled with a sentinel first.  Returns once every rank's pull
        (and so every owner's serve of it) has finished."""
        u = np.full(self.G * self.B, PAD_ID, dtype=np.int64)
        for g, ids in enumerate(mine):
            u[g * self.B:g * self.B + len(ids)] = ids
        self.uniq.copy_(torch.from_numpy(u))
        self.n_dev.copy_(torch.tensor([len(ids) for ids in mine], dtype=torch.int32))
        self.bet_d.fill_(SENTINEL)
        self.bet_w.fill_(SENTINEL)
        check(self.lib.b200ps_xchg_pull(self.h, self.uniq.data_ptr(), self.n_dev.data_ptr(), self.bet_d.data_ptr(),
                                        self.bet_w.data_ptr(), self.group._stream()))
        torch.cuda.synchronize()
        dist.barrier()

    def check_pull(self, lists, what):
        """After pull(lists[rank]) on every rank: bet vs the oracle, rows past n_unique untouched, created rows of
        every table on every shard vs the oracle's, then bet vs the direct pull."""
        self.group.check()
        mine = lists[self.rank]
        for p in range(self.world):  # the oracle serves every rank's pull, creating the rows it creates
            for g, (a, b) in enumerate(self.names):
                for name, bet in ((a, self.bet_d), (b, self.bet_w)):
                    want = oracle_rows(self.servers, name, lists[p][g])
                    if p != self.rank:
                        continue
                    got = self.rows(bet, g, self.B)
                    n = len(mine[g])
                    assert np.array_equal(got[:n], want), self.tag("%s: %s rows differ from the oracle" % (what, name))
                    assert (got[n:] == F(SENTINEL)).all(), self.tag("%s: %s rows past n_unique written" % (what, name))
        for a, b in self.names:
            for name in (a, b):
                for s in range(self.world):
                    got = np.sort(self.group.table_ids(name, s).cpu().numpy())
                    want = np.sort(self.servers[s].tables[name].keys())
                    assert np.array_equal(got, want), self.tag("%s: created rows of %s on shard %d: %d, oracle %d" % (
                        what, name, s, len(got), len(want)))
        dist.barrier()  # every rank has read the created rows before a direct pull creates any
        for g, (a, b) in enumerate(self.names):
            n = len(mine[g])
            if n == 0:
                continue
            ids = self.uniq[g * self.B:g * self.B + n]
            want_d, want_w = self.group.pull_rows([(a, ids), (b, ids)])
            assert torch.equal(self.bet_d[g * self.B:g * self.B + n], want_d), self.tag("%s: %s != direct pull" % (what, a))
            assert torch.equal(self.bet_w[g * self.B:g * self.B + n], want_w), self.tag("%s: %s != direct pull" % (what, b))
        dist.barrier()

    # ---------------------------------------------------------------- push
    def push(self, lists, rnd, lr, what):
        """Every rank pushes gradients for the rows of its last pull, push_begin in rank order (so shard steps and
        Adam's alpha are deterministic); the oracle applies the pushes in rank order 0..N-1."""
        grads = [[None] * self.G for _ in range(self.world)]
        for p in range(self.world):
            for g in range(self.G):
                rs = np.random.RandomState((rnd * 16 + p) * 64 + g + 7)
                n = len(lists[p][g])
                grads[p][g] = (rs.randn(n, 8).astype(F), rs.randn(n, 1).astype(F))
        gd, gw = np.zeros((self.G * self.B, 8), F), np.zeros((self.G * self.B, 1), F)
        for g in range(self.G):
            n = len(lists[self.rank][g])
            gd[g * self.B:g * self.B + n], gw[g * self.B:g * self.B + n] = grads[self.rank][g]
        self.gs_d.copy_(torch.from_numpy(gd))
        self.gs_w.copy_(torch.from_numpy(gw))
        for r in range(self.world):
            if r == self.rank:
                self.group.push_begin(lr, [0] * self.world)
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
            oracle_push(self.servers, named, lr)
        self.pushes += 1
        self.check_state(what)

    def check_state(self, what):
        """Params and every optimizer slot of every created row, deep and wide, equal the oracle's."""
        for a, b in self.names:
            ids = np.sort(np.concatenate([s.tables[a].keys() for s in self.servers]))
            if len(ids) == 0:
                continue
            for name in (a, b):
                for k in range(self.n_slots + 1):
                    got = self.group.slot_rows(name, ids, k).cpu().numpy()
                    want = oracle_rows(self.servers, name, ids, k)
                    if not np.array_equal(got, want):
                        bad = np.nonzero((got != want).any(axis=1))[0]
                        raise AssertionError(self.tag("%s: %s slot %d differs from the oracle on %d of %d rows, first "
                                                      "id %d: %s vs %s" % (what, name, k, len(bad), len(ids),
                                                                           ids[bad[0]], got[bad[0]], want[bad[0]])))

    # ---------------------------------------------------------------- the cases
    def run_rounds(self, counts, rounds):
        for rnd, (kind, lr) in enumerate(rounds):
            lists = (disjoint_lists(self.caps, rnd, self.world) if kind == "disjoint"
                     else collide_lists(self.caps, counts, rnd, self.world))
            if kind == "decoy":  # two pulls, one push: the push updates the rows of the second
                decoy = collide_lists(self.caps, counts, rnd + 100, self.world)
                self.pull(decoy[self.rank])
                self.check_pull(decoy, "round %d decoy pull" % rnd)
            self.pull(lists[self.rank])
            self.check_pull(lists, "round %d %s pull" % (rnd, kind))
            self.push(lists, rnd, lr, "round %d %s push" % (rnd, kind))
        assert self._push() == _lib.ESTATE, self.tag("a second push after one pull")
        state = self.group.snapshot()
        assert [s[:2] for s in state] == [(self.pushes * self.world,) * 2] * self.world, self.tag(state)

    def range_checks(self):
        """Out-of-range ids come back as zero rows, raise in the requester's check() only, and leave the exchange
        working.  Group 1 (3001 rows): ids 0, 5 and 3000 were pushed, so row 5 is not zero."""
        g, (a, b) = 1, self.names[1]
        valid = np.array([0, 5, self.caps[g] - 1], dtype=np.int64)
        assert (oracle_rows(self.servers, a, valid[1:2]) != 0).any()
        rows = -(-self.caps[g] // self.world)
        hi = (1 << 32) + 5
        for bad, who in ((rows * self.world, self.world - 1), (hi, (hi % self.world + 1) % self.world)):
            mine = [np.zeros(0, dtype=np.int64) for _ in range(self.G)]
            mine[g] = np.insert(valid, 1, bad) if self.rank == who else valid
            self.pull(mine)
            try:
                self.group.check()
                raised = False
            except _lib.PSRangeError:
                raised = True
            assert raised == (self.rank == who), self.tag("id %d asked by rank %d: check() raised %s" % (bad, who, raised))
            got_d, got_w = self.rows(self.bet_d, g, len(mine[g])), self.rows(self.bet_w, g, len(mine[g]))
            if self.rank == who:
                assert (got_d[1] == 0).all() and (got_w[1] == 0).all(), self.tag("id %d: %s %s" % (bad, got_d[1], got_w[1]))
                got_d, got_w = np.delete(got_d, 1, axis=0), np.delete(got_w, 1, axis=0)
            assert np.array_equal(got_d, oracle_rows(self.servers, a, valid)), self.tag("id %d: deep rows" % bad)
            assert np.array_equal(got_w, oracle_rows(self.servers, b, valid)), self.tag("id %d: wide rows" % bad)
            dist.barrier()
        lists = collide_lists(self.caps, main_counts, 50, self.world)
        self.pull(lists[self.rank])
        self.check_pull(lists, "valid pull after the out-of-range ones")

    def close(self):
        torch.cuda.synchronize()
        dist.barrier()  # no peer still reads this rank's shards
        self.group.close()


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    # B200_SHARED_GPU=1: every rank is a process on cuda:0 (see tests/mgpu_xchg_check.py)
    shared = os.environ.get("B200_SHARED_GPU") == "1"
    local = 0 if shared else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    for opt in OPTS:
        for paired in (False, True):
            x = Exchange(opt, CAPS, B, paired, world, rank, local, dev)
            x.run_rounds(main_counts, ROUNDS)
            x.range_checks()
            x.close()
    # the most pairs one exchange moves, a few ids each: k_x_post's largest group prefix, counts 0..B
    kx, small_b = _lib.MAX_SEGS // 2, 5
    x = Exchange("amsgrad", [3 + 5 * g for g in range(kx)], small_b, False, world, rank, local, dev)
    x.run_rounds(lambda p, g, rnd, w: min(3 + 5 * g, (g + p + rnd) % (small_b + 1)), (("collide", 0.0), ("collide", 0.05)))
    x.close()
    if rank == 0:
        print("mgpu_xchg_paths_check ok: world=%d, %d optimizer configurations x (plain, paired) + G=%d" % (
            world, len(OPTS), kx))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
