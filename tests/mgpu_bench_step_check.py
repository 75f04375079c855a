"""The DeepFM step bench.py --gpus N times, checked step by step at N ranks (torchrun, one rank per GPU;
B200_SHARED_GPU=1 puts every rank on cuda:0 as its own process, gloo carrying the host plumbing).

Every rank builds what bench.py builds -- PSGroup(N, "Adam", ADAM_ARGS, local_shards=[rank]) and
DeepFMPSEngine(group, B, id_transport=...): the tile tower on rows the owner-computes exchange pulls
(csrc/ps_exchange.cuh) -- and trains on bench.py's batches (seeds 1234 + p + 1000 * rank) through one of its feeds:
the two lookahead graphs on device buffers (the headline), the lookahead host feeder (e2e), capture + step_graph
(--lookahead off) or eager step().  Each leg runs three steps on a fresh group, and after every step t each rank
checks
  1. its plan's dedup against the oracle's first-occurrence dedup, exactly (on the lookahead feeds also the next
     batch's dedup, which ran beside the push);
  2. the rows the exchange handed the tower (bet_w / bet_d) against the pre-step rows read through the direct
     path, bit for bit: every pull of a step is served before any push of that step is applied;
  3. the tower's loss, logits, gradients and per-row sums against the float64 reference on those rows and on the
     dense parameters the step pulled (oracle/tower_oracle.py bound; the batch is conditioned away from ReLU kinks
     against the pre-step state);
  4. the param / m / v of every row of its own shard that any rank pushed, and of a fixed sample of its other
     rows, bit for bit against the oracle's Adam applied to every rank's pushed gradients in rank order 0..N-1.
     The ranks' push_begin calls race for the shard's step counter, so the steps (t-1)N+1 .. tN are assigned to
     the ranks in an order nothing controls; the shard must match under one assignment for all its tables;
  5. the dense parameters: every rank pushes them lock-free into the owner's slab, as the reference's
     PushGradients does (DESIGN.md section 7, "Direct").  At N = 2 every element of a parameter and its two
     slots must be one that an interleaving of the two ranks' element-wise Adam updates produces; the elements
     where one update was lost or the two tore are counted and printed.  At N = 3 they must be finite;
  6. the shard counters (version = step = tN on every shard), the engine's step count and loss ring, and that
     group.check() raises nothing.
A peer's dense push of the same step may land before this rank's pull_dense; if the dense parameters the step
pulled are not the pre-step ones and a sample then lies within the kink margin, that rank-step's tower comparison
is skipped and printed (a leg needs at least one compared step)."""
import itertools
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import ADAM_ARGS  # noqa: E402
from oracle import ps_oracle as O  # noqa: E402
from oracle import tower_oracle as T  # noqa: E402
from tests.test_gpu_engine_bench_path import (BETA1, BETA2, EPS, FULL_SCAN_ROWS, LR, SAMPLE_ROWS, _check_dedup,  # noqa: E402
                                              _condition, _dense, _oracle_dedup, _plan_dedup)

STEPS = 3
FAMS = ("wide", "deep")


def _gather(obj):
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, obj)
    return out


def _sync():
    torch.cuda.synchronize()
    dist.barrier()


def _slots(group, name, ids):
    """(param, m, v) of rows `ids` of table `name` through slot_rows, numpy float32 [len(ids), dim]."""
    t = torch.from_numpy(np.ascontiguousarray(ids, dtype=np.int64))
    return tuple(group.slot_rows(name, t, k).cpu().numpy() for k in range(3))


def _adam(g, p, m, v, step):
    """The oracle's Adam (step `step`) on copies of p / m / v."""
    p, m, v = p.copy(), m.copy(), v.copy()
    O.np_adam(np.ascontiguousarray(g, dtype=np.float32), p, m, v, LR, step, BETA1, BETA2, EPS)
    return p, m, v


class Leg:
    def __init__(self, world, rank, dev, B, transport, feed, label):
        from elasticdl_b200.ps import PSGroup
        from elasticdl_b200.workloads.deepfm import GROUP_ROWS, DeepFMPSEngine

        self.world, self.rank, self.dev, self.feed, self.label = world, rank, dev, feed, label
        self.group = PSGroup(world, "Adam", ADAM_ARGS, device=dev.index, local_shards=[rank])
        self.eng = eng = DeepFMPSEngine(self.group, B, id_transport=transport)
        assert (eng.exchange, eng.row_source, eng.tower_kind) == ("owner", "pull", "tile"), (
            eng.exchange, eng.row_source, eng.tower_kind)
        self.rows = GROUP_ROWS
        rng = np.random.RandomState(11)
        sample = [np.arange(r) if r <= FULL_SCAN_ROWS else np.sort(rng.choice(r, SAMPLE_ROWS, replace=False))
                  for r in self.rows]
        self.sample = [s[s % world == rank] for s in sample]  # the sampled rows of this rank's shard
        self.compared = 0  # steps whose tower outputs were compared with the reference
        self.races = []  # per step: dense elements with a lost or torn update (N = 2)

    def tables(self):
        eng = self.eng
        return [(n, g, "wide") for g, n in enumerate(eng.wide_names)] + [(n, g, "deep") for g, n in enumerate(eng.deep_names)]

    # ------------------------------------------------------------------ before a step
    def pre_state(self, ids):
        """What step t starts from, read after every rank finished step t - 1: every rank's oracle dedup, the rows of
        this rank's batch through the direct path, param / m / v of the rows of this rank's shard that any rank's
        batch holds plus the sample, the dense parameters and their slots."""
        group, eng = self.group, self.eng
        dedup = _oracle_dedup(ids)
        all_uniq = _gather([u for u, _ in dedup])
        batch_rows = group.pull_rows([(n, torch.from_numpy(dedup[g][0])) for n, g, _ in self.tables()])
        batch_rows = {n: r.cpu().numpy() for (n, _, _), r in zip(self.tables(), batch_rows)}
        own = []
        for g in range(eng.G):
            u = np.unique(np.concatenate([au[g] for au in all_uniq] + [self.sample[g]]))
            own.append(u[u % self.world == self.rank])
        own_state = {n: _slots(group, n, own[g]) if len(own[g]) else None for n, g, _ in self.tables()}
        dense = _dense(group, eng)
        return {"dedup": dedup, "batch_rows": batch_rows, "own": own, "own_state": own_state, "dense": dense,
                "flat": self._flat_of(dense)}

    def _flat_of(self, dense):
        flat = torch.zeros_like(self.eng.flat_params)
        for (name, _), (off, n) in zip(self.eng.params, self.eng.flat_views):
            flat[off:off + n] = torch.from_numpy(dense[name][0]).to(flat.device)
        return flat

    # ------------------------------------------------------------------ after a step
    def check_step(self, t, p, ids, dense, labels, pre, next_ids):
        group, eng, N = self.group, self.eng, self.world
        G, B, D = eng.G, eng.B, eng.D
        what = "%s rank %d step %d" % (self.label, self.rank, t)
        # 1. dedup of the batch that trained, and of the next batch where it ran beside the push
        _check_dedup(_plan_dedup(eng.plans[p], G, B), pre["dedup"], what + " dedup")
        if next_ids is not None:
            _check_dedup(_plan_dedup(eng.plans[eng.cur], G, B), _oracle_dedup(next_ids), what + " next-batch dedup")
        # 2. the rows the exchange pulled are the pre-step rows, bit for bit
        n_unique = [len(u) for u, _ in pre["dedup"]]
        bet = {"wide": eng.bet_w.view(G, B, 1).cpu().numpy(), "deep": eng.bet_d.view(G, B, D).cpu().numpy()}
        for name, g, fam in self.tables():
            got, want = bet[fam][g, :n_unique[g]], pre["batch_rows"][name]
            assert np.array_equal(got, want), "%s: %s rows pulled through the exchange != pre-step rows (%d of %d differ)" % (
                what, name, int((got != want).any(axis=1).sum()), n_unique[g])
        # 3. tower outputs against the float64 reference on those rows and the dense parameters the step pulled
        inv, nu, _ = T.first_occurrence_inverse(ids)
        bw = torch.full((G, B), float("nan"), device=self.dev)
        bd = torch.full((G, B, D), float("nan"), device=self.dev)
        for g in range(G):
            bw[g, :n_unique[g]] = eng.bet_w.view(G, B)[g, :n_unique[g]]
            bd[g, :n_unique[g]] = eng.bet_d.view(G, B, D)[g, :n_unique[g]]
        ref = T.tower_reference(inv, nu, bw, bd, dense, labels, eng.flat_params)
        raced = not torch.equal(eng.flat_params, pre["flat"])
        if raced and bool(T.near_relu_kink(ref).any()):
            print("%s: tower comparison skipped: a peer's dense push of this step landed before this rank's "
                  "pull_dense and %d samples lie within the kink margin" % (what, int(T.near_relu_kink(ref).sum())))
        else:
            got = {"loss": eng.loss_buf, "logits": eng.logits_buf, "grads": eng.flat_grads,
                   "gsum_wide": eng.gsum_w.view(G, B), "gsum_deep": eng.gsum_d.view(G, B, D)}
            T.check(got, ref, families=T.FAMILIES, label=what, n_sm=torch.cuda.get_device_properties(self.dev).multi_processor_count)
            self.compared += 1
        # 4. the rows of this rank's shard: the oracle's Adam of every rank's push, in rank order, under one
        # assignment of this step's shard steps to the ranks
        gsum = {"wide": eng.gsum_w.view(G, B, 1).cpu().numpy(), "deep": eng.gsum_d.view(G, B, D).cpu().numpy()}
        pushed = _gather({
            "uniq": [eng.plans[p]["uniq"].view(G, B)[g, :n_unique[g]].cpu().numpy() for g in range(G)],
            "wide": [gsum["wide"][g, :n_unique[g]] for g in range(G)],
            "deep": [gsum["deep"][g, :n_unique[g]] for g in range(G)],
            "flat_grads": eng.flat_grads.cpu().numpy()})
        steps = range((t - 1) * N + 1, t * N + 1)
        cands = list(itertools.permutations(steps))
        matching = set(cands)
        for name, g, fam in self.tables():
            own = pre["own"][g]
            if not len(own):
                continue
            p0, m0, v0 = pre["own_state"][name]
            now = _slots(group, name, own)
            src_rows = []  # per source: (positions in `own`, its gradient rows for them)
            for src in range(N):
                u = pushed[src]["uniq"][g]
                mine = u % N == self.rank
                src_rows.append((np.searchsorted(own, u[mine]), pushed[src][fam][g][mine]))
            touched = np.zeros(len(own), dtype=bool)
            for pos, _ in src_rows:
                touched[pos] = True
            for kind, a, b in zip(("param", "m", "v"), now, (p0, m0, v0)):
                assert np.array_equal(a[~touched], b[~touched]), "%s: %s %s of a row no rank pushed changed" % (
                    what, name, kind)
            for perm in list(matching):
                want = [x.copy() for x in (p0, m0, v0)]
                for src, (pos, gr) in enumerate(src_rows):
                    out = _adam(gr, want[0][pos], want[1][pos], want[2][pos], perm[src])
                    for w, o in zip(want, out):
                        w[pos] = o
                if not all(np.array_equal(a, b) for a, b in zip(now, want)):
                    matching.discard(perm)
            assert matching, ("%s: %s: the shard's rows match the oracle's Adam of the ranks' pushes in rank order "
                              "under no assignment of steps %s to the ranks" % (what, name, list(steps)))
        matching = sorted(matching)
        print("%s: shard %d rows match rank order 0..%d with rank -> step %s" % (
            what, self.rank, N - 1, " or ".join(str(dict(enumerate(m))) for m in matching)))
        # 5. dense parameters: each rank's lock-free update with the alpha of the step it drew on the owner shard
        shard_steps = _gather(matching)
        dense1 = _dense(group, eng)
        races = 0
        for (name, _), (off, n) in zip(eng.params, eng.flat_views):
            now = dense1[name]
            if N != 2:
                assert all(np.isfinite(x).all() for x in now), "%s: dense %s not finite" % (what, name)
                continue
            owner = group.dense_owner[name]
            grads = [pushed[r]["flat_grads"][off:off + n] for r in range(N)]
            ok, serial = self._dense_interleavings(pre["dense"][name], now, grads, shard_steps[owner])
            assert ok.all(), ("%s: dense %s: %d elements no interleaving of the two ranks' Adam updates produces "
                              "(first at %s)" % (what, name, int((~ok).sum()), np.flatnonzero(~ok)[:4].tolist()))
            races += int((~serial).sum())
        if N == 2:
            self.races.append(races)
            print("%s: %d dense elements show a lost or torn update" % (what, races))
        # 6. counters, the loss ring, no error raised
        assert group.snapshot() == [(t * N, t * N, True)] * N, (what, group.snapshot())
        assert eng.steps == t, (what, eng.steps)
        assert eng.loss_host(t - 1) == float(eng.loss_buf), what

    @staticmethod
    def _dense_interleavings(before, now, grads, assignments):
        """(ok, serial) per element of one dense parameter at two ranks.  Each rank loads p, m and v, updates them and
        stores them; the first rank to load reads the pre-step values, the second reads each of p, m, v either
        before the first stored it or after, and the value left is either rank's (the last store); it is the
        second rank's where that rank read the first's.  serial: the element equals one rank's update applied on
        top of the other's (no update lost, none torn)."""
        ok = np.zeros(before[0].shape, dtype=bool)
        serial = np.zeros_like(ok)
        for steps in assignments:
            for first in (0, 1):
                second = 1 - first
                f = _adam(grads[first], *before, steps[first])
                for reads in itertools.product((False, True), repeat=3):  # second rank read the first's p / m / v
                    s = _adam(grads[second], *[fx if r else bx for fx, bx, r in zip(f, before, reads)], steps[second])
                    hit = np.ones_like(ok)
                    for x, sx, fx, r in zip(now, s, f, reads):
                        hit &= (x == sx) | (~np.bool_(r) & (x == fx))
                    ok |= hit
                    if all(reads):
                        serial |= (now[0] == s[0]) & (now[1] == s[1]) & (now[2] == s[2])
        return ok, serial

    def close(self):
        _sync()  # no peer still reads this rank's shard
        self.group.close()


def run_leg(world, rank, dev, B, transport, feed):
    from elasticdl_b200.workloads.deepfm import pack_batch, packed_views, synthetic_batch

    label = "world %d B=%d %s/%s" % (world, B, transport, feed)
    t0 = time.time()
    leg = Leg(world, rank, dev, B, transport, feed, label)
    eng, group = leg.eng, leg.group
    G = eng.G
    try:
        batches = [list(synthetic_batch(B, 1234 + p + 1000 * rank, dev, "zipf")) for p in range(STEPS + 1)]
        ahead = feed in ("device", "host")
        _sync()  # every rank's rows and dense parameters are set before any peer reads them
        _condition(group, eng, *batches[0], seed=1 + 100 * rank)
        feeder, src = None, None
        if feed == "device":
            src = [pack_batch(*b, widths=eng.widths) for b in batches]
        elif feed == "host":
            src = [(pack_batch(*(x.cpu() for x in b), pin=True, widths=eng.widths),) for b in batches]
            feeder = eng.host_feeder(3, lookahead=True)
            for s in src[:2]:
                feeder.submit(*s)
                torch.cuda.synchronize()
        elif feed == "graph":
            eng.capture()
        for t in range(1, STEPS + 1):
            ids, dense, labels = batches[t - 1]
            _sync()
            if t > 1:
                _condition(group, eng, ids, dense, labels, seed=t + 100 * rank)
                if ahead:  # batch t sits in the static buffer the next replay trains on
                    packed_views(eng.s_packed[eng.cur], G, B, eng.widths)[1].copy_(dense)
            pre = leg.pre_state(ids)
            if feed == "device" and t == 1:
                eng.prepare_packed(src[0])
            _sync()  # no rank pushes before every rank has read the pre-step state
            p = eng.cur
            if feed == "device":
                eng.step_ahead_graph(src[t])
            elif feed == "host":
                if t + 1 < len(src):
                    feeder.submit(*src[t + 1])
                    torch.cuda.synchronize()
                feeder.run_next()
            elif feed == "graph":
                eng.step_graph(pack_batch(ids, dense, labels, widths=eng.widths))
            else:
                assert feed == "step"
                eng.step(ids, dense, labels)
            _sync()
            group.check()
            leg.check_step(t, p, ids, dense, labels, pre, batches[t][0] if ahead else None)
        assert leg.compared > 0, "%s rank %d: no step got a tower comparison" % (label, rank)
    finally:
        leg.close()
    return "%s: %.1f s, tower compared on %d of %d steps%s" % (
        label, time.time() - t0, leg.compared, STEPS,
        ", dense lost / torn elements per step %s" % leg.races if world == 2 else "")


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
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    if world == 2:
        legs = [(32768, "narrow", "device"), (32768, "narrow", "host"), (32768, "int32", "device"),
                (32768, "narrow", "graph"), (32768, "narrow", "step")]
    else:  # a last tile of one sample; the groups of 2 rows leave shard 2 owning none of their rows
        legs = [(2 * n_sm * 32 + 1, "narrow", "device"), (2 * n_sm * 32 + 1, "narrow", "step"),
                (32768, "narrow", "device")]
    t0 = time.time()
    lines = [run_leg(world, rank, dev, *leg) for leg in legs]
    _sync()
    for r in range(world):
        if r == rank:
            print("rank %d:\n  %s" % (rank, "\n  ".join(lines)))
            sys.stdout.flush()
        dist.barrier()
    if rank == 0:
        print("mgpu_bench_step_check ok: world=%d in %.0f s" % (world, time.time() - t0))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
