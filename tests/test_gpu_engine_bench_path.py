"""The DeepFM step bench.py times, checked against references over several Adam steps.

bench.py builds PSGroup(1, "Adam", ADAM_ARGS) and DeepFMPSEngine(group, 32768, id_transport=...) -- the tile tower,
reading its rows straight from the table records -- packs every batch with pack_batch(..., widths=engine.widths)
and runs prepare_packed + step_ahead_graph on device buffers (the headline), the lookahead host feeder on pinned
buffers (e2e), capture + step_graph (--lookahead off) and step() on int64 ids (the eager pass).  Every leg here
drives one of those feeds one call at a time and checks each step t against
  1. the oracle's first-occurrence dedup, exactly (and, on the lookahead feeds, the next batch's dedup that ran
     beside the push);
  2. the float64 tower reference of the state the step started from (oracle/tower_oracle.py bound);
  3. the oracle's Adam (step t) applied to the gradients the engine pushed, from the pre-step param / m / v, bit
     for bit; every other row untouched; version = step = t;
  4. the loss ring.
From step 2 on Adam's m, v and step counter are non-zero, so the slot updates and the bias correction are checked
too.  Batches are conditioned as in test_gpu_tower_reference.py: dense rows of samples with a pre-activation
within 1e-4 * M of a ReLU kink are redrawn (against the state the step will start from).
"""
import numpy as np
import pytest
import torch

from bench import ADAM_ARGS
from oracle import ps_oracle as O
from oracle import tower_oracle as T
from tests.test_gpu_layer_trainer import _ps_reference

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
LR, BETA1, BETA2, EPS = 1e-3, 0.9, 0.999, 1e-7  # ADAM_ARGS
FULL_SCAN_ROWS = 16384  # tables up to this size are compared row by row after a push ...
SAMPLE_ROWS = 4096  # ... larger ones at this many seeded rows
BENCH_B, BENCH_STEPS = 32768, 3


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _condition(group, eng, ids, dense, labels, seed, dense_params=None):
    """Redraw, in place, the dense rows of the samples whose float64 pre-activation lies near a ReLU kink under the
    state the PS holds now (dense parameters: `dense_params` where given): their fp32 mask may flip, which no
    rounding bound covers.  Returns the float64 reference of the conditioned batch (_ps_reference)."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    for _ in range(40):
        _, ref = _ps_reference(group, eng, ids, dense, labels, dense_params)
        near = T.near_relu_kink(ref)
        if not bool(near.any()):
            return ref
        dense[near] = torch.randn((int(near.sum()), T.ND), generator=gen, device=DEV)
    raise AssertionError("conditioning did not converge")


def _oracle_dedup(ids):
    """[(unique ids in first-occurrence order, inverse)] per group of int64 ids [G, B]."""
    return [O.unique_first_occurrence(row) for row in ids.cpu().numpy()]


def _plan_dedup(plan, G, B):
    n = plan["n_unique"].cpu().numpy()
    uniq = plan["uniq"].view(G, B).cpu().numpy()
    inv = plan["inv"].view(G, B).cpu().numpy()
    return [(uniq[g, :n[g]].copy(), inv[g].copy()) for g in range(G)]


def _check_dedup(got, want, what):
    for g, ((gu, gi), (wu, wi)) in enumerate(zip(got, want)):
        assert len(gu) == len(wu), "%s, group %d: n_unique %d, oracle %d" % (what, g, len(gu), len(wu))
        assert np.array_equal(gu, wu), "%s, group %d: unique ids differ from the oracle's" % (what, g)
        assert np.array_equal(gi, wi), "%s, group %d: inverse differs from the oracle's" % (what, g)


def _tables(eng):
    """(name, group, family) of the 2G tables."""
    return [(n, g, "wide") for g, n in enumerate(eng.wide_names)] + [(n, g, "deep") for g, n in enumerate(eng.deep_names)]


def _rows(group, name, ids):
    """(param, m, v) of rows `ids` of table `name`, numpy float32 [len(ids), dim]."""
    t = torch.from_numpy(np.ascontiguousarray(ids, dtype=np.int64))
    return (group.pull_rows([(name, t)])[0].cpu().numpy(),
            group.slot_rows(name, t, 1).cpu().numpy(), group.slot_rows(name, t, 2).cpu().numpy())


def _dense(group, eng):
    """{name: (param, m, v)} of the dense parameters, flat numpy float32."""
    out = {}
    for name, _ in eng.params:
        p = group.pull_dense([name])[name]
        out[name] = tuple(x.cpu().numpy().reshape(-1) for x in (p, group.slot_dense(name, 1), group.slot_dense(name, 2)))
    return out


def _pre_state(group, eng, dedup, sample):
    """What the next step starts from: param / m / v of the batch's unique rows of every table (oracle order) and of
    a fixed sample of every table's rows, the dense parameters and their slots, the shard state."""
    tabs = {name: (_rows(group, name, dedup[g][0]), _rows(group, name, sample[g])) for name, g, _ in _tables(eng)}
    return tabs, _dense(group, eng), group.snapshot()


def _check_step(group, eng, t, p, dedup, ref, pre, sample, label):
    """Checks 1-4 of step t (1-based count of pushes this group has seen), trained on plan p."""
    G, B, D = eng.G, eng.B, eng.D
    what = "%s step %d" % (label, t)
    # 1. dedup of the batch that trained
    _check_dedup(_plan_dedup(eng.plans[p], G, B), dedup, what + " dedup")
    # 2. forward, backward, loss within the float64 reference's bound
    got = {"loss": eng.loss_buf, "logits": eng.logits_buf, "grads": eng.flat_grads,
           "gsum_wide": eng.gsum_w.view(G, B), "gsum_deep": eng.gsum_d.view(G, B, D)}
    T.check(got, ref, families=T.FAMILIES, label=what, n_sm=_n_sm())
    # 3. push: oracle Adam (step t) on the gradient rows the engine pushed, from the pre-step state, bit for bit
    tabs, dense0, snap0 = pre
    assert snap0 == [(t - 1, t - 1, True)], (what, snap0)
    gsum = {"wide": eng.gsum_w.view(G, B, 1).cpu().numpy(), "deep": eng.gsum_d.view(G, B, D).cpu().numpy()}
    for name, g, fam in _tables(eng):
        u = dedup[g][0]
        (p0, m0, v0), sample0 = tabs[name]
        want = [x.copy() for x in (p0, m0, v0)]
        O.np_adam(gsum[fam][g, :len(u)].copy(), *want, LR, t, BETA1, BETA2, EPS)
        for kind, a, b in zip(("param", "m", "v"), _rows(group, name, u), want):
            assert np.array_equal(a, b), "%s: %s %s of the pushed rows != oracle Adam (max |diff| %g)" % (
                what, name, kind, float(np.abs(a - b).max()))
        keep = ~np.isin(sample[g], u)
        for kind, a, b in zip(("param", "m", "v"), _rows(group, name, sample[g]), sample0):
            assert np.array_equal(a[keep], b[keep]), "%s: %s %s of a row outside the batch changed" % (what, name, kind)
    flat_g = eng.flat_grads.cpu().numpy()
    dense1 = _dense(group, eng)
    for (name, _), (off, n) in zip(eng.params, eng.flat_views):
        want = [x.copy() for x in dense0[name]]
        O.np_adam(flat_g[off:off + n].copy(), *want, LR, t, BETA1, BETA2, EPS)
        for kind, a, b in zip(("param", "m", "v"), dense1[name], want):
            assert np.array_equal(a, b), "%s: dense %s %s != oracle Adam" % (what, name, kind)
    assert group.snapshot() == [(t, t, True)], what
    # 4. the loss ring holds this step's loss
    assert eng.steps == t, (what, eng.steps)
    assert eng.loss_host(eng.steps - 1) == float(eng.loss_buf), what


def _run_leg(rows, transport, feed, batches, n_steps, label):
    """A fresh group and engine (bench.py's configuration over `rows`), n_steps steps through `feed`, every step
    checked.  batches: [ids int64, dense, labels] device tensors, n_steps + 1 of them (the lookahead feeds load one
    batch ahead); dense is conditioned in place.  Returns the dedup of every step."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch, packed_views

    B = batches[0][0].shape[1]
    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    try:
        eng = DeepFMPSEngine(group, B, group_rows=rows, id_transport=transport)
        assert eng.tower_kind == "tile" and eng.row_source == "table", (eng.tower_kind, eng.row_source)
        G = eng.G
        rng = np.random.RandomState(11)
        sample = [np.arange(r) if r <= FULL_SCAN_ROWS else np.sort(rng.choice(r, SAMPLE_ROWS, replace=False))
                  for r in rows]
        ahead = feed in ("device", "host", "host-tensors")
        # batch 1 is conditioned before it is packed; a lookahead feed loads batch t + 1 during step t, so that batch
        # is conditioned in the static buffer it sits in (only the next replay reads its dense region)
        ref = _condition(group, eng, *batches[0], seed=1)
        feeder, src = None, None
        if feed == "device":
            src = [pack_batch(*b, widths=eng.widths) for b in batches]
        elif feed == "host":
            src = [(pack_batch(*(x.cpu() for x in b), pin=True, widths=eng.widths),) for b in batches]
        elif feed == "host-tensors":
            src = [tuple(x.cpu().pin_memory() for x in b) for b in batches]
        elif feed == "graph":
            eng.capture()
        if feed in ("host", "host-tensors"):
            feeder = eng.host_feeder(3, lookahead=True)
            for s in src[:2]:
                feeder.submit(*s)
                torch.cuda.synchronize()
        dedups = []
        for t in range(1, n_steps + 1):
            ids, dense, labels = batches[t - 1]
            if t > 1:
                ref = _condition(group, eng, ids, dense, labels, seed=t)
                if ahead:
                    packed_views(eng.s_packed[eng.cur], G, B, eng.widths)[1].copy_(dense)
            dedup = _oracle_dedup(ids)
            pre = _pre_state(group, eng, dedup, sample)
            if feed == "device" and t == 1:
                eng.prepare_packed(src[0])
                torch.cuda.synchronize()
            p = eng.cur
            if feed == "device":
                eng.step_ahead_graph(src[t])
            elif feeder is not None:
                if t + 1 < len(src):
                    feeder.submit(*src[t + 1])
                    torch.cuda.synchronize()
                feeder.run_next()
            elif feed == "graph":
                eng.step_graph(pack_batch(ids, dense, labels, widths=eng.widths))
            else:
                assert feed == "step"
                eng.step(ids, dense, labels)
            torch.cuda.synchronize()
            group.check()
            _check_step(group, eng, t, p, dedup, ref, pre, sample, label)
            if ahead:  # the other plan holds the dedup of the batch loaded for the next step
                _check_dedup(_plan_dedup(eng.plans[eng.cur], G, B), _oracle_dedup(batches[t][0]),
                             "%s step %d next-batch dedup" % (label, t))
            dedups.append(_plan_dedup(eng.plans[p], G, B))
        return dedups
    finally:
        group.close()


# (id transport, feed): bench.py's --ids narrow / int32 headline and e2e legs, the e2e leg on separate pinned tensors,
# --lookahead off, and the eager pass
LEGS = [("narrow", "device"), ("narrow", "host"), ("int32", "device"), ("int32", "host"), ("int32", "host-tensors"),
        ("narrow", "graph"), ("narrow", "step")]


@pytest.mark.parametrize("transport,feed", LEGS, ids=["%s-%s" % leg for leg in LEGS])
def test_bench_step_matches_references_over_adam_steps(transport, feed):
    """bench.py's configuration -- B = 32768, the 38 dac_ctr groups at full size, its batches (seeds 1234 + p) --
    three steps through one of its feeds, every step checked against the oracle's dedup, the float64 tower
    reference and the oracle's Adam."""
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, synthetic_batch

    batches = [list(synthetic_batch(BENCH_B, 1234 + p, DEV, "zipf")) for p in range(BENCH_STEPS + 1)]
    _run_leg(GROUP_ROWS, transport, feed, batches, BENCH_STEPS, "%s/%s" % (transport, feed))


# every id width, both sides of the 16384-row bound between the two dedup kernels, 2-byte ids on both sides of the
# int16 sign bit
EDGE_ROWS = [2, 255, 256, 257, 16384, 16385, 32769, 65535, 65536, 65537, 2_000_000]
EDGE_IDS = (127, 128, 255, 256, 32767, 32768, 65535)


def _edge_batch(B, seed, rows):
    """A Zipf batch in which every group also holds 0, rows - 1 and each of EDGE_IDS below rows, spread from the
    first sample to the last."""
    from elasticdl_b200.workloads.deepfm import synthetic_batch

    ids, dense, labels = synthetic_batch(B, seed, DEV, "zipf", group_rows=rows)
    for g, r in enumerate(rows):
        edges = [0, r - 1] + [v for v in EDGE_IDS if v < r]
        pos = torch.linspace(0, B - 1, len(edges), device=DEV).round().long()
        ids[g, pos] = torch.tensor(edges, device=DEV)
    return [ids, dense, labels]


@pytest.mark.parametrize("B", [4096, None], ids=["B4096", "B2xSMx32p1"])
def test_id_width_edges_match_references(B):
    """Ids at every width boundary through the narrow and int32 packed transports and int64 step(): one step each,
    checked as above, and the three dedups identical.  B = None: 2 * #SM * 32 + 1 (a last tile of one sample)."""
    B = B or 2 * _n_sm() * 32 + 1
    batches = [_edge_batch(B, 50, EDGE_ROWS), _edge_batch(B, 51, EDGE_ROWS)]
    got = {}
    for transport, feed in (("narrow", "device"), ("int32", "device"), ("narrow", "step")):
        leg = [[x.clone() for x in b] for b in batches]
        got[transport, feed] = _run_leg(EDGE_ROWS, transport, feed, leg, 1, "edges B=%d %s/%s" % (B, transport, feed))
    first, *rest = got.values()
    for other in rest:
        _check_dedup(other[0], first[0], "edges B=%d dedup across transports" % B)


def test_packed_ids_outside_the_table_raise_the_range_error():
    """An id that fits its group's width but not its table ([rows, 256**w)) passes pack_batch; the dedup kernel reads
    it, counts it as id 0 and sets the range error, which group.check() raises: 1-, 2- and 4-byte ids, on
    k_unique_small (<= 16384 rows) and on the grid-wide k_unique."""
    from elasticdl_b200 import _lib
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch, synthetic_batch

    rows, B = [200, 5000, 40000, 1_000_000], 4096  # small kernel: 1 and 2 bytes; grid-wide kernel: 2 and 4 bytes
    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    try:
        eng = DeepFMPSEngine(group, B, group_rows=rows, id_transport="narrow")
        assert eng.widths == [1, 2, 2, 4]
        ids, dense, labels = synthetic_batch(B, 3, DEV, "zipf", group_rows=rows)
        eng.prepare_packed(pack_batch(ids, dense, labels, widths=eng.widths))
        torch.cuda.synchronize()
        group.check()  # the clean batch raises nothing
        for g, (r, w) in enumerate(zip(rows, eng.widths)):
            for bad in (r, min(256 ** w, 2 ** 31) - 1):
                bad_ids = ids.clone()
                bad_ids[g, B // 3] = bad
                eng.prepare_packed(pack_batch(bad_ids, dense, labels, widths=eng.widths))
                torch.cuda.synchronize()
                with pytest.raises(_lib.PSRangeError):
                    group.check()
                group.check()  # check() cleared the error word
    finally:
        group.close()


@pytest.mark.parametrize("transport", ["narrow", "int32"])
def test_ids_that_do_not_fit_their_width_are_refused_before_any_copy(transport):
    """A negative id, or one of at least min(256**w, 2**31) for its group's width w, is refused with ValueError by
    pack_batch (host and device inputs), HostFeeder.submit(ids, dense, labels) and step_graph(ids, dense, labels)
    before anything reaches a staging or static buffer; the engine then still trains on a valid batch."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch, synthetic_batch

    rows, B = [200, 5000, 1_000_000], 256
    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    try:
        eng = DeepFMPSEngine(group, B, group_rows=rows, id_transport=transport)
        widths = eng.widths
        assert widths == ([1, 2, 4] if transport == "narrow" else [4, 4, 4])
        ids, dense, labels = synthetic_batch(B, 4, DEV, "zipf", group_rows=rows)
        feeder = eng.host_feeder(2)  # captures the plain step graph (eng.s_one)
        torch.cuda.synchronize()
        s_one, slots = eng.s_one.clone(), [s.clone() for s in feeder.slots]
        host_dense, host_labels = dense.cpu().pin_memory(), labels.cpu().pin_memory()
        for g, w in enumerate(widths):
            for bad in (-1, min(256 ** w, 2 ** 31), 2 ** 32 + 5):
                bad_ids = ids.clone()
                bad_ids[g, 7] = bad
                msg = "id group %d: id %d " % (g, bad)
                with pytest.raises(ValueError, match=msg):
                    pack_batch(bad_ids, dense, labels, widths=widths)
                with pytest.raises(ValueError, match=msg):
                    pack_batch(bad_ids.cpu(), dense.cpu(), labels.cpu(), pin=True, widths=widths)
                with pytest.raises(ValueError, match=msg):
                    feeder.submit(bad_ids.cpu().pin_memory(), host_dense, host_labels)
                with pytest.raises(ValueError, match=msg):
                    eng.step_graph(bad_ids, dense, labels)
        torch.cuda.synchronize()
        assert feeder.head == 0 and eng.steps == 0
        assert torch.equal(eng.s_one, s_one) and all(torch.equal(a, b) for a, b in zip(feeder.slots, slots))
        feeder.submit(ids.cpu().pin_memory(), host_dense, host_labels)
        feeder.run_next()
        eng.step_graph(ids, dense, labels)
        torch.cuda.synchronize()
        group.check()
        assert eng.steps == 2 and group.snapshot() == [(2, 2, True)]
    finally:
        group.close()
