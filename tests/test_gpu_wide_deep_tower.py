"""The Wide & Deep tile tower (csrc/deepfm_tower2.cu without the FM term, include/b200_deepfm.h
b200_deepfm_wide_deep_*) against the float64 reference of oracle/wide_deep_oracle.py.

Kernel level, through the C ABI (no PS), every output poisoned with NaN before each call: group counts up to the
tile tower's 38, batches at the tile and wave edges and at 32768, the id patterns that stress the warp-level id
dedup, the value regimes of the DeepFM tests, both row sources (pulled bet_* rows and the table records), the
prologue + main split against the one-call entry, forward-only logits, the comparator's mutations and the refusals.
Batches are conditioned as in test_gpu_tower_reference.py: samples with a DNN pre-activation within 1e-4 * M of a
ReLU kink get a new dense row.

Engine level: DeepFMPSEngine(model="wide_deep") over several Adam steps at B = 32768 on bench.py's Zipf batches,
through the graphed lookahead feed on narrow packed ids, the host feeder and eager step(); every step's dedup, loss,
gradients and Adam push checked as test_gpu_engine_bench_path.py checks DeepFM's, then predict(); and the graphed
pipeline against eager steps."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ps_oracle as O
from oracle import wide_deep_oracle as T
from tests.test_gpu_tower_reference import NAN, Buffers, _batch, _ids, _n_sm

pytestmark = pytest.mark.gpu
TAU = 1e-4
WORST = {}


def _dev():
    return torch.device("cuda", 0)


reference = T.wide_deep_reference


def make_inputs(G, B, pattern="zipf", regime="base", seed=0):
    """Device inputs of one batch in the kernel's layout, conditioned; rows at or past n_unique[g] and the padding
    floats of the parameters are NaN (test_gpu_tower_reference.make_inputs with the Wide & Deep reference)."""
    dev = _dev()
    gen = torch.Generator(device=dev).manual_seed(3000 + seed)
    ids = _ids(pattern, G, B, seed, gen)
    inv, n_unique, _ = T.first_occurrence_inverse(ids)
    sw = sd = 0.5 * (5.0 / max(G, 5)) ** 0.5
    live = torch.arange(B, device=dev).unsqueeze(0) < n_unique.unsqueeze(1).long()
    bet_wide = torch.where(live, torch.randn((G, B), generator=gen, device=dev) * sw, NAN).contiguous()
    bet_deep = torch.where(live.unsqueeze(2), torch.randn((G, B, T.D), generator=gen, device=dev) * sd, NAN).contiguous()
    dense = torch.randn((B, T.ND), generator=gen, device=dev)
    labels = torch.rand(B, generator=gen, device=dev) if regime == "soft" else \
        (torch.rand(B, generator=gen, device=dev) < 0.25).float()
    kw = {}
    if regime == "large_logit":
        kw["wd_std"] = 6.0
    if regime == "dead_l1":
        kw.update(b1=-100.0, b2=[0.5, -0.5, 0.7, 0.3])
    params = T.random_params(G, gen, dev, pad=NAN, **kw)
    for _ in range(40):
        ref = reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params)
        near = T.near_relu_kink(ref, TAU)
        if not bool(near.any()):
            break
        dense[near] = torch.randn((int(near.sum()), T.ND), generator=gen, device=dev)
    else:
        raise AssertionError("conditioning did not converge")
    if regime == "large_logit" and B >= 1000:
        assert float(ref["logits"].abs().max()) > 50
    return (inv, n_unique, bet_wide, bet_deep, dense, labels, params), ref


def _call(kind, a):
    from elasticdl_b200 import _lib

    L = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    p = ctypes.byref(a)
    if kind == "split":
        rc = L.b200_deepfm_wide_deep_tile_prologue(p, st)
        return rc or L.b200_deepfm_wide_deep_tile_main(p, st)
    return {"tile": L.b200_deepfm_wide_deep_fwd_bwd_tile, "forward": L.b200_deepfm_wide_deep_forward_tile}[kind](p, st)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nWide & Deep tile tower, largest err / bound per output family (%s, %d SMs):" % (
            torch.cuda.get_device_name(0), _n_sm()))
        for (kind, fam), r in sorted(WORST.items()):
            print("  %-8s %-10s %.4f" % (kind, fam, r))


def _outputs(buf):
    return {"logits": buf.logits, "loss": buf.loss, "grads": buf.grads, "gsum_wide": buf.gsum_wide,
            "gsum_deep": buf.gsum_deep}


def run_and_check(kind, G, B, pattern="zipf", regime="base", seed=0, calls=2, table_rows=False):
    """`calls` calls on the same buffers, each with a new batch, every output poisoned before."""
    buf = Buffers(G, B)
    backward = kind != "forward"
    out = []
    for k in range(calls):
        inputs, ref = make_inputs(G, B, pattern, regime, seed=seed * 7 + k)
        buf.load(inputs)
        a = buf.args(backward)
        group = None
        if table_rows:
            from tests.test_gpu_tower_table_rows import ADAM, _rows_struct, _table_state

            group, uniq = _table_state(ADAM, inputs, seed * 7 + k)
            rows = _rows_struct(group, G, uniq)
            buf.bet_wide.fill_(NAN)  # the tower must read the tables, not these
            buf.bet_deep.fill_(NAN)
            a.rows = ctypes.pointer(rows)
        try:
            rc = _call(kind, a)
            assert rc == 0, (kind, rc)
            torch.cuda.synchronize()
        finally:
            if group is not None:
                group.close()
        label = "wide_deep %s G=%d B=%d %s/%s%s call %d:" % (kind, G, B, pattern, regime, " table" if table_rows else "",
                                                              k)
        fams = T.FAMILIES if backward else ("logits",)
        rs = T.check({f: v for f, v in _outputs(buf).items() if f in fams}, ref, families=fams, label=label,
                     n_sm=_n_sm())
        for fam, r in rs.items():
            WORST[(kind, fam)] = max(WORST.get((kind, fam), 0.0), r)
        if backward:
            dead = torch.arange(B, device=_dev()).unsqueeze(0) >= inputs[1].unsqueeze(1).long()
            assert torch.isnan(buf.gsum_wide[dead]).all() and torch.isnan(buf.gsum_deep[dead]).all(), label
            if regime == "dead_l1":  # no live hidden unit: dW1, db1 and dW2 are exactly 0
                o = T.layout(G)
                assert (buf.grads[o["w1"]:o["w2"] + T.H2 * T.H1] == 0).all(), label
        out.append((inputs, {f: v.clone() for f, v in _outputs(buf).items()}))
    return out


SHAPES_B = ["1", "31", "32", "33", "tile_wave2", "32768"]


@pytest.mark.parametrize("B", SHAPES_B)
@pytest.mark.parametrize("G", [1, 5, 33, 38])
def test_wide_deep_tower_shapes(G, B):
    run_and_check("tile", G, _batch(B), seed=G)


@pytest.mark.parametrize("B", ["33", "tile_wave2", "32768"])
@pytest.mark.parametrize("pattern", ["equal", "distinct", "zipf", "lanes", "straddle"])
def test_wide_deep_tower_id_patterns(pattern, B):
    run_and_check("tile", 38, _batch(B), pattern=pattern, seed=11)


@pytest.mark.parametrize("B", ["1000", "32768"])
@pytest.mark.parametrize("regime", ["base", "large_logit", "dead_l1", "soft"])
def test_wide_deep_tower_value_regimes(regime, B):
    run_and_check("tile", 38, _batch(B), regime=regime, seed=21)


@pytest.mark.parametrize("B", ["1", "33", "tile_wave2", "32768"])
@pytest.mark.parametrize("G", [5, 38])
def test_wide_deep_tower_table_rows(G, B):
    """Rows straight from the table records (NaN everywhere else in the tables and in bet_*)."""
    run_and_check("tile", G, _batch(B), seed=41, table_rows=True)


@pytest.mark.parametrize("B", SHAPES_B)
def test_wide_deep_split_prologue_main_equals_one_call(B):
    """The branched step's prologue + main kernel: within the bound, and the forward logits equal the one-call
    entry's bit for bit (the forward has no atomics)."""
    Bn = _batch(B)
    split = run_and_check("split", 38, Bn, seed=3, calls=1)
    one = run_and_check("tile", 38, Bn, seed=3, calls=1)
    assert torch.equal(split[0][1]["logits"], one[0][1]["logits"])


@pytest.mark.parametrize("B", SHAPES_B)
@pytest.mark.parametrize("G", [5, 38])
def test_wide_deep_forward_only(G, B):
    """Forward-only logits within the bound of the reference logits, and equal bit for bit to the training call's
    (the same forward code)."""
    Bn = _batch(B)
    fwd = run_and_check("forward", G, Bn, seed=31, calls=1)
    one = run_and_check("tile", G, Bn, seed=31, calls=1)
    assert torch.equal(fwd[0][1]["logits"], one[0][1]["logits"])


@pytest.mark.parametrize("B", SHAPES_B)
@pytest.mark.parametrize("G", [1, 5, 33, 38])
def test_wide_deep_mutations_are_caught(G, B):
    """The comparator rejects each classic tiled-reduction fault (wide_deep_oracle.mutations) at every
    shape tested."""
    Bn = _batch(B)
    inputs, ref = make_inputs(G, Bn, "zipf", seed=G + 100)
    for name, got in T.mutations(ref, inputs).items():
        if name == "loss_not_divided_by_B" and Bn == 1:
            continue  # the same number
        assert T.caught_by(got, ref, n_sm=_n_sm()), (name, G, Bn, {f: v[0] for f, v in T.ratios(got, ref,
                                                                                             n_sm=_n_sm()).items()})


def test_wide_deep_refusals():
    """G = 39 is refused (-1) by every Wide & Deep entry point without a launch, and b200_deepfm_last_error names
    the model and the limit; a row source on the forward-only entry is refused the same way; the engine refuses
    model="wide_deep" on the fused / mma towers and past 38 groups."""
    from elasticdl_b200 import _lib
    from elasticdl_b200._lib import DeepFMRows
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    L = _lib.lib()
    G = 39
    buf = Buffers(G, 64)
    buf.load(make_inputs(G, 64, seed=G)[0])
    for kind in ("tile", "split", "forward"):
        before = L.b200_deepfm_tile_launch_count()
        assert _call(kind, buf.args(kind != "forward")) == -1, kind
        assert L.b200_deepfm_last_error() == b"the Wide & Deep tile tower holds at most 38 id groups", kind
        assert L.b200_deepfm_tile_launch_count() == before, kind
    torch.cuda.synchronize()
    assert torch.isnan(buf.logits).all() and torch.isnan(buf.grads).all()
    G = 5
    buf = Buffers(G, 64)
    buf.load(make_inputs(G, 64, seed=G)[0])
    a = buf.args(False)
    rows = DeepFMRows()
    a.rows = ctypes.pointer(rows)
    before = L.b200_deepfm_tile_launch_count()
    assert _call("forward", a) == -1
    assert L.b200_deepfm_last_error() == b"the forward-only Wide & Deep tile tower reads pulled rows only"
    assert L.b200_deepfm_tile_launch_count() == before
    torch.cuda.synchronize()
    assert torch.isnan(buf.logits).all()
    group = PSGroup(1, "Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", device=0)
    try:
        for tower in ("fused", "mma"):
            with pytest.raises(ValueError, match="wide_deep"):
                DeepFMPSEngine(group, 64, group_rows=[10, 20], tower=tower, model="wide_deep")
        with pytest.raises(ValueError, match="38"):
            DeepFMPSEngine(group, 64, group_rows=[10] * 39, model="wide_deep")
        assert group.tables == {}, sorted(group.tables)  # refused before any table was registered
    finally:
        group.close()


# ---------------------------------------------------------------------------------------------------- engine level

def _ps_reference(group, eng, ids, dense, labels):
    """The float64 Wide & Deep reference of one batch from what the PS holds now (the batch's rows, the dense
    parameters)."""
    G, B, dev = eng.G, eng.B, eng.device
    inv, n_unique, uniq = T.first_occurrence_inverse(ids)
    bet_w = torch.full((G, B), NAN, device=dev)
    bet_d = torch.full((G, B, T.D), NAN, device=dev)
    for g in range(G):
        u = int(n_unique[g])
        touched = uniq[g, :u].cpu()
        bet_w[g, :u] = group.pull_rows([(eng.wide_names[g], touched)])[0].reshape(u).to(dev)
        bet_d[g, :u] = group.pull_rows([(eng.deep_names[g], touched)])[0].reshape(u, T.D).to(dev)
    d = group.pull_dense([n for n, _ in eng.params])
    params = torch.zeros(T.layout(G)["total"], dtype=torch.float32, device=dev)
    for (name, _), (off, n) in zip(eng.params, eng.flat_views):
        params[off:off + n] = torch.as_tensor(d[name]).reshape(-1).to(dev)
    return reference(inv, n_unique, bet_w, bet_d, dense, labels, params)


def _condition(group, eng, ids, dense, labels, seed):
    gen = torch.Generator(device=_dev()).manual_seed(seed)
    for _ in range(40):
        ref = _ps_reference(group, eng, ids, dense, labels)
        near = T.near_relu_kink(ref)
        if not bool(near.any()):
            return ref
        dense[near] = torch.randn((int(near.sum()), T.ND), generator=gen, device=_dev())
    raise AssertionError("conditioning did not converge")


def _check_step(group, eng, t, p, dedup, ref, pre, sample, label):
    """test_gpu_engine_bench_path._check_step against the Wide & Deep reference."""
    from tests.test_gpu_engine_bench_path import BETA1, BETA2, EPS, LR, _check_dedup, _dense, _plan_dedup, _rows, _tables

    G, B, D = eng.G, eng.B, eng.D
    what = "%s step %d" % (label, t)
    _check_dedup(_plan_dedup(eng.plans[p], G, B), dedup, what + " dedup")
    got = {"loss": eng.loss_buf, "logits": eng.logits_buf, "grads": eng.flat_grads,
           "gsum_wide": eng.gsum_w.view(G, B), "gsum_deep": eng.gsum_d.view(G, B, D)}
    T.check(got, ref, label=what, n_sm=_n_sm())
    tabs, dense0, snap0 = pre
    assert snap0 == [(t - 1, t - 1, True)], (what, snap0)
    gsum = {"wide": eng.gsum_w.view(G, B, 1).cpu().numpy(), "deep": eng.gsum_d.view(G, B, D).cpu().numpy()}
    for name, g, fam in _tables(eng):
        u = dedup[g][0]
        (p0, m0, v0), sample0 = tabs[name]
        want = [x.copy() for x in (p0, m0, v0)]
        O.np_adam(gsum[fam][g, :len(u)].copy(), *want, LR, t, BETA1, BETA2, EPS)
        for kind, a, b in zip(("param", "m", "v"), _rows(group, name, u), want):
            assert np.array_equal(a, b), "%s: %s %s of the pushed rows != oracle Adam" % (what, name, kind)
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
    assert eng.steps == t and eng.loss_host(eng.steps - 1) == float(eng.loss_buf), what


def _run_leg(rows, transport, feed, batches, n_steps, label, row_source="auto"):
    from bench import ADAM_ARGS
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, WideDeepTower, pack_batch, packed_views
    from tests.test_gpu_engine_bench_path import FULL_SCAN_ROWS, SAMPLE_ROWS, _check_dedup, _oracle_dedup, \
        _plan_dedup, _pre_state

    B = batches[0][0].shape[1]
    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    try:
        eng = DeepFMPSEngine(group, B, group_rows=rows, id_transport=transport, row_source=row_source,
                             model="wide_deep")
        assert eng.tower_kind == "tile" and eng.row_source == ("table" if row_source == "auto" else row_source)
        assert isinstance(eng.tower, WideDeepTower)
        G = eng.G
        rng = np.random.RandomState(11)
        sample = [np.arange(r) if r <= FULL_SCAN_ROWS else np.sort(rng.choice(r, SAMPLE_ROWS, replace=False))
                  for r in rows]
        ahead = feed in ("device", "host")
        ref = _condition(group, eng, *batches[0], seed=1)
        feeder, src = None, None
        if feed == "device":
            src = [pack_batch(*b, widths=eng.widths) for b in batches]
        elif feed == "host":
            src = [(pack_batch(*(x.cpu() for x in b), pin=True, widths=eng.widths),) for b in batches]
            feeder = eng.host_feeder(3, lookahead=True)
            for s in src[:2]:
                feeder.submit(*s)
                torch.cuda.synchronize()
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
            else:
                assert feed == "step"
                eng.step(ids, dense, labels)
            torch.cuda.synchronize()
            group.check()
            _check_step(group, eng, t, p, dedup, ref, pre, sample, label)
            if ahead:
                _check_dedup(_plan_dedup(eng.plans[eng.cur], G, B), _oracle_dedup(batches[t][0]),
                             "%s step %d next-batch dedup" % (label, t))
        # predict() on the last batch from the state after the last push: the reference forward
        ids, dense, _ = batches[n_steps]
        ref = _ps_reference(group, eng, ids, dense, batches[n_steps][2])
        logits = eng.predict(ids, dense)
        torch.cuda.synchronize()
        T.check({"logits": logits}, ref, families=("logits",), label=label + " predict", n_sm=_n_sm())
    finally:
        group.close()


LEGS = [("narrow", "device", "auto"), ("int32", "host", "auto"), ("narrow", "step", "auto"), ("int32", "step", "pull")]


@pytest.mark.parametrize("transport,feed,row_source", LEGS, ids=["%s-%s-%s" % leg for leg in LEGS])
def test_wide_deep_engine_matches_references_over_adam_steps(transport, feed, row_source):
    """bench.py's configuration with model="wide_deep": B = 32768, the 38 dac_ctr groups at full size, its batches
    (seeds 1234 + p), three Adam steps through one feed, every step checked; then predict()."""
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, synthetic_batch

    batches = [list(synthetic_batch(32768, 1234 + p, _dev(), "zipf")) for p in range(4)]
    _run_leg(GROUP_ROWS, transport, feed, batches, 3, "wide_deep %s/%s/%s" % (transport, feed, row_source), row_source)


def test_wide_deep_engine_graph_equals_eager_step():
    """The captured lookahead graph, the captured one-step graph and eager step() from the same seed and batches:
    losses, rows and dense parameters equal up to the order of fp32 atomic adds (losses rtol 1e-5, parameters
    atol 2e-4 after three Adam steps at lr 1e-3, as test_gpu_layer_trainer.py compares DeepFM's pipelines)."""
    from bench import ADAM_ARGS
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch, synthetic_batch

    rows, B = [5, 10, 1460, 582, 100000, 1000000], 4096
    batches = [synthetic_batch(B, 70 + p, _dev(), "zipf", group_rows=rows) for p in range(4)]
    results = []
    for mode in ("eager", "ahead", "graph"):
        group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
        try:
            eng = DeepFMPSEngine(group, B, group_rows=rows, id_transport="narrow", model="wide_deep")
            losses = []
            if mode == "ahead":
                eng.prepare_packed(pack_batch(*batches[0], widths=eng.widths))
                for t in range(3):
                    eng.step_ahead_graph(pack_batch(*batches[t + 1], widths=eng.widths))
                    losses.append(float(eng.loss_buf))
            elif mode == "graph":
                eng.capture()
                for t in range(3):
                    eng.step_graph(*batches[t])
                    losses.append(float(eng.loss_buf))
            else:
                for t in range(3):
                    eng.step(*batches[t])
                    losses.append(float(eng.loss_buf))
            torch.cuda.synchronize()
            group.check()
            tabs = [group.pull_rows([(n, torch.arange(r))])[0].cpu() for n, r in zip(eng.wide_names + eng.deep_names,
                                                                                     rows + rows)]
            dense = group.pull_dense([n for n, _ in eng.params])
            results.append((losses, tabs, [dense[n].cpu() for n, _ in eng.params]))
        finally:
            group.close()
    l0, t0, d0 = results[0]
    for l1, t1, d1 in results[1:]:
        assert np.allclose(l0, l1, rtol=1e-5), (l0, l1)
        for a, b in zip(t0 + d0, t1 + d1):
            assert torch.allclose(a, b, rtol=0, atol=2e-4), float((a - b).abs().max())
