"""The deepctr DeepFM estimator tower (csrc/deepctr_deepfm_tower.cu, include/b200_deepctr_deepfm.h) and
DeepctrDeepfmEngine against the float64 oracle of oracle/deepctr_deepfm_oracle.py.

Kernel level: batches at the tile and grid edges up to 65536 and one past a full grid pass, with uniform ids, one
hot row per table, a quarter of the cells empty, and logits past +-90; the oracle's mutations; bitwise repeats and
graph replay; forward logits equal to the training logits; the refusals; the 3xTF32 statistic.  Engine level: steps
on one and three shards per group against the oracle's TF1 Adagrad and FTRL fed the engine's gradients, every
parameter and accumulator compared; untouched rows; replay; evaluate; four graphed workers."""
import threading

import numpy as np
import pytest
import torch

from elasticdl_b200.common.evaluation_utils import EvaluationMetrics
from elasticdl_b200.ps import PSGroup
from elasticdl_b200.workloads import deepctr_deepfm as M
from oracle import deepctr_deepfm_oracle as O
from oracle import tf32

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(B, pattern, seed):
    """ids int32 [26, B] (-1 absent), dense [13, B], labels, flat (the initialisers with a non-zero linear model)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    if pattern == "one":
        ids = ((torch.arange(M.FIELDS, device=DEV) * 37 + 5) % M.ROWS).to(torch.int32).unsqueeze(1).repeat(1, B)
    else:
        ids = torch.randint(0, M.ROWS, (M.FIELDS, B), generator=g, device=DEV, dtype=torch.int32)
    if pattern == "empty":
        ids[torch.rand(ids.shape, generator=g, device=DEV) < 0.25] = -1
    dense = torch.rand((M.DENSE, B), generator=g, device=DEV) * 2
    labels = (torch.rand(B, generator=g, device=DEV) < 0.3).float()
    flat = M.initial_params(seed, DEV)
    v = M.flat_views(flat)
    for n in M.LIN_NAMES + M.NUM_NAMES:
        v[n].copy_(torch.randn(v[n].shape, generator=g, device=DEV) * 0.05)
    for n in M.EMB_NAMES:
        v[n].mul_(0.3)
    v[M.BIAS_NAME].fill_(0.2)
    if pattern == "saturated":  # logits past +-90: bias_weights +-95 by halves of the batch through I13's weight
        dense[12] = torch.where(torch.rand(B, generator=g, device=DEV) < 0.5, 1.0, -1.0)
        v[M.NUM_NAMES[12]].fill_(95.0)
    return ids.contiguous(), dense.contiguous(), labels, flat


def _batches():
    return [1, 63, 64, 65, 4096, 65536, 64 * _n_sm() + 1]


@pytest.mark.parametrize("pattern", ["uniform", "one", "empty", "saturated"])
@pytest.mark.parametrize("i", range(7))
def test_tower_matches_oracle(i, pattern):
    B = _batches()[i]
    ids, dense, labels, flat = _inputs(B, pattern, seed=B % 991 + len(pattern))
    out = M.deepctr_deepfm_tower(ids, dense, labels, flat)
    ref = O.reference(ids, dense, labels, flat)
    O.check(out, ref, n_sm=_n_sm(), label="B=%d %s" % (B, pattern))
    if pattern == "saturated":
        assert bool((ref["logits"].abs() > 90).all()) and bool(torch.isfinite(out["loss"]))
    fwd = M.deepctr_deepfm_tower(ids, dense, None, flat, train=False)
    assert torch.equal(fwd["logits"], out["logits"])
    touched = torch.zeros((M.FIELDS, M.ROWS), dtype=torch.bool, device=DEV)
    keep = ids >= 0
    touched[torch.arange(M.FIELDS, device=DEV).unsqueeze(1).expand_as(ids)[keep], ids[keep].long()] = True
    assert int(torch.count_nonzero(out["grads"][:O.O_DNN].view(M.FIELDS, M.ROWS, M.DIM)[~touched])) == 0


@pytest.mark.parametrize("B", [300, 65536])
def test_tower_from_raw_rows_with_empty_strings(B):
    """A quarter of the strings empty: the GPU transform drops them (id -1) and the other ids equal Fingerprint64 %
    1000 of the raw bytes; the tower matches the oracle from those raw rows."""
    dense, strings, labels = M.synthetic_batch(B, 7, DEV, empty_fraction=0.25)
    ids, _ = M.transform(DEV)(dense, strings)
    host = strings.cpu().numpy()
    raw = [[bytes(host[j, b]).rstrip(b"\0") for b in range(B)] for j in range(M.FIELDS)]
    want = O.ids_from_raw(raw)
    assert torch.equal(ids.cpu().long(), want) and int((want == -1).sum()) > 0
    flat = M.initial_params(3, DEV)
    dense = dense / 1e4
    out = M.deepctr_deepfm_tower(ids, dense, labels, flat)
    O.check(out, O.reference(want, dense, labels, flat), n_sm=_n_sm(), label="raw B=%d" % B)


def test_mutations_are_caught():
    B = 4096
    dense, strings, labels = M.synthetic_batch(B, 9, DEV)
    dense = dense / 1e4
    ids, _ = M.transform(DEV)(dense, strings)
    host = strings.cpu().numpy()
    raw = [[bytes(host[j, b]).rstrip(b"\0") for b in range(B)] for j in range(M.FIELDS)]
    _, _, _, flat = _inputs(B, "uniform", 4)
    got = M.deepctr_deepfm_tower(ids, dense, labels, flat)
    ref = O.reference(ids, dense, labels, flat)
    assert not O.caught_by(got, ref, n_sm=_n_sm())
    muts = O.mutations(ids, dense, labels, flat, raw)
    assert set(muts) == set(O.MUTATIONS)
    for name, mut in muts.items():
        if name not in O.SATURATED_MUTATIONS:
            assert O.caught_by(mut, ref, n_sm=_n_sm()), name
    M.flat_views(flat)[M.BIAS_NAME].fill_(100.0)  # every logit near +100 with every label 1
    labels = torch.ones_like(labels)
    got = M.deepctr_deepfm_tower(ids, dense, labels, flat)
    ref = O.reference(ids, dense, labels, flat)
    assert not O.caught_by(got, ref, n_sm=_n_sm())
    for name, mut in O.mutations(ids, dense, labels, flat, names=O.SATURATED_MUTATIONS).items():
        assert O.caught_by(mut, ref, n_sm=_n_sm()), name


def test_deterministic_and_graph_replay():
    B = 65536
    ids, dense, labels, flat = _inputs(B, "empty", 9)
    call = M.DeepctrDeepfmCall(B, DEV)
    bufs = [call.loss, call.logits, call.grads]
    call.launch(ids, dense, labels, flat)
    first = [b.clone() for b in bufs]
    call.launch(ids, dense, labels, flat)
    for a, b in zip(first, bufs):
        assert torch.equal(a, b)
    for b in bufs:
        b.fill_(float("nan"))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call.launch(ids, dense, labels, flat)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(first, bufs):
            assert torch.equal(a, b)


def test_refusals():
    B = 64
    ids, dense, labels, flat = _inputs(B, "uniform", 1)
    with pytest.raises(ValueError, match="ids must be"):
        M.deepctr_deepfm_tower(ids.long(), dense, labels, flat)
    with pytest.raises(ValueError, match="dense must be"):
        M.deepctr_deepfm_tower(ids, dense[:12].contiguous(), labels, flat)
    with pytest.raises(ValueError, match="labels must be"):
        M.deepctr_deepfm_tower(ids, dense, labels.double(), flat)
    with pytest.raises(ValueError, match="params must be"):
        M.deepctr_deepfm_tower(ids, dense, labels, flat[:-1])
    with pytest.raises(ValueError, match="batch size"):
        M.DeepctrDeepfmCall(0, DEV)
    with pytest.raises(ValueError, match="batch size"):
        M.DeepctrDeepfmCall(4194305, DEV)
    with pytest.raises(ValueError, match="16-byte aligned"):
        call = M.DeepctrDeepfmCall(B, DEV)
        call.launch(ids, dense, labels, torch.zeros(M.N_PARAMS + 1, device=DEV)[1:])
    bad = ids.clone()
    bad[3, 5] = 1000
    bad[7, 9] = -2
    bad[8, 9] = -1  # absent, not an error
    with pytest.raises(ValueError, match="2 deepctr DeepFM ids outside"):
        M.deepctr_deepfm_tower(bad, dense, labels, flat)
    bad[3, 5] = bad[7, 9] = -1  # an out-of-range id is read as absent
    want = M.deepctr_deepfm_tower(bad, dense, labels, flat)
    bad[3, 5], bad[7, 9] = 1000, -2
    call = M.DeepctrDeepfmCall(B, DEV)
    call.launch(bad, dense, labels, flat)
    assert torch.equal(call.grads, want["grads"]) and torch.equal(call.logits, want["logits"])
    lt, la = M.optimizers()[0]
    dt, da = M.optimizers()[1]
    with pytest.raises(ValueError, match="sync-SGD"):
        M.DeepctrDeepfmEngine(PSGroup(1, dt, da, device=0), PSGroup(1, lt, la, device=0, use_async=False), B)
    with pytest.raises(ValueError, match="lr_staleness_modulation"):
        M.DeepctrDeepfmEngine(PSGroup(1, dt, da, device=0, lr_staleness_modulation=True), PSGroup(1, lt, la, device=0),
                              B)
    eng = M.DeepctrDeepfmEngine(PSGroup(1, dt, da, device=0), PSGroup(1, lt, la, device=0), B)
    d, strings, lab = M.synthetic_batch(B, 3, DEV)
    with pytest.raises(ValueError, match="strings must be"):
        eng.step(d, strings.int(), lab)
    with pytest.raises(ValueError, match="schedule"):
        eng.set_lr_schedule(object())


# As test_gpu_deepctr_wdl.py: r = ||got - ref|| / ||1xTF32 - ref|| over the elements one contraction kind feeds, on
# single-tile batches, where no ReLU mask of the oracle sits within fp32 noise of zero.
@pytest.mark.parametrize("B", [33, 64])
def test_contractions_are_3xtf32(B):
    ids, dense, labels, flat = _inputs(B, "uniform", 21)
    out = M.deepctr_deepfm_tower(ids, dense, labels, flat)
    ref = O.reference(ids, dense, labels, flat)
    touched = torch.zeros((M.FIELDS, M.ROWS), dtype=torch.bool, device=DEV)
    touched[torch.arange(M.FIELDS, device=DEV).unsqueeze(1).expand_as(ids), ids.long()] = True
    emb_rows = torch.zeros(M.N_PARAMS, dtype=torch.bool, device=DEV)
    emb_rows[:O.O_DNN] = touched.unsqueeze(2).expand(-1, -1, M.DIM).reshape(-1)
    weights = torch.zeros(M.N_PARAMS, dtype=torch.bool, device=DEV)
    for n in ("dnn/dnn/kernel0:0", "dnn/dnn/kernel1:0", "dnn/dnn/kernel2:0"):
        weights[M.OFFSETS[n]:M.OFFSETS[n] + int(np.prod(dict(M.PARAMS)[n]))] = True
    checks = [("forward", "logits", None), ("data", "grads", emb_rows), ("weight", "grads", weights)]
    rs = {}
    for kind, fam, sel in checks:
        emu = O.reference(ids, dense, labels, flat, contraction={kind: "1x"})
        rs[kind] = tf32.ratio(out[fam], ref[fam], emu[fam], sel)
    print("B=%d ||got - ref|| / ||1xTF32 - ref||: %s" % (B, rs))
    assert all(r <= tf32.R_MAX for r in rs.values()), (B, rs)


# ---------------------------------------------------------------------------------------------------- engine
def _data(B, n, seed):
    return [(d / 1e4, s, y) for d, s, y in (M.synthetic_batch(B, seed + k, DEV) for k in range(n))]


def _groups(n_shards):
    (lt, la), (dt, da) = M.optimizers()
    return PSGroup(n_shards, dt, da, device=0), PSGroup(n_shards, lt, la, device=0)


class _Oracle:
    """Every parameter in float64 with its TF1 optimizer state, stepped by the engine's gradients."""

    def __init__(self, dnn, lin, eng):
        state = {**dnn.pull_dense(M.DNN_NAMES), **lin.pull_dense(M.LINEAR_NAMES)}
        self.p = {n: state[n].double() for n in M.NAMES}
        self.acc = {n: O.adagrad_init(self.p[n]) for n in M.DNN_NAMES}
        self.ftrl = {n: O.ftrl_init(self.p[n]) for n in M.LINEAR_NAMES}

    def step(self, grads):
        g = {n: v.double() for n, v in M.flat_views(grads).items()}
        for n in M.DNN_NAMES:
            self.p[n], self.acc[n] = O.adagrad_step(self.p[n], self.acc[n], g[n])
        for n in M.LINEAR_NAMES:
            a, li = self.ftrl[n]
            self.p[n], a, li = O.ftrl_step(self.p[n], a, li, g[n])
            self.ftrl[n] = (a, li)

    def compare(self, dnn, lin):
        state = {**dnn.pull_dense(M.DNN_NAMES), **lin.pull_dense(M.LINEAR_NAMES)}
        for n in M.NAMES:
            torch.testing.assert_close(state[n].double(), self.p[n], rtol=2e-5, atol=1e-7, msg=n)
        for n in M.DNN_NAMES:
            torch.testing.assert_close(dnn.slot_dense(n, 1).double(), self.acc[n], rtol=1e-5, atol=1e-9, msg=n)
        for n in M.LINEAR_NAMES:
            for k in (0, 1):
                torch.testing.assert_close(lin.slot_dense(n, k + 1).double(), self.ftrl[n][k], rtol=1e-4, atol=1e-7,
                                           msg=(n, k))


@pytest.mark.parametrize("n_shards", [1, 3])
def test_engine_matches_oracle(n_shards):
    B, steps = 300, 5
    dnn, lin = _groups(n_shards)
    eng = M.DeepctrDeepfmEngine(dnn, lin, B, seed=3)
    for n in M.LINEAR_NAMES:  # FTRL's initial accumulator reaches the dense parameters' slot
        assert bool((lin.slot_dense(n, 1) == 0.1).all()) and bool((lin.slot_dense(n, 2) == 0).all())
    for n in M.DNN_NAMES:
        assert bool((dnn.slot_dense(n, 1) == np.float32(0.1)).all())
    orc = _Oracle(dnn, lin, eng)
    for step, (dense, strings, labels) in enumerate(_data(B, steps, 100)):
        loss = eng.step(dense, strings, labels)
        torch.cuda.synchronize()
        eng.check()
        ref = O.reference(eng.ids, dense, labels, eng.flat)
        O.check(eng.tower.outputs(), ref, n_sm=_n_sm(), label="step %d" % step)
        assert abs(float(loss) - float(ref["loss"])) <= 1e-5 * float(ref["M"]["loss"])
        orc.step(eng.tower.grads)
    torch.cuda.synchronize()
    orc.compare(dnn, lin)
    assert [v for v, _, _ in dnn.snapshot()] == [steps] * n_shards
    assert [v for v, _, _ in lin.snapshot()] == [steps] * n_shards


def test_untouched_rows():
    """Embedding rows no batch read, and their Adagrad accumulators, keep their initial bits; a linear row read by the
    first batch only gets g = lambda w at the next step and moves by FTRL on it; linear rows never read stay 0."""
    B = 64
    dnn, lin = _groups(1)
    eng = M.DeepctrDeepfmEngine(dnn, lin, B, seed=2)
    before = dnn.pull_dense(M.EMB_NAMES)
    data = _data(B, 2, 5)
    seen = torch.zeros((M.FIELDS, M.ROWS), dtype=torch.bool, device=DEV)
    states, grads = [], []
    for dense, strings, labels in data:
        eng.step(dense, strings, labels)
        torch.cuda.synchronize()
        ids = eng.ids.long()
        keep = ids >= 0
        seen[torch.arange(M.FIELDS, device=DEV).unsqueeze(1).expand_as(ids)[keep], ids[keep]] = True
        n = M.LIN_NAMES[0]
        states.append((lin.pull_dense([n])[n][:, 0], lin.slot_dense(n, 1)[:, 0], lin.slot_dense(n, 2)[:, 0],
                       ids[0].clone()))
        grads.append(M.flat_views(eng.tower.grads)[n][:, 0].clone())
    after = dnn.pull_dense(M.EMB_NAMES)
    lin_after = lin.pull_dense(M.LIN_NAMES)
    for j in range(M.FIELDS):
        n = M.EMB_NAMES[j]
        assert torch.equal(after[n][~seen[j]], before[n][~seen[j]])
        assert bool((dnn.slot_dense(n, 1)[~seen[j]] == np.float32(0.1)).all())
        assert int(torch.count_nonzero(lin_after[M.LIN_NAMES[j]][~seen[j]])) == 0
    (w1, a1, l1, ids1), (w2, _, _, ids2) = states
    once = torch.zeros(M.ROWS, dtype=torch.bool, device=DEV)
    once[ids1[ids1 >= 0]] = True
    once[ids2[ids2 >= 0]] = False
    once &= w1 != 0  # a row whose occurrences' dz cancel to 0 in fp32 never moved
    assert int(once.sum()) > 0
    g = grads[1][once]
    torch.testing.assert_close(g.double(), 1e-5 * w1[once].double(), rtol=1e-6, atol=0)
    want, _, _ = O.ftrl_step(w1[once].double(), a1[once].double(), l1[once].double(), g.double())
    torch.testing.assert_close(w2[once].double(), want, rtol=1e-5, atol=1e-12)


def test_replay_equals_step():
    B = 200
    ga, la = _groups(2)
    gb, lb = _groups(2)
    ea = M.DeepctrDeepfmEngine(ga, la, B, seed=4)
    eb = M.DeepctrDeepfmEngine(gb, lb, B, seed=4)
    for dense, strings, labels in _data(B, 4, 50):
        ea.step(dense, strings, labels)
        eb.replay(dense, strings, labels)
    torch.cuda.synchronize()
    for (x, y), names in (((ga, gb), M.DNN_NAMES), ((la, lb), M.LINEAR_NAMES)):
        sa, sb = x.pull_dense(names), y.pull_dense(names)
        for n in names:
            assert torch.equal(sa[n], sb[n]), n


def test_evaluate_matches_oracle_forward():
    B = 500
    dnn, lin = _groups(1)
    eng = M.DeepctrDeepfmEngine(dnn, lin, B, seed=6)
    metrics = EvaluationMetrics(M.eval_metrics_fn())
    zs, labs = [], []
    for dense, strings, labels in _data(B, 2, 900):
        logits = eng.evaluate(dense, strings, labels, metrics)
        torch.cuda.synchronize()
        ref = O.reference(eng.ids, dense, labels, eng.flat)
        O.check({"logits": logits}, ref, n_sm=_n_sm())
        zs.append(ref["logits"])
        labs.append(labels.double())
    got = metrics.get_evaluation_summary()
    z, y = torch.cat(zs), torch.cat(labs)
    p = torch.sigmoid(z)
    assert got["logits"]["LogLoss"] == pytest.approx(float((z.clamp(min=0) - z * y + torch.log1p(torch.exp(-z.abs())))
                                                           .mean()), rel=1e-5)
    assert got["probs"]["prediction/mean"] == pytest.approx(float(p.mean()), rel=1e-5)
    assert got["probs"]["label/mean"] == pytest.approx(float(y.mean()), rel=1e-12)
    ref_metrics = EvaluationMetrics({"probs": {"AUC": M.eval_metrics_fn()["probs"]["AUC"]}})
    ref_metrics.update_evaluation_metrics({"probs": p.float()}, y.float())
    assert abs(got["probs"]["AUC"] - ref_metrics.get_evaluation_summary()["probs"]["AUC"]) < 1e-3
    assert [v for v, _, _ in dnn.snapshot()] == [0] and [v for v, _, _ in lin.snapshot()] == [0]


def _four_workers(B):
    dnn, lin = _groups(2)
    engines = [M.DeepctrDeepfmEngine(dnn, lin, B, seed=5, register=(w == 0)) for w in range(4)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(4)]
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.capture()
    torch.cuda.synchronize()
    return dnn, lin, engines, streams


def test_four_workers_concurrent():
    B, steps = 256, 10
    dnn, lin, engines, streams = _four_workers(B)
    data = [_data(B, 2, 1000 * (w + 1)) for w in range(4)]
    torch.cuda.synchronize()
    errors = []

    def run(w):
        try:
            with torch.cuda.stream(streams[w]):
                for s in range(steps):
                    engines[w].replay(*data[w][s % 2])
            streams[w].synchronize()
        except Exception as e:  # noqa: BLE001
            errors.append((w, repr(e)))

    threads = [threading.Thread(target=run, args=(w,)) for w in range(4)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors
    torch.cuda.synchronize()
    assert [v for v, _, _ in dnn.snapshot()] == [4 * steps] * 2
    assert [v for v, _, _ in lin.snapshot()] == [4 * steps] * 2
    for e in engines:
        e.check()


def test_four_workers_serialised_match_oracle():
    B, rounds = 256, 2
    dnn, lin, engines, streams = _four_workers(B)
    orc = _Oracle(dnn, lin, engines[0])
    data = [_data(B, rounds, 1000 * (w + 1)) for w in range(4)]
    for r in range(rounds):
        for w in range(4):
            with torch.cuda.stream(streams[w]):
                engines[w].replay(*data[w][r])
            streams[w].synchronize()
            orc.step(engines[w].tower.grads)
    orc.compare(dnn, lin)
