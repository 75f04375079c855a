"""Learning-rate schedules evaluated by the push on the device (b200ps_set_lr_schedule): the lr every push applies
against oracle/lr_schedule_oracle.py, the optimizers that fold the lr, the graphed trainer, the engines, views,
checkpoints and the ABI's refusals.

The applied lr is observed exactly through SGD on dense parameters reset to 0 before each push with gradient 1:
0 - lr * 1 = -lr."""
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch

from elasticdl_b200 import callbacks as cb
from oracle import lr_schedule_oracle as orc
from oracle import ps_oracle as O

pytestmark = pytest.mark.gpu
F = np.float32
SGD = ("SGD", "learning_rate=0.01;momentum=0.0;nesterov=false;")
ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")

# (device schedule, float64 oracle of x)
CASES = {
    "piecewise": (cb.PiecewiseConstantDecay([2, 5, 9.5], [0.1, 0.05, 0.02, 0.001]),
                  lambda x: orc.piecewise_constant(x, [2, 5, 9.5], [0.1, 0.05, 0.02, 0.001])),
    "piecewise_negative": (cb.PiecewiseConstantDecay([3], [0.2, -1.0]),
                           lambda x: orc.piecewise_constant(x, [3], [0.2, -1.0])),
    "exponential": (cb.ExponentialDecay(0.1, 3, 0.9), lambda x: orc.exponential(x, 0.1, 3, 0.9)),
    "exponential_staircase": (cb.ExponentialDecay(0.1, 2.5, 0.5, staircase=True),
                              lambda x: orc.exponential(x, 0.1, 2.5, 0.5, True)),
    "inverse_time": (cb.InverseTimeDecay(0.2, 3, 0.7), lambda x: orc.inverse_time(x, 0.2, 3, 0.7)),
    "inverse_time_staircase": (cb.InverseTimeDecay(0.2, 2, 1.5, staircase=True),
                               lambda x: orc.inverse_time(x, 0.2, 2, 1.5, True)),
    "polynomial": (cb.PolynomialDecay(0.1, 6), lambda x: orc.polynomial(x, 0.1, 6)),
    "polynomial_to_zero": (cb.PolynomialDecay(0.1, 5, end_learning_rate=0.0),  # 0 from x = 5: the fallback
                           lambda x: orc.polynomial(x, 0.1, 5, 0.0)),
    "polynomial_cycle": (cb.PolynomialDecay(0.1, 4, 0.01, power=0.5, cycle=True),
                         lambda x: orc.polynomial(x, 0.1, 4, 0.01, 0.5, True)),
}


def _probe_group(n_shards, opt=SGD, **kw):
    from elasticdl_b200.ps import PSGroup

    g = PSGroup(n_shards, *opt, device=0, **kw)
    for s in range(n_shards):
        g.register_dense("w%d" % s, (4,), s)
    g.commit()
    return g


def _push_and_read(g, request_lr=0.5, versions=None):
    """One push of gradient 1 on every shard's zeroed probe; returns the lr each shard applied."""
    n = g.n_shards
    zero = torch.zeros(4, device="cuda")
    ones = torch.ones(4, device="cuda")
    g.set_dense([("w%d" % s, zero) for s in range(n)])
    g.push_begin(request_lr, versions if versions is not None else [0] * n)
    g.push_dense([(g.lookup("w%d" % s)[0], 0, None, None, ones) for s in range(n)])
    g.push_end()
    out = g.pull_dense(["w%d" % s for s in range(n)])
    return [float(-out["w%d" % s][0].item()) for s in range(n)]


def _expected(ref, versions, opt_lr=0.01, staleness=1):
    v64 = ref(orc.schedule_argument(versions))
    if np.float32(v64) <= 0:
        return {orc.effective_lr(v64, opt_lr, staleness)}
    return {orc.effective_lr(f, opt_lr, staleness) for f in orc.acceptable_f32(v64)}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("n_shards", [1, 3])
def test_applied_lr_equals_oracle(case, n_shards):
    sched, ref = CASES[case]
    g = _probe_group(n_shards)
    for s in range(n_shards):  # different versions per shard: the schedule takes the largest
        g.set_shard_state(s, version=2 * s)
    g.set_lr_schedule(sched)
    for _ in range(14):
        versions = [v for v, _, _ in g.snapshot()]
        got = _push_and_read(g)
        want = _expected(ref, versions)
        assert all(x in want for x in got), (case, versions, got, want)
    g.set_lr_schedule(None)  # the request's lr again
    assert _push_and_read(g, 0.25) == [0.25] * n_shards
    g.close()


def test_staleness_modulation_divides_the_scheduled_lr():
    sched, ref = CASES["exponential"]
    g = _probe_group(2, lr_staleness_modulation=True)
    g.set_lr_schedule(sched)
    for step in range(8):
        versions = [v for v, _, _ in g.snapshot()]
        pulled = [max(v - step % 3, 0) for v in versions]  # 0, 1 or 2 versions stale
        got = _push_and_read(g, 0.5, pulled)
        for s in range(2):
            staleness = versions[s] - pulled[s]
            assert got[s] in _expected(ref, versions, staleness=max(staleness, 1)), (step, s, got)
    g.close()


def test_bump_step_and_single_shard_push_with_a_schedule():
    sched, ref = CASES["piecewise"]
    g = _probe_group(3)
    g.set_lr_schedule(sched)
    g.bump_step()
    assert [st for _, st, _ in g.snapshot()] == [1, 1, 1]
    g.set_shard_state(2, version=7)
    lib = g.lib
    ones = torch.ones(4, device="cuda")
    g.set_dense([("w1", torch.zeros(4, device="cuda"))])
    from elasticdl_b200._lib import check

    check(lib.b200ps_push_begin_shard(g._h, 1, ctypes.c_float(0.5), None, g._stream()))
    g.push_dense([(g.lookup("w1")[0], 0, None, None, ones)])
    check(lib.b200ps_push_end_shard(g._h, 1, g._stream()))
    got = -float(g.pull_dense(["w1"])["w1"][0].item())
    assert got in _expected(ref, [0, 0, 7])  # every shard's version counts, the pushed shard's included
    assert [v for v, _, _ in g.snapshot()] == [0, 1, 7]
    g.close()


# ------------------------------------------------------------------ the optimizers that fold the lr
FOLD_OPTS = {
    "adam": ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;"),
    "ftrl": ("Ftrl", "learning_rate=0.1;initial_accumulator_value=0.1;l1_regularization_strength=0.01;"
                     "l2_regularization_strength=0.02;l2_shrinkage_regularization_strength=0.0;beta=0.5;"),
    "adamax": ("Adamax", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;"),
    "nadam": ("Nadam", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;"),
}


@pytest.mark.parametrize("opt", list(FOLD_OPTS))
def test_folding_optimizers_match_oracle_fed_the_scheduled_lr(opt):
    from oracle import keras_optim_oracle as K
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from tests.test_gpu_parity import _grads, _setup_model

    ot, oa = FOLD_OPTS[opt]
    n_shards = 2
    base = float(oa.split(";")[0].split("=")[1])
    sched = cb.ExponentialDecay(2 * base, 2, 0.7)
    group = PSGroup(n_shards, ot, oa, device=0)
    client = PSClient(group)
    Srv = K.KerasOracleServer if opt in ("adamax", "nadam") else O.OracleServer
    oc = O.OraclePSClient([Srv(i, ot, oa, num_ps=n_shards) for i in range(n_shards)])
    rng = np.random.RandomState(zlib.crc32(repr(("sched", opt)).encode()))
    dims = (1, 8)
    dense = _setup_model(client, oc, rng, dims)
    group.set_lr_schedule(sched)
    versions = [0] * n_shards
    for step in range(6):
        (grads, edl), (ograds, oedl) = _grads(rng, dims, step, False)
        lr = float(np.float32(orc.exponential(orc.schedule_argument(versions), 2 * base, 2, 0.7)))
        acc, v = client.push_gradients(grads, edl, 0.123, versions)  # the request's lr is ignored
        oacc, ov = oc.push_gradients(ograds, oedl, lr, list(versions))
        assert (acc, v) == (oacc, ov) == (True, step + 1)
        versions = [v] * n_shards
    for name in dense:
        srv = oc.servers[oc.parameter_to_ps[name]]
        assert np.array_equal(group.pull_dense([name])[name].cpu().numpy(), srv.dense[name]), name
        for k, sn in enumerate(srv.opt.slot_names):
            assert np.array_equal(group.slot_dense(name, k + 1).cpu().numpy(), srv.opt.dense_slots[sn][name]), name
    ids = np.arange(500, dtype=np.int64)
    for d in dims:
        name = "e%d" % d
        got = client.pull_embedding_vectors(name, ids)
        for s in oc.servers:
            m = ids % n_shards == s.id
            touched = np.isin(ids[m], s.tables[name].keys())
            assert np.array_equal(got[m][touched], s.tables[name].get(ids[m][touched])), name
    group.close()


# ------------------------------------------------------------------ the graphed drop-in trainer
def test_graphed_trainer_keeps_one_capture_under_a_per_step_schedule():
    import types

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer
    from elasticdl_b200.workloads.deepfm import DeepFMLayersModel

    rows, B, steps = [7, 300, 5000, 40, 1200], 512, 12
    sched = cb.ExponentialDecay(0.01, 2, 0.8)
    gen = torch.Generator().manual_seed(5)
    batches = []
    for _ in range(steps):
        ids = torch.stack([torch.randint(0, r, (B,), generator=gen) for r in rows]).cuda()
        dense = torch.randn(B, 13, generator=gen).cuda()
        labels = (torch.rand(B, generator=gen) < 0.3).float().cuda()
        batches.append((DeepFMLayersModel.features_of(ids, dense), labels))

    def run(graphed):
        torch.manual_seed(3)
        model = DeepFMLayersModel(rows, lr=0.01, initializer="uniform").cuda()
        group = PSGroup(1, *ADAM, device=0, seed=11)
        client = PSClient(group)
        client.dense_output = "torch"
        trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
            get_model_steps=1, batched_embedding_lookups=True, cuda_graph=graphed, cuda_graph_warmup=2))
        schedule = sched if graphed else (lambda v: sched(v))  # eager: the same schedule as a host callable
        out = trainer.train_loop(batches, callbacks=[cb.LearningRateScheduler(schedule)])
        assert [v for v, _ in out] == list(range(1, steps + 1))
        if graphed:
            assert trainer.graph_fallback_reason is None, trainer.graph_fallback_reason
            assert isinstance(trainer._graph_state, dict) and trainer._graph_state["recaptures"] == 0
            assert group.lr_schedule is sched
        else:
            assert group.lr_schedule is None
        tabs = {}
        for g, r in enumerate(rows):
            for fam in ("deep", "wide"):
                name = "%s_%d/embeddings:0" % (fam, g)
                tabs[name] = client.pull_embedding_vectors(name, torch.arange(r).cuda()).cpu()
        params, _ = client.pull_dense_parameters([0], [-1])
        params = {k: v.cpu() for k, v in params.items()}
        group.close()
        return [float(l) for _, l in out], tabs, params

    l_g, t_g, p_g = run(True)
    l_e, t_e, p_e = run(False)
    assert np.allclose(l_g, l_e, rtol=1e-5, atol=1e-6), (l_g, l_e)
    for name in t_e:
        assert torch.allclose(t_g[name], t_e[name], rtol=1e-5, atol=1e-7), name
    for name in p_e:
        assert torch.allclose(p_g[name], p_e[name], rtol=1e-5, atol=1e-7), name


# ------------------------------------------------------------------ engines
def _census_batches(B, n):
    from elasticdl_b200.workloads.census_features import synthetic_raw_batch

    out = []
    for s in range(n):
        numeric, strings, _, _ = synthetic_raw_batch(B, 60 + s, torch.device("cuda", 0))
        labels = (torch.arange(B, device="cuda") % 3 == s % 3).float()
        out.append((numeric, strings, labels))
    return out


def _frappe_batches(B, n):
    from elasticdl_b200.workloads.frappe import synthetic_frappe_batch

    return [synthetic_frappe_batch(B, 80 + s, torch.device("cuda", 0)) for s in range(n)]


@pytest.mark.parametrize("model", ["census", "frappe"])
def test_engine_replays_a_schedule_from_one_capture(model):
    """The schedule crosses its boundary at the fourth push.  One capture replays every step and leaves the same
    parameters as eager steps given each step's scheduled lr through set_lr, up to the order of the atomic
    row-gradient sums."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads import census as C
    from elasticdl_b200.workloads import frappe as FR

    sched = cb.PiecewiseConstantDecay([2], [0.3, 0.1])
    B, steps = 256, 6
    if model == "census":
        data = _census_batches(B, steps)
        make = lambda g, **kw: C.CensusWideDeepEngine(g, B, 0.2, seed=3, **kw)  # noqa: E731
    else:
        data = _frappe_batches(B, steps)
        make = lambda g, **kw: FR.FrappeDeepFMEngine(g, B, 0.2, input_dim=FR.INPUT_DIM, seed=3, **kw)  # noqa: E731
    ga, gb = (PSGroup(2, *SGD, device=0) for _ in range(2))
    ea = make(ga, lr_schedule=sched)
    eb = make(gb)
    with pytest.raises(ValueError, match="schedule"):
        ea.set_lr(0.5)
    captures = 0
    for i, batch in enumerate(data):
        before = ea.graph
        ea.replay(*batch)
        captures += ea.graph is not before
        eb.set_lr(sched(i - 1))  # the version a push begins on is i: x = i - 1
        eb.step(*batch)
    torch.cuda.synchronize()
    ea.check()
    eb.check()
    assert captures == 1
    names = [n for n, (_, _, is_dense, _) in ga.tables.items() if is_dense]
    sa, sb = ga.pull_dense(names), gb.pull_dense(names)
    for n in names:
        assert torch.allclose(sa[n], sb[n], rtol=1e-5, atol=1e-6), (n, float((sa[n] - sb[n]).abs().max()))
    ga.close()
    gb.close()


def test_deepfm_lookahead_graphs_apply_the_schedule():
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, HostFeeder, synthetic_batch
    from tests.test_gpu_layer_trainer import _engine_state

    rows, B, steps = [11, 700, 5000, 9, 64], 256, 6
    sched = cb.ExponentialDecay(0.01, 1, 0.6)
    batches = [synthetic_batch(B, 40 + i, torch.device("cuda", 0), "zipf", group_rows=rows) for i in range(steps)]
    results = []
    for mode in ("plain", "ahead"):
        group = PSGroup(2, *ADAM, device=0)
        losses = []
        if mode == "plain":  # the pushed lr set by hand to the schedule's value at x = i - 1
            eng = DeepFMPSEngine(group, B, group_rows=rows)
            for i, (ids, dense, labels) in enumerate(batches):
                eng.lr = float(np.float32(sched(i - 1)))
                losses.append(float(eng.step(ids, dense, labels)))
        else:
            eng = DeepFMPSEngine(group, B, group_rows=rows, lr=0.5, lr_schedule=sched)
            feeder = HostFeeder(eng, 3, lookahead=True)
            host = [tuple(t.cpu().pin_memory() for t in b) for b in batches]
            feeder.submit(*host[0])
            feeder.submit(*host[1])
            for i in range(steps):
                if i + 2 < steps:
                    feeder.submit(*host[i + 2])
                losses.append(float(feeder.run_next()))
        group.check()
        results.append((losses, _engine_state(group, eng, rows)))
        group.close()
    (l0, s0), (l1, s1) = results
    assert np.allclose(l0, l1, rtol=1e-5, atol=0), (l0, l1)
    for a, b in zip(s0, s1):  # the tolerance test_engine_lookahead_pipeline_matches_plain_steps uses
        assert np.allclose(a, b, rtol=0, atol=2e-4), float(np.abs(a - b).max())


# ------------------------------------------------------------------ views and checkpoints
def test_each_view_applies_its_own_schedule():
    sched, ref = CASES["inverse_time"]
    g = _probe_group(2)
    view = g.clone_view()
    assert view.lr_schedule is None
    view.set_lr_schedule(sched)
    for step in range(8):
        versions = [v for v, _, _ in g.snapshot()]
        if step % 2:
            assert _push_and_read(g, 0.25) == [0.25, 0.25]
        else:
            got = _push_and_read(view, 0.25)
            assert all(x in _expected(ref, versions) for x in got), (step, got)
    assert g.lr_schedule is None
    view.close()
    g.close()


def test_checkpoint_restore_continues_the_schedule(tmp_path):
    from elasticdl_b200.ps import checkpoint as ck
    from elasticdl_b200.worker.ps_client import PSClient

    sched, ref = CASES["exponential"]
    g = _probe_group(2)
    g.set_lr_schedule(sched)
    for _ in range(5):
        _push_and_read(g)
    vdir = ck.save(g, str(tmp_path), keep_checkpoint_max=1, dense_names=[])
    g.close()
    g2 = _probe_group(2)
    assert ck.load(g2, PSClient(g2), vdir) == 5
    g2.set_lr_schedule(sched)
    got = _push_and_read(g2)
    assert all(x in _expected(ref, [5, 5]) for x in got), got
    assert got[0] != float(np.float32(sched(0)))
    g2.close()


def test_sync_group_refuses_a_schedule():
    from elasticdl_b200.ps import PSGroup

    g = PSGroup(1, *SGD, device=0, use_async=False)
    with pytest.raises(ValueError, match="async"):
        g.set_lr_schedule(CASES["exponential"][0])
    g.set_lr_schedule(None)
    g.close()


# ------------------------------------------------------------------ ABI refusals
def _raw(**kw):
    from elasticdl_b200._lib import LrSchedule

    s = LrSchedule(kind=2, initial_learning_rate=0.1, decay_steps=2.0, decay_rate=0.5)
    for k, v in kw.items():
        setattr(s, k, v)
    return s


def _piecewise(n, bounds, values):
    from elasticdl_b200._lib import LrSchedule

    s = LrSchedule(kind=1, n_boundaries=n)
    for i, b in enumerate(bounds):
        s.boundaries[i] = b
    for i, v in enumerate(values):
        s.values[i] = v
    return s


REFUSED = [
    (lambda: _raw(kind=0), "unknown learning-rate schedule kind"),
    (lambda: _raw(kind=5), "unknown learning-rate schedule kind"),
    (lambda: _raw(decay_steps=0.0), "decay_steps must be > 0"),
    (lambda: _raw(decay_steps=-1.0), "decay_steps must be > 0"),
    (lambda: _raw(decay_rate=math.nan), "not finite"),
    (lambda: _raw(kind=4, power=math.inf), "not finite"),
    (lambda: _raw(initial_learning_rate=-math.inf), "not finite"),
    (lambda: _piecewise(-1, [], [0.1]), "boundaries"),
    (lambda: _piecewise(33, list(range(32)), [0.1] * 33), "boundaries"),
    (lambda: _piecewise(2, [3, 3], [0.1, 0.2, 0.3]), "strictly increasing"),
    (lambda: _piecewise(1, [math.nan], [0.1, 0.2]), "not finite"),
    (lambda: _piecewise(1, [1], [0.1, math.inf]), "not finite"),
]


@pytest.mark.parametrize("i", range(len(REFUSED)))
def test_abi_refuses_bad_schedules_and_launches_nothing(i):
    from elasticdl_b200 import _lib

    make, msg = REFUSED[i]
    g = _probe_group(1)
    g.set_lr_schedule(cb.PiecewiseConstantDecay([], [0.125]))
    launches = g.launch_count
    rc = g.lib.b200ps_set_lr_schedule(g._h, ctypes.byref(make()))
    assert rc == _lib.EINVAL
    assert msg in g.lib.b200ps_last_error().decode()
    assert g.launch_count == launches
    assert _push_and_read(g) == [0.125]  # the installed schedule is unchanged
    g.close()


# ------------------------------------------------------------------ the eager trainer
class _OneParam(torch.nn.Module):
    """loss = sum(w): every push carries gradient 1 for each entry of w, so w on the PS moves by -lr per push."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(4))
        self.optimizer = torch.optim.SGD([self.w], lr=0.5)
        self.loss = lambda labels, out: out

    def forward(self, features):
        return self.w.sum() + 0.0 * features.sum()


class _PSValue(cb.Callback):
    def __init__(self, group):
        self.group, self.seen = group, []

    def on_train_batch_begin(self, batch, logs=None):
        if "w" in self.group.tables:
            self.seen.append(float(self.group.pull_dense(["w"])["w"][0].item()))


@pytest.mark.parametrize("case", ["exponential", "polynomial_to_zero"])
def test_eager_trainer_staleness_and_fallback_with_a_schedule(case):
    """get_model_steps=3 with lr staleness modulation (an eager job): the k-th minibatch after a pull pushes the
    versions of that pull, k versions stale, and the PS divides the scheduled lr by k.  polynomial_to_zero reaches
    0 at x = 5, from where the PS applies its optimizer's own lr (0.01)."""
    import types

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    sched, ref = CASES[case]
    model = _OneParam().cuda()
    group = PSGroup(1, *SGD, device=0, lr_staleness_modulation=True)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
        get_model_steps=3, batched_embedding_lookups=True, cuda_graph=True))
    probe = _PSValue(group)
    steps = 10
    x = torch.zeros(2, device="cuda")
    out = trainer.train_loop([(x, x)] * steps, callbacks=[probe, cb.LearningRateScheduler(sched)])
    assert [v for v, _ in out] == list(range(1, steps + 1))
    assert trainer.graph_fallback_reason is not None and group.lr_schedule is sched
    seen = probe.seen + [float(group.pull_dense(["w"])["w"][0].item())]  # w on the PS after each push
    assert len(seen) == steps
    start = 0.0
    for i, after in enumerate(seen):
        want = _expected(ref, [i], staleness=max(i % 3, 1))
        assert any(abs((start - after) - w) <= 1e-6 + 1e-5 * w for w in want), (case, i, start - after, want)
        start = after
    group.close()


def test_sync_group_trainer_keeps_the_schedule_on_the_host():
    """A sync-SGD group has no device schedule: train_loop evaluates a declarative scheduler on the host only, as
    the reference does, and the job trains."""
    import types

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    sched = cb.PiecewiseConstantDecay([1], [0.25, 0.125])
    model = _OneParam().cuda()
    group = PSGroup(1, *SGD, device=0, use_async=False, grads_to_wait=1)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
        get_model_steps=1, batched_embedding_lookups=True, cuda_graph=False))
    x = torch.zeros(2, device="cuda")
    out = trainer.train_loop([(x, x)] * 4, callbacks=[cb.LearningRateScheduler(sched)])
    assert all(v is not None for v, _ in out), out
    assert group.lr_schedule is None
    assert model.optimizer.param_groups[0]["lr"] == 0.125  # set from model version 2 before the last minibatch
    group.close()


# ------------------------------------------------------------------ the owner-computes exchange, two ranks
def test_exchange_applies_each_source_ranks_schedule_via_torchrun():
    from tests.test_gpu_layer_trainer import _torchrun_two_ranks

    out = _torchrun_two_ranks("mgpu_lr_schedule_check.py", 29561)
    assert out.returncode == 0 and "mgpu_lr_schedule_check ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]
