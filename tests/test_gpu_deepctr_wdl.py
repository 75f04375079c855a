"""The deepctr WDL tower (csrc/deepctr_wdl_tower.cu, include/b200_deepctr_wdl.h) and DeepctrWdlEngine against the
float64 oracle of oracle/deepctr_wdl_oracle.py.

Kernel level: batches at the tile and grid edges up to 65536, with uniform ids, every sample on one row per table
(a hot row summed over every occurrence), raw dense values large enough to clip p at both ends, and a quarter of
the strings empty; the oracle's mutations; bitwise repeats and graph replay; the refusals; and the 3xTF32
statistic of test_gpu_tensor_core_precision.py for the forward, data and weight contractions.  Engine level: five
SGD and Adam steps on one and three shards against OracleServer fed the engine's gradients, every row compared;
the whole-table update of an untouched row; evaluate; the drop-in trainer over the twin; four graphed workers."""
import threading
import types

import numpy as np
import pytest
import torch

from elasticdl_b200.common.evaluation_utils import EvaluationMetrics
from elasticdl_b200.ps import PSGroup
from elasticdl_b200.workloads import deepctr_wdl as M
from oracle import deepctr_wdl_oracle as O
from oracle import tf32
from oracle.ps_oracle import OracleServer

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
OPTS = {"sgd": ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", 0.1), "adam": M.optimizer()}


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _inputs(B, pattern, seed):
    """ids int32 [26, B], dense [13, B], labels, flat (the initialisers with non-zero linear rows and global bias,
    so that every term of z carries weight)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    if pattern == "one":
        ids = ((torch.arange(M.FIELDS, device=DEV) * 37 + 5) % M.ROWS).to(torch.int32).unsqueeze(1).repeat(1, B)
    else:
        ids = torch.randint(0, M.ROWS, (M.FIELDS, B), generator=g, device=DEV, dtype=torch.int32)
    dense = torch.rand((M.DENSE, B), generator=g, device=DEV) * 2
    if pattern == "clip":  # raw dense values: p clipped at both ends for about half the samples
        dense = dense + (torch.rand(B, generator=g, device=DEV) < 0.5).float() * \
            torch.where(torch.rand(B, generator=g, device=DEV) < 0.5, 300.0, -300.0)
    labels = (torch.rand(B, generator=g, device=DEV) < 0.3).float()
    flat = M.initial_params(seed, DEV)
    v = M.flat_views(flat)
    for n in M.LINEAR_NAMES:
        v[n].copy_(torch.randn(v[n].shape, generator=g, device=DEV) * 0.05)
    for n in M.DEEP_NAMES:
        v[n].mul_(3e3)
    v["prediction_layer/global_bias:0"].fill_(0.2)
    return ids.contiguous(), dense.contiguous(), labels, flat


def _batches():
    n = 64 * _n_sm()
    return [1, 32, 63, 64, 65, n - 1, n, n + 1, 65536]


@pytest.mark.parametrize("pattern", ["uniform", "one", "clip"])
@pytest.mark.parametrize("i", range(9))
def test_tower_matches_oracle(i, pattern):
    B = _batches()[i]
    ids, dense, labels, flat = _inputs(B, pattern, seed=B % 991 + len(pattern))
    out = M.deepctr_wdl_tower(ids, dense, labels, flat)
    ref = O.reference(ids, dense, labels, flat)
    O.check(out, ref, n_sm=_n_sm(), label="B=%d %s" % (B, pattern))
    fwd = M.deepctr_wdl_tower(ids, dense, None, flat, train=False)
    assert torch.equal(fwd["logits"], out["logits"])


@pytest.mark.parametrize("B", [300, 65536])
def test_tower_from_raw_rows_with_empty_strings(B):
    """A quarter of the strings empty: "" hashes to an ordinary bucket (Q30); ids from the GPU transform equal
    Fingerprint64 % 10000 of the raw bytes, and the tower matches the oracle from those raw rows."""
    dense, strings, labels = M.synthetic_batch(B, 7, DEV, empty_fraction=0.25)
    ids, _ = M.transform(DEV)(dense, strings)
    host = strings.cpu().numpy()
    raw = [[bytes(host[j, b]).rstrip(b"\0") for b in range(B)] for j in range(M.FIELDS)]
    want = O.ids_from_raw(raw)
    assert torch.equal(ids.cpu().long(), want)
    flat = M.initial_params(3, DEV)
    dense = dense / 1e4  # away from the clip edge, as _data
    out = M.deepctr_wdl_tower(ids, dense, labels, flat)
    O.check(out, O.reference(want, dense, labels, flat), n_sm=_n_sm(), label="raw B=%d" % B)


def test_mutations_are_caught():
    B = 4096
    dense, strings, labels = M.synthetic_batch(B, 9, DEV)
    dense = dense / 1e4
    ids, _ = M.transform(DEV)(dense, strings)
    host = strings.cpu().numpy()
    raw = [[bytes(host[j, b]).rstrip(b"\0") for b in range(B)] for j in range(M.FIELDS)]
    flat = M.initial_params(4, DEV)
    v = M.flat_views(flat)
    for n in M.LINEAR_NAMES:
        v[n].normal_(0, 0.05)
    v["prediction_layer/global_bias:0"].fill_(0.2)
    got = M.deepctr_wdl_tower(ids, dense, labels, flat)
    ref = O.reference(ids, dense, labels, flat)
    assert not O.caught_by(got, ref, n_sm=_n_sm())
    muts = O.mutations(ids, dense, labels, flat, raw)
    assert set(muts) == set(O.MUTATIONS)
    for name, mut in muts.items():
        if name != "unclipped":
            assert O.caught_by(mut, ref, n_sm=_n_sm()), name
    ids, dense, labels, flat = _inputs(B, "clip", 5)
    ref = O.reference(ids, dense, labels, flat)
    assert O.caught_by(O.mutations(ids, dense, labels, flat, names=("unclipped",))["unclipped"], ref, n_sm=_n_sm())


def test_deterministic_and_graph_replay():
    B = 65536
    ids, dense, labels, flat = _inputs(B, "uniform", 9)
    call = M.DeepctrWdlCall(B, DEV)
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
        M.deepctr_wdl_tower(ids.long(), dense, labels, flat)
    with pytest.raises(ValueError, match="dense must be"):
        M.deepctr_wdl_tower(ids, dense[:12].contiguous(), labels, flat)
    with pytest.raises(ValueError, match="labels must be"):
        M.deepctr_wdl_tower(ids, dense, labels.double(), flat)
    with pytest.raises(ValueError, match="params must be"):
        M.deepctr_wdl_tower(ids, dense, labels, flat[:-1])
    with pytest.raises(ValueError, match="batch size"):
        M.DeepctrWdlCall(0, DEV)
    with pytest.raises(ValueError, match="batch size"):
        M.DeepctrWdlCall(4194305, DEV)
    with pytest.raises(ValueError, match="16-byte aligned"):
        call = M.DeepctrWdlCall(B, DEV)
        call.launch(ids, dense, labels, torch.zeros(M.N_PARAMS + 1, device=DEV)[1:])
    bad = ids.clone()
    bad[3, 5] = 10000
    bad[7, 9] = -1
    with pytest.raises(ValueError, match="2 deepctr WDL ids outside"):
        M.deepctr_wdl_tower(bad, dense, labels, flat)
    opt_type, opt_args, lr = OPTS["sgd"]
    with pytest.raises(ValueError, match="sync-SGD"):
        M.DeepctrWdlEngine(PSGroup(1, opt_type, opt_args, device=0, use_async=False), B, lr)
    with pytest.raises(ValueError, match="lr_staleness_modulation"):
        M.DeepctrWdlEngine(PSGroup(1, opt_type, opt_args, device=0, lr_staleness_modulation=True), B, lr)
    eng = M.DeepctrWdlEngine(PSGroup(1, opt_type, opt_args, device=0), B, lr)
    dense, strings, labels = M.synthetic_batch(B, 3, DEV)
    with pytest.raises(ValueError, match="strings must be"):
        eng.step(dense, strings.int(), labels)
    with pytest.raises(ValueError, match="labels must be"):
        eng.step(dense, strings, labels[:-1])


# Thresholds and reasoning of test_gpu_tensor_core_precision.py: r = ||got - ref|| / ||1xTF32 - ref|| over the
# elements one contraction kind feeds; 3xTF32 sits at fp32 noise, far under tf32.R_MAX = 1/4, one product near 1.
# The forward feeds the logits; the data pass the table rows' gradients (dx); the weight pass dW0, dW1, dW2.
# The oracle takes its own ReLU masks, not the kernel's: on a batch of thousands of samples a few of the 448
# pre-activations per sample lie within fp32 noise of zero, and each mask that flips there moves a gradient by far
# more than the 1xTF32 yardstick (r = 3.1 and 3.3 for the data and weight passes at B = 4096 on an H100, with the
# forward at 0.007 and every output within the per-element bound).  So the statistic runs on short batches, where
# no mask sits that close to zero, and the per-element bound of test_tower_matches_oracle covers the long ones.
@pytest.mark.parametrize("B", [33, 64])
def test_contractions_are_3xtf32(B):
    ids, dense, labels, flat = _inputs(B, "uniform", 21)
    out = M.deepctr_wdl_tower(ids, dense, labels, flat)
    ref = O.reference(ids, dense, labels, flat)
    touched = torch.zeros((M.FIELDS, M.ROWS), dtype=torch.bool, device=DEV)
    touched[torch.arange(M.FIELDS, device=DEV).unsqueeze(1).expand_as(ids), ids.long()] = True
    deep_rows = torch.zeros(M.N_PARAMS, dtype=torch.bool, device=DEV)
    deep_rows[:O.O_LIN] = touched.unsqueeze(2).expand(-1, -1, M.DIM).reshape(-1)
    weights = torch.zeros(M.N_PARAMS, dtype=torch.bool, device=DEV)
    for n in ("dnn/kernel0:0", "dnn/kernel1:0", "dnn/kernel2:0"):
        weights[M.OFFSETS[n]:M.OFFSETS[n] + int(np.prod(dict(M.PARAMS)[n]))] = True
    checks = [("forward", "logits", None), ("data", "grads", deep_rows), ("weight", "grads", weights)]
    rs = {}
    for kind, fam, sel in checks:
        emu = O.reference(ids, dense, labels, flat, contraction={kind: "1x"})
        rs[kind] = tf32.ratio(out[fam], ref[fam], emu[fam], sel)
    print("B=%d ||got - ref|| / ||1xTF32 - ref||: %s" % (B, rs))
    assert all(r <= tf32.R_MAX for r in rs.values()), (B, rs)


# ---------------------------------------------------------------------------------------------------- engine
def _data(B, n, seed):
    out = []
    for s in range(n):
        dense, strings, labels = M.synthetic_batch(B, seed + s, DEV)
        out.append((dense / 1e4, strings, labels))  # raw counts put p at the clip edge; see test_gpu_fc_dnn._batches
    return out


def _make(opt, n_shards, B, seed=3):
    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(n_shards, opt_type, opt_args, device=0)
    return group, M.DeepctrWdlEngine(group, B, lr, seed=seed), lr


def _servers(group, eng, opt):
    opt_type, opt_args, _ = OPTS[opt]
    N = group.n_shards
    servers = [OracleServer(s, opt_type, opt_args, num_ps=N) for s in range(N)]
    state = group.pull_dense(M.NAMES)
    for s, srv in enumerate(servers):
        srv.push_model(dense={n: state[n].cpu().numpy() for n in M.NAMES if eng.owner[n] == s})
    return servers


def _push_to_oracle(servers, eng, lr):
    per = {s: {} for s in range(len(servers))}
    for n, v in M.flat_views(eng.tower.grads).items():
        per[eng.owner[n]][n] = v.cpu().numpy()
    for s, srv in enumerate(servers):
        ok, _ = srv.push_gradients(per[s], {}, lr, 0)
        assert ok


def _compare_state(group, servers, eng, opt):
    state = group.pull_dense(M.NAMES)
    for n in M.NAMES:
        srv = servers[eng.owner[n]]
        np.testing.assert_allclose(state[n].cpu().numpy(), srv.dense[n], rtol=1e-6, atol=1e-9, err_msg=n)
        if opt == "adam":
            for k, sn in enumerate(("m", "v")):
                np.testing.assert_allclose(group.slot_dense(n, k + 1).cpu().numpy(), srv.opt.dense_slots[sn][n],
                                           rtol=1e-5, atol=1e-15, err_msg=(n, sn))


@pytest.mark.parametrize("n_shards", [1, 3])
@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_engine_matches_oracle(opt, n_shards):
    B, steps = 300, 5
    group, eng, lr = _make(opt, n_shards, B)
    servers = _servers(group, eng, opt)
    for step, (dense, strings, labels) in enumerate(_data(B, steps, 100)):
        loss = eng.step(dense, strings, labels)
        torch.cuda.synchronize()
        eng.check()
        ref = O.reference(eng.ids, dense, labels, eng.flat)
        O.check(eng.tower.outputs(), ref, n_sm=_n_sm(), label="step %d" % step)
        assert abs(float(loss) - float(ref["loss"])) <= 1e-5 * float(ref["M"]["loss"])
        _push_to_oracle(servers, eng, lr)
    torch.cuda.synchronize()
    _compare_state(group, servers, eng, opt)
    assert [v for v, _, _ in group.snapshot()] == [steps] * n_shards


def test_untouched_rows_move_by_the_dense_update():
    """After one Adam step a deep-table row no sample read moves by Adam's first step on g = 2 lambda w (about
    0.63 % of w: epsilon-dominated), and the untouched rows of the zero-initialised linear tables stay zero."""
    B = 64
    group, eng, lr = _make("adam", 1, B)
    before = group.pull_dense(M.NAMES)
    dense, strings, labels = _data(B, 1, 5)[0]
    eng.step(dense, strings, labels)
    torch.cuda.synchronize()
    after = group.pull_dense(M.NAMES)
    ids = eng.ids.long()
    for j in (0, 13, 25):
        touched = torch.zeros(M.ROWS, dtype=torch.bool, device=DEV)
        touched[ids[j]] = True
        w = before[M.DEEP_NAMES[j]][~touched].double()
        g = 2e-5 * w.float().double()
        m, v = 0.1 * g, 0.001 * g * g
        lr_t = 1e-3 * np.sqrt(1 - 0.999) / (1 - 0.9)
        want = w - lr_t * m / (torch.sqrt(v) + 1e-7)
        got = after[M.DEEP_NAMES[j]][~touched].double()
        torch.testing.assert_close(got, want, rtol=2e-6, atol=1e-12)
        moved = ((w - got).abs() / w.abs()).median()
        assert 0.005 < float(moved) < 0.0075
        assert torch.count_nonzero(after[M.LINEAR_NAMES[j]][~touched]) == 0
        assert torch.count_nonzero(after[M.LINEAR_NAMES[j]][touched]) > 0


def test_replay_equals_step():
    B = 200
    ga, ea, _ = _make("adam", 2, B, seed=4)
    gb, eb, _ = _make("adam", 2, B, seed=4)
    for dense, strings, labels in _data(B, 4, 50):
        ea.step(dense, strings, labels)
        eb.replay(dense, strings, labels)
    torch.cuda.synchronize()
    sa, sb = ga.pull_dense(M.NAMES), gb.pull_dense(M.NAMES)
    for n in M.NAMES:
        assert torch.equal(sa[n], sb[n]), n


def test_evaluate_matches_oracle_forward():
    B = 500
    group, eng, _ = _make("sgd", 1, B)
    metrics = EvaluationMetrics(M.eval_metrics_fn())
    probs, labs = [], []
    for dense, strings, labels in _data(B, 2, 900):
        logits = eng.evaluate(dense, strings, labels, metrics)
        torch.cuda.synchronize()
        ref = O.reference(eng.ids, dense, labels, eng.flat)
        O.check({"logits": logits}, ref, n_sm=_n_sm())
        probs.append(torch.sigmoid(logits).clone())
        labs.append(labels)
    auc = float(metrics.get_evaluation_summary()["probs"]["auc"])
    ref_metrics = EvaluationMetrics(M.eval_metrics_fn())
    for p, l in zip(probs, labs):
        ref_metrics.update_evaluation_metrics({"probs": p}, l)
    assert abs(auc - float(ref_metrics.get_evaluation_summary()["probs"]["auc"])) < 1e-6
    assert [v for v, _, _ in group.snapshot()] == [0]


def test_engine_matches_dropin_trainer():
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    B, steps = 128, 4
    group_e, eng, lr = _make("adam", 1, B, seed=6)
    opt_type, opt_args, _ = OPTS["adam"]
    group_d = PSGroup(1, opt_type, opt_args, device=0)
    twin = M.DeepctrWdl(lr=lr).to(DEV)
    twin.load_flat(torch.cat([group_e.pull_dense([n])[n].reshape(-1) for n in M.NAMES]))
    client = PSClient(group_d)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(twin, client, args=types.SimpleNamespace(cuda_graph=True))
    for step, (dense, strings, labels) in enumerate(_data(B, steps, 700)):
        loss_e = float(eng.step(dense, strings, labels))
        ids, _ = M.transform(DEV)(dense, strings)
        accepted, version, loss_d = trainer.train_minibatch({"ids": ids.long(), "dense": dense}, labels)
        assert accepted and version == step + 1
        assert abs(loss_e - float(loss_d)) <= 1e-4 * max(1.0, abs(loss_e)), (step, loss_e, float(loss_d))
    torch.cuda.synchronize()
    group_d.check()
    de = group_e.pull_dense(M.NAMES)
    dd = group_d.pull_dense([n for n, _ in twin.named_parameters()])
    names_d = {id(p): k for k, p in twin.named_parameters()}
    for n, p in zip(M.NAMES, twin.ordered()):
        torch.testing.assert_close(de[n], dd[names_d[id(p)]].reshape(de[n].shape), rtol=1e-4, atol=1e-6)


def _four_workers(opt, B):
    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(2, opt_type, opt_args, device=0)
    engines = [M.DeepctrWdlEngine(group, B, lr, seed=5, register=(w == 0)) for w in range(4)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(4)]
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.capture()
    torch.cuda.synchronize()
    return group, engines, streams, lr


def test_four_workers_concurrent():
    B, steps = 256, 10
    group, engines, streams, _ = _four_workers("sgd", B)
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
    assert [v for v, _, _ in group.snapshot()] == [4 * steps] * 2
    for e in engines:
        e.check()


def test_four_workers_serialised_match_oracle():
    B, rounds = 256, 2
    group, engines, streams, lr = _four_workers("adam", B)
    servers = _servers(group, engines[0], "adam")
    data = [_data(B, rounds, 1000 * (w + 1)) for w in range(4)]
    for r in range(rounds):
        for w in range(4):
            with torch.cuda.stream(streams[w]):
                engines[w].replay(*data[w][r])
            streams[w].synchronize()
            _push_to_oracle(servers, engines[w], lr)
    _compare_state(group, servers, engines[0], "adam")
    assert [v for v, _, _ in group.snapshot()] == [4 * rounds] * 2
