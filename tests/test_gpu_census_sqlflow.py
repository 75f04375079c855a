"""The census_model_sqlflow models on the GPU: the feature transform of both id rules against
oracle/census_sqlflow_oracle.py's restatement; the tower (csrc/census_sqlflow_tower.cu) against the float64 oracle
at tile and grid edges, with absent ids and whole groups absent, in both reshape modes; the oracle's mutations;
bitwise repeats and graph replay; CensusSqlflowEngine against OracleServer on SGD and Adam over one and three
shards, with a schedule applied by model version; evaluate; the engine against the drop-in trainer over the torch
twin; four graphed workers."""
import threading
import types

import numpy as np
import pytest
import torch

from elasticdl_b200 import callbacks as cb
from elasticdl_b200.common.evaluation_utils import EvaluationMetrics
from elasticdl_b200.ps import PSGroup
from elasticdl_b200.workloads import census_sqlflow as M
from elasticdl_b200.workloads import census_sqlflow_features as F
from oracle import census_sqlflow_oracle as O
from oracle import feature_oracle as FO
from oracle.lr_schedule_oracle import piecewise_constant, schedule_argument
from oracle.ps_oracle import OracleServer

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
OPTS = {"sgd": ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", 0.1), "adam": M.optimizer()}


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _oracle_ids(num, raw, variant, mutate=None):
    return O.sqlflow_ids(num, raw, variant, F.FEATURES, list(F.FEATURE_GROUPS.values()), F.NUMERIC_KEYS,
                         F.STRING_KEYS, mutate=mutate)


@pytest.mark.parametrize("variant", F.VARIANTS)
@pytest.mark.parametrize("B", [1, 1000, 70000])
def test_transform_matches_oracle(variant, B):
    numeric, strings, num, raw = F.synthetic_batch(B, 7 + B % 13, DEV, empty_fraction=0.1, zero_fraction=0.1)
    if B >= 100:  # every boundary value, "?", OOV strings and "" in every lookup column
        for j, name in enumerate(F.NUMERIC_KEYS):
            bnd = F.FEATURES[name][1]
            num[j, :len(bnd)] = bnd
        for name in ("workclass", "marital_status", "relationship", "race", "sex"):
            col = raw[F.STRING_KEYS.index(name)]
            col[:4] = ["?", "", "Unseen", F.FEATURES[name][1][-1]]
        numeric = torch.from_numpy(num).to(DEV)
        from elasticdl_b200.preprocessing.layers import encode_strings

        strings = torch.stack([encode_strings(r, F.STRING_WIDTH, device="cpu") for r in raw]).to(DEV)
    ids, _ = F.transform(variant, DEV)(numeric, strings)
    want = _oracle_ids(num, raw, variant)
    np.testing.assert_array_equal(ids.cpu().numpy(), want)
    if B >= 100:
        assert (want == -1).any()
        for m in O.ID_MUTATIONS:
            assert not np.array_equal(ids.cpu().numpy(), _oracle_ids(num, raw, variant, m)), m


def test_existing_transforms_unchanged_by_absent_default():
    """A spec without "absent" keeps the old ids: an empty string still hashes, 0.0 still buckets."""
    from elasticdl_b200.preprocessing.layers import FeatureTransform, encode_strings

    strings = encode_strings([["", "a", ""]], 8, device=DEV)
    numeric = torch.tensor([[0.0, 1.0, 0.0]], device=DEV)
    specs = [{"kind": "hash", "column": 0, "num_bins": 7, "offset": 3},
             {"kind": "discretize", "column": 0, "bins": [0.5], "offset": 10}]
    old, _ = FeatureTransform(specs, (), torch.int32, device=DEV)(numeric, strings)
    new, _ = FeatureTransform([dict(s, absent=True) for s in specs], (), torch.int32, device=DEV)(numeric, strings)
    assert old[:, 0].tolist() == [3 + int(FO.hashing([""], 7)[0]), 10]
    assert new[:, 0].tolist() == [-1, -1] and new[:, 1].tolist() == old[:, 1].tolist()


def _ids(B, pattern, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rows = []
    for g, r in enumerate(O.GROUP_ROWS):
        if pattern == "one":
            v = torch.full((4, B), (7 * g + 3) % r, dtype=torch.int32, device=DEV)
        else:
            u = torch.rand((4, B), generator=gen, device=DEV)
            v = torch.clamp((r * u ** 2).floor(), max=r - 1).to(torch.int32)
            v[torch.rand((4, B), generator=gen, device=DEV) < 0.3] = -1
        if pattern == "group_absent":
            v[:] = -1 if g == 1 else v
        rows.append(v)
    ids = torch.cat(rows)
    if pattern == "all_absent":
        ids[:, ::3] = -1
    return ids.contiguous()


def _inputs(B, pattern, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    labels = (torch.rand(B, generator=gen, device=DEV) < 0.3).float()
    return _ids(B, pattern, seed), labels, O.random_params(gen, DEV)


def _dense(out):
    gs = []
    for t in range(5):
        n = int(out["n_unique"][t])
        d = torch.zeros_like(out["gsum"][t])
        d[out["uniq"][t][:n]] = out["gsum"][t][:n]
        gs.append(d)
    return {"logits": out["logits"], "loss": out["loss"], "grads": out["grads"], "gsum": gs}


def _check_exact_rows(out, ref):
    for t in range(5):
        n = int(out["n_unique"][t])
        assert n == ref["n_unique"][t], t
        assert torch.equal(out["uniq"][t][:n].cpu(), ref["uniq"][t].cpu()), t


def _b(B):
    return _n_sm() * M.TILE + 1 if B == "wave+1" else B


@pytest.mark.parametrize("pattern", ["mixed", "one", "group_absent", "all_absent"])
@pytest.mark.parametrize("B", [1, 255, 256, 257, 4096, "wave+1", 65536])
@pytest.mark.parametrize("q11", [False, True])
def test_tower_matches_oracle(q11, B, pattern):
    Bn = _b(B)
    ids, labels, flat = _inputs(Bn, pattern, seed=Bn % 1000)
    out = M.census_sqlflow_tower(ids, labels, flat, q11)
    ref = O.csql_reference(ids, labels, flat, q11)
    _check_exact_rows(out, ref)
    O.check(_dense(out), ref, n_sm=_n_sm(), label="B=%d %s q11=%s" % (Bn, pattern, q11))
    fwd = M.census_sqlflow_tower(ids, None, flat, q11, train=False)
    assert torch.equal(fwd["logits"], out["logits"])


@pytest.mark.parametrize("B", [600, "wave+1"])
@pytest.mark.parametrize("q11", [False, True])
def test_mutations_are_caught(q11, B):
    Bn = _b(B)
    ids, labels, flat = _inputs(Bn, "mixed", seed=5)
    ref = O.csql_reference(ids, labels, flat, q11)
    got = _dense(M.census_sqlflow_tower(ids, labels, flat, q11))
    assert not O.caught_by(got, ref, n_sm=_n_sm())
    muts = O.mutations(ref, (ids, labels, flat, q11))
    assert set(muts) == set(O.TOWER_MUTATIONS)
    for name, mut in muts.items():
        assert O.caught_by(mut, ref, n_sm=_n_sm()), (name, Bn)


@pytest.mark.parametrize("q11", [False, True])
def test_deterministic_and_graph_replay(q11):
    B = 65536
    ids, labels, flat = _inputs(B, "mixed", seed=9)
    call = M.CsqlTowerCall(B, DEV)
    bufs = [call.loss, call.logits, call.grads, call.uniq, call.n_unique, call.gsum]
    call.launch(ids, labels, flat, q11)
    first = [b.clone() for b in bufs]
    call.launch(ids, labels, flat, q11)
    for a, b in zip(first, bufs):
        assert torch.equal(a, b)
    for b in bufs:
        b.fill_(float("nan") if b.is_floating_point() else -1)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call.launch(ids, labels, flat, q11)
    for _ in range(2):  # the arrival counter is back at zero after every replay
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(first, bufs):
            assert torch.equal(a, b)
    call.check_error()


def test_refusals():
    B = 64
    ids, labels, flat = _inputs(B, "mixed", seed=1)
    bad = ids.clone()
    bad[5, 3] = 73  # group 2's rows are 0..72
    bad[11, 0] = -2
    with pytest.raises(ValueError, match="2 census_sqlflow ids outside"):
        M.census_sqlflow_tower(bad, labels, flat)
    with pytest.raises(ValueError, match="ids must be"):
        M.census_sqlflow_tower(ids.long(), labels, flat)
    with pytest.raises(ValueError, match="labels must be"):
        M.census_sqlflow_tower(ids, labels.double(), flat)
    with pytest.raises(ValueError, match="params must be"):
        M.census_sqlflow_tower(ids, labels, flat[:-1])
    opt_type, opt_args, lr = OPTS["sgd"]
    with pytest.raises(ValueError, match="unknown model"):
        M.CensusSqlflowEngine(PSGroup(1, opt_type, opt_args, device=0), "census_wide_deep", B, lr)
    with pytest.raises(ValueError, match="sync-SGD"):
        M.CensusSqlflowEngine(PSGroup(1, opt_type, opt_args, device=0, use_async=False),
                              "wide_deep_functional_keras", B, lr)
    eng = M.CensusSqlflowEngine(PSGroup(1, opt_type, opt_args, device=0), "wide_deep_functional_keras", B, lr)
    numeric, strings, _, _ = F.synthetic_batch(B, 3, DEV)
    with pytest.raises(ValueError, match="numeric must be"):
        eng.step(numeric[:, :-1].contiguous(), strings, labels)
    with pytest.raises(ValueError, match="strings must be"):
        eng.step(numeric, strings.int(), labels)


# ---------------------------------------------------------------------------------------------------- engine
def _batches(B, n, seed):
    out = []
    for s in range(n):
        numeric, strings, num, raw = F.synthetic_batch(B, seed + s, DEV)
        labels = (torch.rand(B, generator=torch.Generator(device=DEV).manual_seed(seed + s), device=DEV) < 0.25).float()
        out.append((numeric, strings, labels))
    return out


def _servers(group, eng, opt):
    opt_type, opt_args, _ = OPTS[opt]
    servers = [OracleServer(s, opt_type, opt_args, num_ps=group.n_shards) for s in range(group.n_shards)]
    state = group.pull_dense(eng.names)
    for s, srv in enumerate(servers):
        srv.push_model(dense={n: state[n].cpu().numpy() for n in eng.names if eng.owner[n] == s})
    return servers


def _oracle_flat(servers, eng):
    return torch.cat([torch.from_numpy(servers[eng.owner[n]].dense[n]).reshape(-1) for n in eng.names])


def _push_to_oracle(servers, eng, lr):
    out = eng.tower.outputs()
    per = {s: ({}, {}) for s in range(len(servers))}
    for i, n in enumerate(M.MLP_NAMES):
        per[eng.owner[n]][0][n] = M.flat_views(out["grads"].cpu())[i].numpy()
    for t, n in enumerate(eng.names[6:]):
        k = int(out["n_unique"][t])
        per[eng.owner[n]][1][n] = (out["uniq"][t][:k].cpu().numpy().astype(np.int64),
                                   np.ascontiguousarray(out["gsum"][t][:k].cpu().numpy()))
    for s, srv in enumerate(servers):
        ok, _ = srv.push_gradients(per[s][0], per[s][1], lr, 0)
        assert ok


def _compare_state(group, servers, eng, opt):
    state = group.pull_dense(eng.names)
    for n in eng.names:
        srv = servers[eng.owner[n]]
        np.testing.assert_allclose(state[n].cpu().numpy(), srv.dense[n], rtol=1e-6, atol=1e-8, err_msg=n)
        if opt == "adam":
            for k, sn in enumerate(("m", "v")):
                np.testing.assert_allclose(group.slot_dense(n, k + 1).cpu().numpy(), srv.opt.dense_slots[sn][n],
                                           rtol=1e-5, atol=1e-12, err_msg=(n, sn))
    assert [v for v, _, _ in group.snapshot()] == [srv.version for srv in servers]


@pytest.mark.parametrize("n_shards", [1, 3])
@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("model", ["wide_deep_functional_keras", "wide_deep_functional_tensor_interface_fc"])
def test_engine_matches_oracle(model, opt, n_shards):
    """Five steps; the schedule (0.5x then 0.25x the optimizer's lr, crossing at the fourth push) is applied by the
    push from the versions it begins on, and the oracle applies the same values at the same versions."""
    B, steps = 512, 5
    opt_type, opt_args, lr = OPTS[opt]
    sched = cb.PiecewiseConstantDecay([1], [lr / 2, lr / 4])
    group = PSGroup(n_shards, opt_type, opt_args, device=0)
    eng = M.CensusSqlflowEngine(group, model, B, lr, seed=11, lr_schedule=sched)
    variant, q11 = M.model_of(model)
    servers = _servers(group, eng, opt)
    for step in range(steps):
        numeric, strings, num, raw = F.synthetic_batch(B, 100 + step, DEV)
        labels = (torch.rand(B, generator=torch.Generator(device=DEV).manual_seed(step), device=DEV) < 0.25).float()
        before = _oracle_flat(servers, eng)
        loss = eng.step(numeric, strings, labels)
        torch.cuda.synchronize()
        eng.check()
        torch.testing.assert_close(eng.flat.cpu(), before, rtol=1e-6, atol=1e-8)
        assert np.array_equal(eng.ids.cpu().numpy(), _oracle_ids(num, raw, variant))
        ref = O.csql_reference(eng.ids, labels, eng.flat, q11)
        assert abs(float(loss) - float(ref["loss"])) <= 1e-5 * float(ref["M"]["loss"])
        out = eng.tower.outputs()
        _check_exact_rows(out, ref)
        O.check(_dense(out), ref, n_sm=_n_sm(), label="step %d" % step)
        versions = [srv.version for srv in servers]
        _push_to_oracle(servers, eng, piecewise_constant(schedule_argument(versions), [1], [lr / 2, lr / 4]))
    torch.cuda.synchronize()
    _compare_state(group, servers, eng, opt)
    assert [v for v, _, _ in group.snapshot()] == [steps] * n_shards


@pytest.mark.parametrize("model", ["wide_deep_subclass_keras", "wide_deep_functional_fc"])
def test_evaluate_matches_oracle_forward(model):
    B = 500
    group = PSGroup(1, *OPTS["sgd"][:2], device=0)
    eng = M.CensusSqlflowEngine(group, model, B, 0.1)
    _, q11 = M.model_of(model)
    metrics = EvaluationMetrics({"logits": M.eval_metrics_fn()["logits"]})
    hits = 0
    data = _batches(B, 2, 900)
    for numeric, strings, labels in data:
        logits = eng.evaluate(numeric, strings, labels, metrics)
        torch.cuda.synchronize()
        ref = O.csql_reference(eng.ids, labels, eng.flat, q11)
        O.check({"logits": logits}, ref, n_sm=_n_sm())
        hits += int(((ref["logits"] > 0.5).int() == labels.int()).sum())  # Q12: the logit, not the probability
    acc = metrics.get_evaluation_summary()["logits"]["accuracy"]
    assert abs(float(acc) - hits / (2 * B)) < 1e-6
    assert [v for v, _, _ in group.snapshot()] == [0]  # nothing pushed
    eng.check()


@pytest.mark.parametrize("model", ["wide_deep_functional_keras", "wide_deep_functional_tensor_interface_fc"])
def test_engine_matches_dropin_trainer(model):
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    B, steps = 128, 6
    opt_type, opt_args, lr = OPTS["sgd"]
    group_e = PSGroup(1, opt_type, opt_args, device=0)
    eng = M.CensusSqlflowEngine(group_e, model, B, lr, seed=6)
    group_d = PSGroup(1, opt_type, opt_args, device=0)
    twin = M.CensusSqlflowWideDeep(model, lr=lr).to(DEV)
    twin.load_mlp(torch.cat([group_e.pull_dense([n])[n].reshape(-1) for n in eng.names]))
    client = PSClient(group_d)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(twin, client, args=types.SimpleNamespace(cuda_graph=False))
    tables = eng.names[6:]
    start = group_e.pull_dense(tables)
    group_d.set_rows([(n, torch.arange(start[n].shape[0], device=DEV), start[n]) for n in tables])
    for step, (numeric, strings, labels) in enumerate(_batches(B, steps, 700)):
        loss_e = float(eng.step(numeric, strings, labels))
        accepted, version, loss_d = trainer.train_minibatch((numeric, strings), labels)
        assert accepted and version == step + 1
        assert abs(loss_e - float(loss_d)) <= 1e-4 * max(1.0, abs(loss_e)), (step, loss_e, float(loss_d))
    torch.cuda.synchronize()
    group_d.check()
    end = group_e.pull_dense(tables)
    for n in tables:
        torch.testing.assert_close(end[n], group_d.pull_rows([(n, torch.arange(end[n].shape[0], device=DEV))])[0],
                                   rtol=1e-4, atol=1e-6)
    dense_d = group_d.pull_dense([n for n, _ in twin.dense.named_parameters(prefix="dense")])
    mlp = group_e.pull_dense(M.MLP_NAMES)
    for i in range(3):
        torch.testing.assert_close(mlp[M.MLP_NAMES[2 * i]].t(), dense_d["dense.%d.weight" % i], rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(mlp[M.MLP_NAMES[2 * i + 1]], dense_d["dense.%d.bias" % i], rtol=1e-4, atol=1e-6)


def _four_workers(opt, B, model="wide_deep_functional_keras"):
    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(2, opt_type, opt_args, device=0)
    engines = [M.CensusSqlflowEngine(group, model, B, lr, seed=5, register=(w == 0)) for w in range(4)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(4)]
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.capture()
    torch.cuda.synchronize()
    return group, engines, streams, lr


def test_four_workers_concurrent():
    B, steps = 256, 20
    group, engines, streams, _ = _four_workers("sgd", B)
    data = [_batches(B, 4, 1000 * (w + 1)) for w in range(4)]
    torch.cuda.synchronize()
    errors = []

    def run(w):
        try:
            with torch.cuda.stream(streams[w]):
                for s in range(steps):
                    engines[w].replay(*data[w][s % 4])
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
    B, rounds = 256, 3
    group, engines, streams, lr = _four_workers("adam", B, "wide_deep_functional_fc")
    servers = _servers(group, engines[0], "adam")
    data = [_batches(B, rounds, 1000 * (w + 1)) for w in range(4)]
    for r in range(rounds):
        for w in range(4):
            with torch.cuda.stream(streams[w]):
                engines[w].replay(*data[w][r])
            streams[w].synchronize()
            _push_to_oracle(servers, engines[w], lr)
    _compare_state(group, servers, engines[0], "adam")
    assert [v for v, _, _ in group.snapshot()] == [4 * rounds] * 2
