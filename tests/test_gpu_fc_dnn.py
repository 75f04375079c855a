"""The feature-column DNN tower (csrc/fc_dnn_tower.cu, include/b200_fc_dnn.h) and FeatureColumnDNNEngine for
census_dnn_model and heart_functional_api against the float64 oracle of oracle/fc_dnn_oracle.py.

Kernel level: batches at the warp, tile and grid edges up to 65536; uniform buckets, every sample in one bucket,
half the strings empty, and a last bias of +-20 that clips every probability; the oracle's mutations; bitwise
repeats and graph replay; the transform's buckets against feature_oracle's FarmHash; the refusals.  Engine level:
five SGD and Adam steps on one and three shards against OracleServer fed the engine's own gradients, evaluate with
the model's metrics, the drop-in trainer over the torch twin, and four graphed workers on cloned views, concurrent
and serialised."""
import threading
import types

import numpy as np
import pytest
import torch

from elasticdl_b200.common.evaluation_utils import EvaluationMetrics
from elasticdl_b200.ps import PSGroup
from elasticdl_b200.workloads import fc_dnn as M
from oracle import fc_dnn_oracle as O
from oracle import feature_oracle as FO
from oracle.ps_oracle import EmbeddingTableInfo, OracleServer

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
OPTS = {"sgd": ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", 0.1),
        "adam": ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", 1e-3)}
MODELS = ["census_dnn_model", "heart_functional_api"]


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _kernel_inputs(L, B, pattern, seed):
    """numeric, ids (buckets), strings (only their emptiness matters to the tower), inv, n_unique, rows, labels,
    flat -- and the oracle's view of them."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    T = len(L.tables)
    numeric = torch.randn((len(L.numeric_keys), B), generator=g, device=DEV)
    ids = torch.zeros((T + len(L.buckets), B), dtype=torch.int32, device=DEV)
    for i, (_, bins) in enumerate(L.buckets):
        ids[T + i] = torch.randint(0, len(bins) + 1, (B,), generator=g, device=DEV, dtype=torch.int32)
    p_empty = 0.5 if pattern == "empty" else 0.05
    present = torch.rand((len(L.string_keys), B), generator=g, device=DEV) >= p_empty
    strings = torch.zeros((len(L.string_keys), B, M.STRING_WIDTH), dtype=torch.uint8, device=DEV)
    strings[:, :, 0] = present.to(torch.uint8) * 97
    inv = torch.zeros((T, B), dtype=torch.int32, device=DEV)
    n_unique = torch.zeros(T, dtype=torch.int32, device=DEV)
    rows = torch.zeros(L.row_off[-1], dtype=torch.float32, device=DEV)
    rows_list = []
    for k, (key, r, d) in enumerate(L.tables):
        if pattern == "one":
            bucket = torch.full((B,), (5 * k + 3) % r, dtype=torch.int64, device=DEV)
        else:
            bucket = torch.randint(0, r, (B,), generator=g, device=DEV)
        bucket[~present[L.string_keys.index(key)]] = 0
        u, iv = torch.unique(bucket, return_inverse=True)
        inv[k] = iv.to(torch.int32)
        n_unique[k] = u.numel()
        vals = (torch.rand((u.numel(), d), generator=g, device=DEV) * 2 - 1) * 0.5
        rows[L.row_off[k]:L.row_off[k] + u.numel() * d] = vals.reshape(-1)
        rows_list.append(vals)
    labels = (torch.rand(B, generator=g, device=DEV) < 0.3).float()
    flat = torch.cat([(torch.rand(int(np.prod(s)), generator=g, device=DEV) * 2 - 1) * 0.4 for _, s in L.mlp])
    if pattern == "clip+":
        flat[-1] = 20.0
    elif pattern == "clip-":
        flat[-1] = -20.0
    kern = (numeric, ids, strings, inv, n_unique, rows, labels, flat)
    empty = torch.stack([~present[L.string_keys.index(key)] for key, _, _ in L.tables])
    orc = (numeric, ids, empty, inv, n_unique.tolist(), rows_list, labels, flat)
    return kern, orc


def _got(out, n_unique):
    return {"logits": out["logits"], "loss": out["loss"], "grads": out["grads"],
            "gsum": [g[:int(n)] for g, n in zip(out["gsum"], n_unique)]}


BATCHES = [1, 31, 32, 33, 63, 64, 65, 4096, 65536]


@pytest.mark.parametrize("pattern", ["uniform", "one", "empty", "clip+", "clip-"])
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("model", MODELS)
def test_tower_matches_oracle(model, B, pattern):
    L = M.layout_of(model)
    kern, orc = _kernel_inputs(L, B, pattern, seed=B % 997 + len(pattern))
    out = M.fc_dnn_tower(model, *kern)
    ref = O.fc_dnn_reference(L.spec(), *orc)
    O.check(_got(out, orc[4]), ref, n_sm=_n_sm(), label="%s B=%d %s" % (model, B, pattern))
    if pattern.startswith("clip"):
        assert torch.count_nonzero(out["grads"]) == 0
    fwd = M.fc_dnn_tower(model, *kern[:6], None, kern[7], train=False)
    assert torch.equal(fwd["logits"], out["logits"])


@pytest.mark.parametrize("model", MODELS)
def test_mutations_are_caught(model):
    L = M.layout_of(model)
    kern, orc = _kernel_inputs(L, 4096, "empty", seed=5)
    got = _got(M.fc_dnn_tower(model, *kern), orc[4])
    ref = O.fc_dnn_reference(L.spec(), *orc)
    assert not O.caught_by(got, ref, n_sm=_n_sm())
    for name, mut in O.mutations(L.spec(), orc).items():
        if name == "clip_grad_kept":
            continue
        assert O.caught_by(mut, ref, n_sm=_n_sm()), name
    kern, orc = _kernel_inputs(L, 4096, "clip+", seed=6)
    ref = O.fc_dnn_reference(L.spec(), *orc)
    assert O.caught_by(O.mutations(L.spec(), orc, ("clip_grad_kept",))["clip_grad_kept"], ref, n_sm=_n_sm())


@pytest.mark.parametrize("model", MODELS)
def test_deterministic_and_graph_replay(model):
    L = M.layout_of(model)
    B = 65536
    kern, _ = _kernel_inputs(L, B, "uniform", seed=9)
    call = M.FcDnnTowerCall(L, B, DEV)
    bufs = [call.loss, call.logits, call.grads, call.gsum]
    call.launch(*kern)
    first = [b.clone() for b in bufs]
    call.launch(*kern)
    for a, b in zip(first, bufs):
        assert torch.equal(a, b)
    for b in bufs:
        b.fill_(float("nan"))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call.launch(*kern)
    for _ in range(2):  # the arrival counter is back at zero after every replay
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(first, bufs):
            assert torch.equal(a, b)


def test_transform_buckets_match_farmhash():
    B = 1000
    numeric, strings = M.synthetic_census_batch(B, 3, DEV, empty_fraction=0.1)
    L = M.CENSUS_DNN
    ids, _ = L.transform(DEV)(numeric, strings)
    host = strings.cpu().numpy()
    raw = [[bytes(host[c, b]).rstrip(b"\0") for b in range(B)] for c in range(8)]
    for k, (key, r, _) in enumerate(L.tables):
        col = L.string_keys.index(key)
        np.testing.assert_array_equal(ids[k].cpu().numpy(), FO.hashing(raw[col], r), err_msg=key)
    M.fill_empty(L, ids, strings)
    for k, (key, r, _) in enumerate(L.tables):
        col = L.string_keys.index(key)
        want = np.where([len(s) == 0 for s in raw[col]], 0, FO.hashing(raw[col], r))
        np.testing.assert_array_equal(ids[k].cpu().numpy(), want, err_msg=key)
    numeric, strings, _ = M.synthetic_heart_batch(B, 4, DEV)
    ids, _ = M.HEART.transform(DEV)(numeric, strings)
    np.testing.assert_array_equal(ids[1].cpu().numpy(), FO.discretize(numeric[0].cpu().numpy(), M.HEART_AGE_BOUNDARIES))


def test_refusals():
    L = M.CENSUS_DNN
    B = 64
    kern, _ = _kernel_inputs(L, B, "uniform", seed=1)
    numeric, ids, strings, inv, n_unique, rows, labels, flat = kern
    with pytest.raises(ValueError, match="numeric must be"):
        M.fc_dnn_tower(L, numeric[:3].contiguous(), *kern[1:])
    with pytest.raises(ValueError, match="ids must be"):
        M.fc_dnn_tower(L, numeric, ids.long(), *kern[2:])
    with pytest.raises(ValueError, match="strings must be"):
        M.fc_dnn_tower(L, numeric, ids, strings.int(), *kern[3:])
    with pytest.raises(ValueError, match="inv must be"):
        M.fc_dnn_tower(L, numeric, ids, strings, inv[:, :-1].contiguous(), *kern[4:])
    with pytest.raises(ValueError, match="labels must be"):
        M.fc_dnn_tower(L, *kern[:6], labels.double(), flat)
    with pytest.raises(ValueError, match="params must be"):
        M.fc_dnn_tower(L, *kern[:7], flat[:-1])
    with pytest.raises(ValueError, match="batch size"):
        M.FcDnnTowerCall(L, 0, DEV)
    with pytest.raises(ValueError, match="unknown model"):
        M.FcDnnTowerCall("census_model_sqlflow", B, DEV)
    bad = M.Layout("bad", ["a"], ["s"], tables=[("s", 600, 4)], buckets=[], columns=[("a", M.NUMERIC, "a"),
                                                                                      ("s_embedding", M.EMBEDDING, "s")],
                   loss_mean=True, optimizer=None)
    with pytest.raises(ValueError, match="512 rows"):
        M.fill_empty(bad, torch.zeros((1, B), dtype=torch.int32, device=DEV), strings[:1].contiguous())
    opt_type, opt_args, lr = OPTS["sgd"]
    with pytest.raises(ValueError, match="sync-SGD"):
        M.FeatureColumnDNNEngine(PSGroup(1, opt_type, opt_args, device=0, use_async=False), L, B, lr)
    with pytest.raises(ValueError, match="lr_staleness_modulation"):
        M.FeatureColumnDNNEngine(PSGroup(1, opt_type, opt_args, device=0, lr_staleness_modulation=True), L, B, lr)
    with pytest.raises(ValueError, match="batch size"):
        M.FeatureColumnDNNEngine(PSGroup(1, opt_type, opt_args, device=0), L, 0, lr)
    with pytest.raises(ValueError, match="unknown model"):
        M.FeatureColumnDNNEngine(PSGroup(1, opt_type, opt_args, device=0), "wide_deep", B, lr)
    eng = M.FeatureColumnDNNEngine(PSGroup(1, opt_type, opt_args, device=0), L, B, lr)
    numeric, strings = M.synthetic_census_batch(B, 3, DEV)
    with pytest.raises(ValueError, match="numeric must be"):
        eng.step(numeric[:, :-1].contiguous(), strings, labels)
    with pytest.raises(ValueError, match="strings must be"):
        eng.step(numeric, strings.int(), labels)
    with pytest.raises(ValueError, match="labels must be"):
        eng.step(numeric, strings, labels[:-1])


# ---------------------------------------------------------------------------------------------------- engine
def _batches(L, B, n, seed):
    """Raw rows with the numeric columns scaled down: the raw Adult and heart values (capital gains up to 20000)
    saturate the sigmoid, and a probability one float32 ulp from the clip edge takes or drops a large gradient
    (Q19) by rounding alone, which no rounding bound can hold."""
    out = []
    for s in range(n):
        if L is M.CENSUS_DNN:
            numeric, strings = M.synthetic_census_batch(B, seed + s, DEV)
            numeric = numeric / 1e4
            labels = (torch.rand(B, generator=torch.Generator(device=DEV).manual_seed(seed + s), device=DEV)
                      < 0.25).float()
        else:
            numeric, strings, labels = M.synthetic_heart_batch(B, seed + s, DEV)
            numeric = numeric / 100.0
        out.append((numeric, strings, labels))
    return out


def _make(model, opt, n_shards, B, seed=3, register=True, group=None):
    opt_type, opt_args, lr = OPTS[opt]
    group = group or PSGroup(n_shards, opt_type, opt_args, device=0)
    return group, M.FeatureColumnDNNEngine(group, model, B, lr, seed=seed, register=register), lr


def _all_ids(L):
    return [torch.arange(r, device=DEV) for _, r, _ in L.tables]


def _servers(group, eng, opt):
    """Oracle servers holding the group's dense parameters and every table row (all created here)."""
    L = eng.layout
    opt_type, opt_args, _ = OPTS[opt]
    N = group.n_shards
    servers = [OracleServer(s, opt_type, opt_args, num_ps=N) for s in range(N)]
    state = group.pull_dense(M.MLP_NAMES)
    rows = group.pull_rows(list(zip(L.table_names, _all_ids(L))))
    for s, srv in enumerate(servers):
        infos = [EmbeddingTableInfo(n, d, "zero", None) for n, (_, _, d) in zip(L.table_names, L.tables)]
        tables = {}
        for n, ids, r in zip(L.table_names, _all_ids(L), rows):
            m = ids % N == s
            tables[n] = (ids[m].cpu().numpy(), r[m].cpu().numpy())
        srv.push_model(dense={n: state[n].cpu().numpy() for n in M.MLP_NAMES if eng.owner[n] == s}, infos=infos,
                       tables=tables)
    return servers


def _oracle_flat(servers, eng):
    return torch.cat([torch.from_numpy(servers[eng.owner[n]].dense[n]).reshape(-1) for n in M.MLP_NAMES])


def _check_step(eng, numeric, strings, labels, label):
    L = eng.layout
    nu = eng.n_unique.tolist()
    rows = [eng.tower.table_view(eng.rows, k)[:n] for k, n in enumerate(nu)]
    empty = torch.stack([strings[L.string_keys.index(k), :, 0] == 0 for k, _, _ in L.tables])
    ref = O.fc_dnn_reference(L.spec(), numeric, eng.ids, empty, eng.inv, nu, rows, labels, eng.flat)
    O.check(_got(eng.tower.outputs(), nu), ref, n_sm=_n_sm(), label=label)
    return ref


def _push_to_oracle(servers, eng, lr):
    L, t = eng.layout, eng.tower
    N = len(servers)
    per = {s: ({}, {}) for s in range(N)}
    for n, v in L.flat_views(t.grads).items():
        per[eng.owner[n]][0][n] = v.cpu().numpy()
    for k, n in enumerate(L.table_names):
        U = int(eng.n_unique[k])
        uniq = eng.uniq[k * eng.B:k * eng.B + U].cpu().numpy().astype(np.int64)
        g = np.ascontiguousarray(t.table_view(t.gsum, k)[:U].cpu().numpy())
        for s in range(N):
            m = uniq % N == s
            per[s][1][n] = (uniq[m], g[m])
    for s, srv in enumerate(servers):
        ok, _ = srv.push_gradients(per[s][0], per[s][1], lr, 0)
        assert ok


def _compare_state(group, servers, eng, opt):
    L = eng.layout
    N = group.n_shards
    state = group.pull_dense(M.MLP_NAMES)
    for n in M.MLP_NAMES:
        srv = servers[eng.owner[n]]
        np.testing.assert_allclose(state[n].cpu().numpy(), srv.dense[n], rtol=1e-6, atol=1e-8, err_msg=n)
        if opt == "adam":
            for k, sn in enumerate(("m", "v")):
                np.testing.assert_allclose(group.slot_dense(n, k + 1).cpu().numpy(), srv.opt.dense_slots[sn][n],
                                           rtol=1e-5, atol=1e-12, err_msg=(n, sn))
    for n, ids in zip(L.table_names, _all_ids(L)):
        ids_np = ids.cpu().numpy()
        for s in range(N):
            m = ids_np % N == s
            mine = ids[torch.from_numpy(m).to(DEV)]
            np.testing.assert_allclose(group.pull_rows([(n, mine)])[0].cpu().numpy(), servers[s].tables[n].get(ids_np[m]),
                                       rtol=1e-6, atol=1e-8, err_msg=n)
            if opt == "adam":
                for k, sn in enumerate(("m", "v")):
                    np.testing.assert_allclose(group.slot_rows(n, mine, k + 1).cpu().numpy(),
                                               servers[s].opt.table_slots[sn][n].get(ids_np[m]),
                                               rtol=1e-5, atol=1e-12, err_msg=(n, sn))
    assert [v for v, _, _ in group.snapshot()] == [srv.version for srv in servers]


@pytest.mark.parametrize("n_shards", [1, 3])
@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("model", MODELS)
def test_engine_matches_oracle(model, opt, n_shards):
    B, steps = 300, 5
    group, eng, lr = _make(model, opt, n_shards, B)
    data = _batches(eng.layout, B, steps, 100)
    servers = _servers(group, eng, opt)
    for step, (numeric, strings, labels) in enumerate(data):
        before = _oracle_flat(servers, eng)
        loss = eng.step(numeric, strings, labels)
        torch.cuda.synchronize()
        eng.check()
        torch.testing.assert_close(eng.flat.cpu(), before, rtol=1e-6, atol=1e-8)
        ref = _check_step(eng, numeric, strings, labels, "step %d" % step)
        assert abs(float(loss) - float(ref["loss"])) <= 1e-5 * float(ref["M"]["loss"])
        _push_to_oracle(servers, eng, lr)
    torch.cuda.synchronize()
    _compare_state(group, servers, eng, opt)
    assert [v for v, _, _ in group.snapshot()] == [steps] * n_shards


@pytest.mark.parametrize("model", MODELS)
def test_replay_equals_step(model):
    B = 200
    ga, ea, _ = _make(model, "adam", 2, B, seed=4)
    gb, eb, _ = _make(model, "adam", 2, B, seed=4)
    L = ea.layout
    rows = ga.pull_rows(list(zip(L.table_names, _all_ids(L))))
    gb.set_rows([(n, ids, r) for n, ids, r in zip(L.table_names, _all_ids(L), rows)])
    for numeric, strings, labels in _batches(L, B, 4, 50):
        ea.step(numeric, strings, labels)
        eb.replay(numeric, strings, labels)
    torch.cuda.synchronize()
    sa, sb = ga.pull_dense(M.MLP_NAMES), gb.pull_dense(M.MLP_NAMES)
    for n in M.MLP_NAMES:
        assert torch.equal(sa[n], sb[n]), n
    for n, ids in zip(L.table_names, _all_ids(L)):
        assert torch.equal(ga.pull_rows([(n, ids)])[0], gb.pull_rows([(n, ids)])[0]), n
        assert torch.equal(ga.slot_rows(n, ids, 2), gb.slot_rows(n, ids, 2)), n


@pytest.mark.parametrize("model", MODELS)
def test_evaluate_matches_oracle_forward(model):
    B = 500
    group, eng, _ = _make(model, "sgd", 1, B)
    L = eng.layout
    metrics = EvaluationMetrics(M.eval_metrics_fn(model))
    hits = n = 0
    for numeric, strings, labels in _batches(L, B, 2, 900):
        logits = eng.evaluate(numeric, strings, labels, metrics)
        torch.cuda.synchronize()
        nu = eng.n_unique.tolist()
        rows = [eng.tower.table_view(eng.rows, k)[:u] for k, u in enumerate(nu)]
        empty = torch.stack([strings[L.string_keys.index(k), :, 0] == 0 for k, _, _ in L.tables])
        ref = O.fc_dnn_reference(L.spec(), numeric, eng.ids, empty, eng.inv, nu, rows, labels, eng.flat)
        O.check({"logits": logits}, ref, n_sm=_n_sm())
        if L is M.CENSUS_DNN:
            hits += int(((ref["logits"] > 0).int() == labels.int()).sum())
        else:
            hits += int((labels == 0).sum())  # Q20
        n += B
    acc = metrics.get_evaluation_summary()["logits"]["accuracy"]
    assert abs(float(acc) - hits / n) < 1e-6
    assert [v for v, _, _ in group.snapshot()] == [0]  # nothing pushed


@pytest.mark.parametrize("model", MODELS)
def test_engine_matches_dropin_trainer(model):
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    B, steps = 128, 6
    group_e, eng, lr = _make(model, "sgd", 1, B, seed=6)
    L = eng.layout
    opt_type, opt_args, _ = OPTS["sgd"]
    group_d = PSGroup(1, opt_type, opt_args, device=0)
    twin = M.FeatureColumnDNN(model, lr=lr, optimizer="sgd").to(DEV)
    twin.load_mlp(torch.cat([group_e.pull_dense([n])[n].reshape(-1) for n in M.MLP_NAMES]))
    client = PSClient(group_d)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(twin, client, args=types.SimpleNamespace(cuda_graph=True))
    rows = group_e.pull_rows(list(zip(L.table_names, _all_ids(L))))
    group_d.set_rows([(n, ids, r) for n, ids, r in zip(L.table_names, _all_ids(L), rows)])
    transform = L.transform(DEV)
    for step, (numeric, strings, labels) in enumerate(_batches(L, B, steps, 700)):
        loss_e = float(eng.step(numeric, strings, labels))
        accepted, version, loss_d = trainer.train_minibatch(M.twin_features(L, numeric, strings, transform), labels)
        assert accepted and version == step + 1
        assert abs(loss_e - float(loss_d)) <= 1e-4 * max(1.0, abs(loss_e)), (step, loss_e, float(loss_d))
    torch.cuda.synchronize()
    group_d.check()
    assert trainer.graph_fallback_reason is None and isinstance(trainer._graph_state, dict)
    de, dd = group_e.pull_dense(M.MLP_NAMES), group_d.pull_dense(M.MLP_NAMES)
    for n in M.MLP_NAMES:
        torch.testing.assert_close(de[n], dd[n], rtol=1e-4, atol=1e-6)
    for n, ids in zip(L.table_names, _all_ids(L)):
        torch.testing.assert_close(group_e.pull_rows([(n, ids)])[0], group_d.pull_rows([(n, ids)])[0],
                                   rtol=1e-4, atol=1e-6)


def _four_workers(model, opt, B):
    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(2, opt_type, opt_args, device=0)
    engines = [M.FeatureColumnDNNEngine(group, model, B, lr, seed=5, register=(w == 0)) for w in range(4)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(4)]
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.capture()
    torch.cuda.synchronize()
    return group, engines, streams, lr


def test_four_workers_concurrent():
    B, steps = 256, 20
    group, engines, streams, _ = _four_workers("census_dnn_model", "sgd", B)
    data = [_batches(M.CENSUS_DNN, B, 4, 1000 * (w + 1)) for w in range(4)]
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


@pytest.mark.parametrize("model", MODELS)
def test_four_workers_serialised_match_oracle(model):
    B, rounds = 256, 3
    group, engines, streams, lr = _four_workers(model, "adam", B)
    servers = _servers(group, engines[0], "adam")
    data = [_batches(engines[0].layout, B, rounds, 1000 * (w + 1)) for w in range(4)]
    for r in range(rounds):
        for w in range(4):
            with torch.cuda.stream(streams[w]):
                engines[w].replay(*data[w][r])
            streams[w].synchronize()
            _push_to_oracle(servers, engines[w], lr)
    _compare_state(group, servers, engines[0], "adam")
    assert [v for v, _, _ in group.snapshot()] == [4 * rounds] * 2
