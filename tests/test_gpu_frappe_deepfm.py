"""The frappe DeepFM tower (csrc/frappe_tower.cu, include/b200_frappe.h) and FrappeDeepFMEngine against the float64
oracle of oracle/frappe_oracle.py.

Kernel level: batches at the tile edges, 4096, 32768 and one sample past a full persistent grid's first pass, on
uniform, per-field Zipf, 30 % padded, all-padding and one-hot-row batches; id 0's rows exactly 0; the comparator's
mutations; repeated launches and graph replay within the bound (the header promises no bit-determinism); the
refusals.  Engine level: SGD / Adam x hashed / bounded x 1 / 2 shards against OracleServer fed the engine's own
gradients; replay against step, predict against the training logits; the engine against the drop-in trainer
over FrappeDeepFM; a sanity run on a teacher-labelled task."""
import numpy as np
import pytest
import torch

from elasticdl_b200 import ops
from elasticdl_b200._lib import PSRangeError
from elasticdl_b200.ps import PSGroup
from elasticdl_b200.workloads import frappe as FR
from oracle import frappe_oracle as O
from oracle.ps_oracle import EmbeddingTableInfo, OracleServer

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
OPTS = {"sgd": ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", 0.1),
        "adam": ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", 1e-3)}


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ids(B, pattern, seed):
    if pattern == "uniform":
        g = torch.Generator(device=DEV).manual_seed(seed)
        u = torch.rand((B, 10), generator=g, device=DEV)
        size = torch.tensor(FR.FIELD_SIZES, device=DEV, dtype=torch.float32)
        return (u * size).long().clamp(max=size.long() - 1) + torch.tensor(FR.FIELD_START, device=DEV)
    if pattern == "all_pad":
        return torch.zeros((B, 10), dtype=torch.int64, device=DEV)
    if pattern == "hot":  # one id in every position of every sample
        return torch.full((B, 10), 5041, dtype=torch.int64, device=DEV)
    return FR.synthetic_frappe_batch(B, seed, DEV, pad_fraction=0.3 if pattern == "pad30" else 0.0)[0]


def _inputs(B, pattern, seed):
    ids = _ids(B, pattern, seed).contiguous()
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    table_d = (torch.rand((FR.INPUT_DIM, 64), generator=g, device=DEV) * 2 - 1) * 0.5
    table_w = (torch.rand((FR.INPUT_DIM, 1), generator=g, device=DEV) * 2 - 1) * 0.5
    labels = (torch.rand(B, generator=g, device=DEV) < 0.3).float()
    flat = O.random_params(g, DEV)
    uniq, inv, n = ops.unique(ids.reshape(-1), 1)
    U = int(n.item())
    bet_d = torch.zeros((10 * B, 64), device=DEV)
    bet_w = torch.zeros((10 * B, 1), device=DEV)
    bet_d[:U] = table_d[uniq[:U]]
    bet_w[:U] = table_w[uniq[:U]]
    return ids, inv, n, bet_d, bet_w, labels, flat, U


def _run(inputs):
    ids, inv, n, bet_d, bet_w, labels, flat, U = inputs
    out = FR.frappe_tower(ids, inv, n, bet_d, bet_w, labels, flat)
    ref = O.frappe_reference(ids, inv, U, bet_d, bet_w, labels, flat)
    got = {"logits": out["logits"], "loss": out["loss"], "grads": out["grads"], "gsum_deep": out["gsum_deep"][:U],
           "gsum_wide": out["gsum_wide"][:U]}
    return got, ref


BATCHES = [1, 63, 64, 65, 4096, 32768, "wave+1"]


def _b(B):
    return 2 * _n_sm() * FR.TILE + 1 if B == "wave+1" else B


@pytest.mark.parametrize("pattern", ["uniform", "zipf", "pad30", "all_pad", "hot"])
@pytest.mark.parametrize("B", BATCHES)
def test_tower_matches_oracle(B, pattern):
    Bn = _b(B)
    got, ref = _run(_inputs(Bn, pattern, seed=Bn % 997))
    O.check(got, ref, label="B=%d %s" % (Bn, pattern))
    pad = ref["row_id"] == 0
    assert bool((got["gsum_deep"][pad] == 0).all()) and bool((got["gsum_wide"][pad] == 0).all())
    if pattern == "all_pad" or (pattern == "pad30" and Bn >= 64):
        assert bool(pad.any())


@pytest.mark.parametrize("B", [64, 4096])
def test_mutations_are_caught(B):
    inputs = _inputs(B, "pad30", seed=5)
    got, ref = _run(inputs)
    assert not O.caught_by(got, ref)
    ids, inv, n, bet_d, bet_w, labels, flat, U = inputs
    for name, mut in O.mutations(ref, (ids, inv, U, bet_d, bet_w, labels, flat)).items():
        if name == "drop_one_sample" and B > 64:
            continue  # one sample of 4096 moves each batch sum by less than the sqrt(n)-scaled bound
        assert O.caught_by(mut, ref), (name, B)


def test_repeated_launches_and_graph_replay():
    B = 32768
    ids, inv, n, bet_d, bet_w, labels, flat, U = _inputs(B, "pad30", seed=9)
    ref = O.frappe_reference(ids, inv, U, bet_d, bet_w, labels, flat)
    call = FR.FrappeTowerCall(B, DEV)
    args = (ids, inv, n, bet_d, bet_w, labels, flat)

    def got():
        o = call.outputs(U)
        return {k: o[k].clone() for k in O.FAMILIES}

    call.launch(*args)
    first = got()
    call.launch(*args)
    second = got()
    assert torch.equal(first["logits"], second["logits"])  # per-sample, fixed order
    for o in (first, second):
        O.check(o, ref, label="eager")
    for b in (call.loss, call.logits, call.grads, call.gsum_deep, call.gsum_wide):
        b.fill_(float("nan"))
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call.launch(*args)
    for _ in range(2):  # the accumulators and the arrival counter are back at zero after every replay
        graph.replay()
        torch.cuda.synchronize()
        O.check(got(), ref, label="replay")


def test_refusals():
    B = 64
    ids, inv, n, bet_d, bet_w, labels, flat, U = _inputs(B, "zipf", seed=1)
    with pytest.raises(ValueError, match="ids must be"):
        FR.frappe_tower(ids.int(), inv, n, bet_d, bet_w, labels, flat)
    with pytest.raises(ValueError, match="ids must be"):
        FR.frappe_tower(ids[:, :9].contiguous(), inv, n, bet_d, bet_w, labels, flat)
    with pytest.raises(ValueError, match="inv must be"):
        FR.frappe_tower(ids, inv.long(), n, bet_d, bet_w, labels, flat)
    with pytest.raises(ValueError, match="labels must be"):
        FR.frappe_tower(ids, inv, n, bet_d, bet_w, labels.double(), flat)
    with pytest.raises(ValueError, match="params must be"):
        FR.frappe_tower(ids, inv, n, bet_d, bet_w, labels, flat[:-1])
    with pytest.raises(ValueError, match="batch size"):
        FR.FrappeTowerCall(0, DEV)
    opt_type, opt_args, lr = OPTS["sgd"]
    with pytest.raises(ValueError, match="sync-SGD"):
        FR.FrappeDeepFMEngine(PSGroup(1, opt_type, opt_args, device=0, use_async=False), B, lr)
    with pytest.raises(ValueError, match="lr_staleness_modulation"):
        FR.FrappeDeepFMEngine(PSGroup(1, opt_type, opt_args, device=0, lr_staleness_modulation=True), B, lr)
    with pytest.raises(ValueError, match="batch size"):
        FR.FrappeDeepFMEngine(PSGroup(1, opt_type, opt_args, device=0), 0, lr)
    eng = FR.FrappeDeepFMEngine(PSGroup(1, opt_type, opt_args, device=0), B, lr, input_dim=FR.INPUT_DIM)
    with pytest.raises(ValueError, match="ids must be"):
        eng.step(ids.int(), labels)
    with pytest.raises(ValueError, match="labels must be"):
        eng.step(ids, labels[:-1])
    bad = ids.clone()
    bad[3, 4] = FR.INPUT_DIM
    eng.step(bad, labels)
    with pytest.raises(PSRangeError):
        eng.check()
    eng.check()  # the error was cleared
    eng.step(ids, labels)
    eng.check()


# ---------------------------------------------------------------------------------------------------- engine
def _batches(B, n, seed):
    return [FR.synthetic_frappe_batch(B, seed + s, DEV, pad_fraction=0.3) for s in range(n)]


def _table_names():
    return [(FR.DEEP_NAME, 64), (FR.WIDE_NAME, 1)]


def _make_engine(opt, hashed, n_shards, B, seed=3):
    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(n_shards, opt_type, opt_args, device=0)
    eng = FR.FrappeDeepFMEngine(group, B, lr, input_dim=None if hashed else FR.INPUT_DIM, seed=seed,
                                expected_rows=1 << 14)
    return group, eng, lr


def _create_rows(group, data):
    """Hashed tables: create every row the batches use (their first pull draws the initial values); returns the
    ids and {name: rows}."""
    ids = torch.unique(torch.cat([i.reshape(-1) for i, _ in data]))
    rows = group.pull_rows([(n, ids) for n, _ in _table_names()])
    return ids, {n: r for (n, _), r in zip(_table_names(), rows)}


def _servers(group, eng, opt, hashed, data):
    opt_type, opt_args, _ = OPTS[opt]
    N = group.n_shards
    servers = [OracleServer(s, opt_type, opt_args, num_ps=N) for s in range(N)]
    names = FR.DENSE_NAMES + ([] if hashed else [n for n, _ in _table_names()])
    state = group.pull_dense(names)
    ids, rows = _create_rows(group, data) if hashed else (None, None)
    for s, srv in enumerate(servers):
        dense = {n: state[n].cpu().numpy() for n in names if eng.owner[n] == s}
        if hashed:
            m = (ids % N == s)
            infos = [EmbeddingTableInfo(n, d, "zero", None) for n, d in _table_names()]
            tables = {n: (ids[m].cpu().numpy(), rows[n][m].cpu().numpy()) for n, _ in _table_names()}
            srv.push_model(dense=dense, infos=infos, tables=tables)
        else:
            srv.push_model(dense=dense)
    return servers, ids


def _oracle_flat(servers, eng):
    flat = torch.zeros(FR.N_PARAMS, dtype=torch.float32)
    v = FR.flat_views(flat)
    for n in FR.DENSE_NAMES:
        v[n].copy_(torch.from_numpy(servers[eng.owner[n]].dense[n]).view(v[n].shape))
    return flat


def _push_to_oracle(servers, eng, lr, hashed):
    U = int(eng.n_unique.item())
    t = eng.tower
    uniq = eng.uniq[:U].cpu().numpy().astype(np.int64)
    N = len(servers)
    per = {s: ({}, {}) for s in range(N)}
    for n, s in FR.DENSE_PARAMS:
        o = FR.OFFSETS[n]
        per[eng.owner[n]][0][n] = t.grads[o:o + int(np.prod(s))].cpu().numpy().reshape(s)
    for (n, _), gs in zip(_table_names(), (t.gsum_deep, t.gsum_wide)):
        g = np.ascontiguousarray(gs[:U].cpu().numpy())
        if hashed:
            for s in range(N):
                m = uniq % N == s
                per[s][1][n] = (uniq[m], g[m])
        else:
            per[eng.owner[n]][1][n] = (uniq, g)
    for s, srv in enumerate(servers):
        ok, _ = srv.push_gradients(per[s][0], per[s][1], lr, 0)
        assert ok


def _compare_state(group, servers, eng, opt, hashed, ids):
    N = group.n_shards
    state = group.pull_dense(FR.DENSE_NAMES)
    for n in FR.DENSE_NAMES:
        srv = servers[eng.owner[n]]
        np.testing.assert_allclose(state[n].cpu().numpy(), srv.dense[n], rtol=1e-6, atol=1e-8, err_msg=n)
        if opt == "adam":
            for k, sn in enumerate(("m", "v")):
                np.testing.assert_allclose(group.slot_dense(n, k + 1).cpu().numpy(), srv.opt.dense_slots[sn][n],
                                           rtol=1e-5, atol=1e-12, err_msg=(n, sn))
    for n, _ in _table_names():
        if hashed:
            ids_np = ids.cpu().numpy()
            for s in range(N):
                m = ids_np % N == s
                mine = ids[torch.from_numpy(m).to(DEV)]
                srv = servers[s]
                np.testing.assert_allclose(group.pull_rows([(n, mine)])[0].cpu().numpy(), srv.tables[n].get(ids_np[m]),
                                           rtol=1e-6, atol=1e-8, err_msg=n)
                if opt == "adam":
                    for k, sn in enumerate(("m", "v")):
                        np.testing.assert_allclose(group.slot_rows(n, mine, k + 1).cpu().numpy(),
                                                   srv.opt.table_slots[sn][n].get(ids_np[m]),
                                                   rtol=1e-5, atol=1e-12, err_msg=(n, sn))
        else:
            srv = servers[eng.owner[n]]
            np.testing.assert_allclose(group.pull_dense([n])[n].cpu().numpy(), srv.dense[n], rtol=1e-6, atol=1e-8,
                                       err_msg=n)
            if opt == "adam":
                for k, sn in enumerate(("m", "v")):
                    np.testing.assert_allclose(group.slot_dense(n, k + 1).cpu().numpy(), srv.opt.dense_slots[sn][n],
                                               rtol=1e-5, atol=1e-12, err_msg=(n, sn))
    assert [v for v, _, _ in group.snapshot()] == [srv.version for srv in servers]


def _row0(group, hashed, name):
    if hashed:
        return group.pull_rows([(name, torch.zeros(1, dtype=torch.int64, device=DEV))])[0][0].clone()
    return group.pull_dense([name])[name][0].clone()


@pytest.mark.parametrize("n_shards", [1, 2])
@pytest.mark.parametrize("hashed", [True, False])
@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_engine_matches_oracle(opt, hashed, n_shards):
    B, steps = 256, 5
    group, eng, lr = _make_engine(opt, hashed, n_shards, B)
    if n_shards == 2:
        assert len({eng.owner[n] for n in eng.owner}) == 2
    data = _batches(B, steps, 300)
    servers, ids_all = _servers(group, eng, opt, hashed, data)
    row0 = _row0(group, hashed, FR.DEEP_NAME)
    for step, (ids, labels) in enumerate(data):
        before = _oracle_flat(servers, eng)
        loss = eng.step(ids, labels)
        torch.cuda.synchronize()
        eng.check()
        torch.testing.assert_close(eng.flat.cpu(), before, rtol=0, atol=0)
        U = int(eng.n_unique.item())
        ref = O.frappe_reference(ids, eng.inv, U, eng.bet_deep, eng.bet_wide, labels, eng.flat)
        out = eng.tower.outputs(U)
        O.check({k: out[k] for k in O.FAMILIES}, ref, label="step %d" % step)
        assert abs(float(loss) - float(ref["loss"])) <= 1e-5 * float(ref["M"]["loss"])
        _push_to_oracle(servers, eng, lr, hashed)
    torch.cuda.synchronize()
    _compare_state(group, servers, eng, opt, hashed, ids_all)
    assert [v for v, _, _ in group.snapshot()] == [steps] * n_shards
    # id 0 is pushed with a zero gradient every step; from zero slots neither optimizer moves it
    assert torch.equal(_row0(group, hashed, FR.DEEP_NAME), row0)


@pytest.mark.parametrize("hashed", [True, False])
def test_replay_equals_step_and_predict(hashed):
    B = 200
    data = _batches(B, 4, 50)
    _, ea, _ = _make_engine("adam", hashed, 2, B, seed=4)
    ga, eb, _ = _make_engine("adam", hashed, 2, B, seed=4)
    if hashed:  # the same initial rows in both groups
        ids, rows = _create_rows(ea.group, data)
        eb.group.set_rows([(n, ids, rows[n]) for n, _ in _table_names()])
    for ids, labels in data:
        logits = ea.predict(ids)
        ea.step(ids, labels)
        torch.cuda.synchronize()
        assert torch.equal(logits, ea.tower.logits)  # the forward instance gives the training instance's logits
        eb.replay(ids, labels)
    torch.cuda.synchronize()
    ea.check()
    eb.check()
    names = FR.DENSE_NAMES
    sa, sb = ea.group.pull_dense(names), eb.group.pull_dense(names)
    for n in names:  # float atomics: the same within rounding, not bit for bit
        torch.testing.assert_close(sa[n], sb[n], rtol=1e-4, atol=1e-6)
    ids = torch.unique(torch.cat([i.reshape(-1) for i, _ in data]))
    for n, _ in _table_names():
        if hashed:
            ra, rb = ea.group.pull_rows([(n, ids)])[0], eb.group.pull_rows([(n, ids)])[0]
        else:
            ra, rb = ea.group.pull_dense([n])[n], eb.group.pull_dense([n])[n]
        torch.testing.assert_close(ra, rb, rtol=1e-4, atol=1e-6)
    assert ea.graph is None and eb.graph is not None
    eb.set_lr(5e-4)
    eb.replay(*data[0])  # a new learning rate re-captures
    assert eb._graph_lr == 5e-4


@pytest.mark.parametrize("hashed", [True, False])
def test_engine_matches_dropin_trainer(hashed):
    import types

    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    B, steps = 128, 5
    data = _batches(B, steps, 700)
    group_e, eng, lr = _make_engine("sgd", hashed, 1, B, seed=6)
    opt_type, opt_args, _ = OPTS["sgd"]
    group_d = PSGroup(1, opt_type, opt_args, device=0)
    model = FR.FrappeDeepFM(lr, input_dim=None if hashed else FR.INPUT_DIM).to(DEV)
    model.load_mlp(torch.cat([group_e.pull_dense([n])[n].reshape(-1) for n in FR.DENSE_NAMES]))
    client = PSClient(group_d)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(cuda_graph=True))
    if hashed:
        ids, rows = _create_rows(group_e, data)
    else:
        ids = torch.arange(FR.INPUT_DIM, device=DEV)
        rows = group_e.pull_dense([n for n, _ in _table_names()])
    group_d.set_rows([(n, ids, rows[n]) for n, _ in _table_names()])
    for step, (x, labels) in enumerate(data):
        loss_e = float(eng.step(x, labels))
        accepted, version, loss_d = trainer.train_minibatch(x, labels)
        assert accepted and version == step + 1
        assert abs(loss_e - float(loss_d)) <= 1e-5 * max(1.0, abs(loss_e)), (step, loss_e, float(loss_d))
    torch.cuda.synchronize()
    eng.check()
    group_d.check()
    assert trainer.graph_fallback_reason is None and isinstance(trainer._graph_state, dict)
    de, dd = group_e.pull_dense(FR.DENSE_NAMES), group_d.pull_dense(FR.DENSE_NAMES)
    for n in FR.DENSE_NAMES:
        torch.testing.assert_close(de[n], dd[n], rtol=1e-4, atol=1e-6)
    for n, _ in _table_names():
        re = group_e.pull_rows([(n, ids)])[0] if hashed else group_e.pull_dense([n])[n]
        torch.testing.assert_close(re, group_d.pull_rows([(n, ids)])[0], rtol=1e-4, atol=1e-6)


def test_sanity_teacher_task():
    """200 SGD 0.1 steps of batch 64 on batches labelled by a fixed random teacher of the same model (the task the
    CPU oracle learns in tests/test_oracle_frappe_deepfm.py) reach the reference's 0.65 held-out accuracy."""
    ref_ids, _ = FR.synthetic_frappe_batch(8192, 12345, "cpu", pad_fraction=0.1)
    teacher = O.make_teacher(0, ref_ids)
    group, eng, _ = _make_engine("sgd", True, 1, 64, seed=0)
    for step in range(200):
        ids, _ = FR.synthetic_frappe_batch(64, 100 + step, DEV, pad_fraction=0.1)
        eng.replay(ids, O.teacher_labels(teacher, ids))
    torch.cuda.synchronize()
    eng.check()
    hits, n = 0, 0
    for k in range(8):
        ids, _ = FR.synthetic_frappe_batch(64, 10_000 + k, DEV, pad_fraction=0.1)
        y = O.teacher_labels(teacher, ids)
        hits += int(((eng.predict(ids) > 0).float() == y).sum())
        n += 64
    assert hits / n > 0.65, hits / n
