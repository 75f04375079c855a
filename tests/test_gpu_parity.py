"""GPU parity tests: the CUDA path (through the C ABI, via PSGroup/PSClient)
against the CPU oracle on the same seeded inputs.  Bit-exact for ids / gathers /
integer work; fp32 optimizer state within 1e-5 relative (BASELINE.json
north_star), and bit-exact where no duplicate-id summation is involved."""
import numpy as np
import pytest
import torch

from oracle import ps_oracle as O

pytestmark = pytest.mark.gpu
F = np.float32

OPTS = {
    "sgd": ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;"),
    "momentum": ("SGD", "learning_rate=0.1;momentum=0.9;nesterov=false;"),
    "nesterov": ("SGD", "learning_rate=0.1;momentum=0.9;nesterov=true;"),
    "adam": ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;"),
    "amsgrad": ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=true;"),
    "adagrad": ("Adagrad", "learning_rate=0.1;epsilon=1e-07;"),
    "ftrl": ("Ftrl", "learning_rate=0.1;initial_accumulator_value=0.1;l1_regularization_strength=0.01;"
                     "l2_regularization_strength=0.02;l2_shrinkage_regularization_strength=0.0;beta=0.0;"),
    "ftrl_shrink": ("Ftrl", "learning_rate=0.05;initial_accumulator_value=0.1;l1_regularization_strength=0.0;"
                            "l2_regularization_strength=0.0;l2_shrinkage_regularization_strength=0.1;beta=0.5;"),
}


def make_pair(n_shards, opt="sgd", **kw):
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient

    ot, oa = OPTS[opt]
    group = PSGroup(n_shards, ot, oa, device=0, **kw)
    client = PSClient(group)
    servers = [O.OracleServer(i, ot, oa, num_ps=n_shards,
                              lr_staleness_modulation=kw.get("lr_staleness_modulation", False),
                              reproduce_q1=kw.get("reproduce_q1", False)) for i in range(n_shards)]
    return group, client, O.OraclePSClient(servers)


def info(name, dim, init="zero", capacity=1000):
    from elasticdl_b200.common.tensor_utils import EmbeddingTableInfo

    return EmbeddingTableInfo(name, dim, init, 1, capacity)


def oinfo(name, dim, init="zero"):
    return O.EmbeddingTableInfo(name, dim, init, 1)


def close(a, b, rtol=1e-5, atol=1e-7):
    return np.allclose(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), rtol=rtol, atol=atol)


# ------------------------------------------------------------------ pull (bit exact)
@pytest.mark.parametrize("n_shards", [1, 2, 3, 8])
@pytest.mark.parametrize("dim", [1, 4, 8, 10, 64])
def test_pull_bit_exact(n_shards, dim):
    group, client, oc = make_pair(n_shards)
    rng = np.random.RandomState(n_shards * 100 + dim)
    cap = 5000
    client.push_embedding_table_infos([info("emb", dim, capacity=cap)])
    oc.push_embedding_table_infos([oinfo("emb", dim)])
    ids = rng.permutation(cap)[:3000].astype(np.int64)
    vals = rng.randn(3000, dim).astype(F)
    group.set_rows([("emb", ids, vals)])
    for s in oc.servers:
        m = ids % n_shards == s.id
        s.tables["emb"].set(ids[m], vals[m])
    q = rng.choice(ids, size=4096).astype(np.int64)  # with repeats, arbitrary order
    got = client.pull_embedding_vectors("emb", q)
    want = oc.pull_embedding_vectors("emb", q)
    assert got.dtype == np.float32 and got.shape == (4096, dim)
    assert np.array_equal(got, want)
    # never-written rows of a "zero" table read back as zeros and become created rows
    fresh = np.setdiff1d(np.arange(cap), ids)[:50].astype(np.int64)
    assert np.array_equal(client.pull_embedding_vectors("emb", fresh), np.zeros((50, dim), dtype=F))
    assert group.table_size("emb") == len(np.unique(np.concatenate([ids, fresh])))
    # torch in -> torch out, same bits
    tq = torch.from_numpy(q).cuda()
    assert np.array_equal(client.pull_embedding_vectors("emb", tq).cpu().numpy(), want)
    group.close()


def test_pull_ordering_worker_ps_interaction_test_py_153():
    group, client, _ = make_pair(2)
    client.push_embedding_table_infos([info("emb", 8, capacity=16)])
    all_ids = np.arange(11, dtype=np.int64)
    group.set_rows([("emb", all_ids, np.repeat(all_ids[:, None], 8, 1).astype(F))])
    ids = [3, 5, 1, 6, 10, 2, 1, 2, 4, 7, 9]
    out = client.pull_embedding_vectors("emb", ids)
    assert np.array_equal(out, np.repeat(np.array(ids)[:, None], 8, 1).astype(F))
    group.close()


def test_uniform_initializer_matches_oracle_generator():
    from elasticdl_b200.ps.group import table_seed

    group, client, _ = make_pair(3, seed=11)
    client.push_embedding_table_infos([info("u", 8, "uniform", capacity=999), info("RandomUniform", 8, "RandomUniform")])
    ids = np.array([0, 1, 2, 500, 998, 7], dtype=np.int64)
    got = client.pull_embedding_vectors("u", ids)
    seed = table_seed(11, "u")
    want = np.array([[O.lib.oracle_uniform_init(seed, int(i), c) for c in range(8)] for i in ids], dtype=F)
    assert np.array_equal(got, want)
    assert got.min() >= -0.05 and got.max() < 0.05
    # quirk Q6: any initializer string other than the literal "uniform" zero-fills
    assert not client.pull_embedding_vectors("RandomUniform", ids).any()
    group.close()


# ------------------------------------------------------------------ unique / dedup
@pytest.mark.parametrize("k,hi,T", [(7, 9, 1), (1000, 50, 1), (4096, 100000, 3), (100000, 3000, 2), (1, 5, 4)])
def test_unique_first_occurrence(k, hi, T):
    group, _, _ = make_pair(1)
    rng = np.random.RandomState(k + hi)
    ids = rng.randint(0, hi, size=(T, k)).astype(np.int64)
    if k == 7:
        ids[0] = [0, 1, 3, 8, 3, 2, 3]  # layer_test.py:135 vector
    uniq, inv, n = group.unique(torch.from_numpy(ids).cuda().view(-1), T)
    uniq, inv, n = uniq.cpu().numpy().reshape(T, k), inv.cpu().numpy().reshape(T, k), n.cpu().numpy()
    for t in range(T):
        wu, wi = O.unique_first_occurrence(ids[t])
        assert n[t] == len(wu)
        assert np.array_equal(uniq[t, : n[t]], wu)
        assert np.array_equal(inv[t], wi)
    group.close()


@pytest.mark.parametrize("dim", [1, 4, 8, 10])
def test_segment_sum_matches_dedup(dim):
    group, _, _ = make_pair(1)
    rng = np.random.RandomState(dim)
    k = 20000
    ids = rng.zipf(1.3, size=k).astype(np.int64) % 4000
    vals = rng.randn(k, dim).astype(F)
    uniq, inv, n = group.unique(torch.from_numpy(ids).cuda(), 1)
    out = group.segment_sum(torch.from_numpy(vals).cuda(), inv, 1, k, dim).cpu().numpy().reshape(k, dim)
    wv, wi = O.deduplicate_indexed_slices(vals, ids)
    u = int(n.item())
    assert u == len(wi) and np.array_equal(uniq.cpu().numpy()[:u], wi)
    # hot ids are summed thousands of times in a different (atomic) order than the oracle's
    # left-to-right loop: both are within the fp32 accumulation bound of the exact sum
    exact = np.zeros((u, dim), dtype=np.float64)
    mag = np.zeros((u, dim), dtype=np.float64)
    rank = {int(x): r for r, x in enumerate(wi)}
    r_of = np.array([rank[int(x)] for x in ids])
    np.add.at(exact, r_of, vals.astype(np.float64))
    np.add.at(mag, r_of, np.abs(vals).astype(np.float64))
    bound = 4e-6 * mag + 1e-7
    assert np.all(np.abs(out[:u] - exact) <= bound)
    assert np.all(np.abs(wv - exact) <= bound)
    few = np.bincount(r_of, minlength=u) <= 4  # lightly duplicated ids: 1e-5 relative
    assert np.allclose(out[:u][few], wv[few], rtol=1e-5, atol=1e-6)
    assert not out[u:].any()
    # no duplicates -> bit exact
    ids2 = rng.permutation(50000)[:k].astype(np.int64)
    uniq, inv, n = group.unique(torch.from_numpy(ids2).cuda(), 1)
    out = group.segment_sum(torch.from_numpy(vals).cuda(), inv, 1, k, dim).cpu().numpy().reshape(k, dim)
    assert np.array_equal(out, vals)
    g = group.gather_rows(torch.from_numpy(vals).cuda(), inv, 1, k, dim).cpu().numpy().reshape(k, dim)
    assert np.array_equal(g, vals)
    group.close()


# ------------------------------------------------------------------ push: all optimizers
def _setup_model(client, oc, rng, dims=(1, 8, 10)):
    from elasticdl_b200.common.tensor_utils import Tensor

    client.push_embedding_table_infos([info("e%d" % d, d, capacity=500) for d in dims])
    oc.push_embedding_table_infos([oinfo("e%d" % d, d) for d in dims])
    dense = {"t1": rng.randn(2, 3).astype(F), "t2": rng.randn(64, 8).astype(F), "bias": rng.randn(7).astype(F),
             "big": rng.randn(1000, 16).astype(F)}
    for c in (client, oc):
        c.partition_dense_parameters(dense.keys())
        for ps_id in range(c.ps_num):
            params = [(Tensor if c is client else O.Tensor)(n, v.copy(), None) for n, v in dense.items()]
            if any(c.parameter_to_ps[n] == ps_id for n in dense):
                c.push_dense_parameters(params, ps_id, 0)
            else:
                # shards without dense params still need Initialized for parity of pull
                pass
    return dense


def _grads(rng, dims, step, dup):
    from elasticdl_b200.common.tensor_utils import Tensor

    dense = [("t1", rng.randn(2, 3).astype(F)), ("t2", rng.randn(64, 8).astype(F) if step % 2 else None),
             ("bias", rng.randn(7).astype(F)), ("big", rng.randn(1000, 16).astype(F))]
    sparse_dense = ("t2", rng.randn(20, 8).astype(F),
                    (rng.randint(0, 64, 20) if dup else rng.permutation(64)[:20]).astype(np.int64))
    edl = []
    for d in dims:
        k = 300
        ids = (rng.randint(0, 200, k) if dup else rng.permutation(500)[:k]).astype(np.int64)
        edl.append(("e%d" % d, rng.randn(k, d).astype(F), ids))
    def build(T):
        grads = [T(n, v.copy(), None) for n, v in dense if v is not None]
        if not step % 2:
            grads.append(T(sparse_dense[0], sparse_dense[1].copy(), sparse_dense[2].copy()))
        return grads, [T(n, v.copy(), i.copy()) for n, v, i in edl]
    return build(Tensor), build(O.Tensor)


@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("n_shards", [1, 3])
@pytest.mark.parametrize("dup", [False, True])
def test_push_gradients_all_optimizers(opt, n_shards, dup):
    group, client, oc = make_pair(n_shards, opt)
    import zlib
    rng = np.random.RandomState(zlib.crc32(repr((opt, n_shards, dup)).encode()))
    dims = (1, 8, 10)
    dense = _setup_model(client, oc, rng, dims)
    versions, oversions = [0] * n_shards, [0] * n_shards
    for step in range(4):
        (grads, edl), (ograds, oedl) = _grads(rng, dims, step, dup)
        lr = 0.05 if step == 2 else 0.0  # 0 -> optimizer's own lr (server.go:183-187)
        acc, v = client.push_gradients(grads, edl, lr, versions)
        oacc, ov = oc.push_gradients(ograds, oedl, lr, oversions)
        assert (acc, v) == (oacc, ov) == (True, step + 1)
        versions = [v] * n_shards
        oversions = [ov] * n_shards
    state = group.snapshot()
    assert [s[0] for s in state] == [4] * n_shards and [s[1] for s in state] == [4] * n_shards
    exact = not dup
    cmp = (lambda a, b: np.array_equal(a, b)) if exact else (lambda a, b: close(a, b, 1e-5, 1e-6))
    n_slots = len(oc.servers[0].opt.slot_names)
    for name in dense:
        ps = oc.parameter_to_ps[name]
        assert client.parameter_to_ps[name] == ps
        srv = oc.servers[ps]
        got = group.pull_dense([name])[name].cpu().numpy()
        assert cmp(got, srv.dense[name]), name
        for k, sn in enumerate(srv.opt.slot_names):
            gs = group.slot_dense(name, k + 1).cpu().numpy()
            assert cmp(gs, srv.opt.dense_slots[sn][name]), (name, sn)
    all_ids = np.arange(500, dtype=np.int64)
    for d in dims:
        name = "e%d" % d
        got = client.pull_embedding_vectors(name, all_ids)
        for s in oc.servers:
            m = all_ids % n_shards == s.id
            touched = np.isin(all_ids[m], s.tables[name].keys())
            ids_t = all_ids[m][touched]
            assert cmp(got[m][touched], s.tables[name].get(ids_t)), name
            assert not got[m][~touched].any()
            for k, sn in enumerate(s.opt.slot_names):
                gs = group.slot_rows(name, ids_t, k + 1).cpu().numpy()
                assert cmp(gs, s.opt.table_slots[sn][name].get(ids_t)), (name, sn)
    assert n_slots == {"sgd": 0, "momentum": 1, "nesterov": 1, "adam": 2, "amsgrad": 3, "adagrad": 1,
                       "ftrl": 2, "ftrl_shrink": 2}[opt]
    group.close()


# ------------------------------------------------------------------ reference golden vectors on the GPU path
def test_gpu_sgd_optimizer_test_go_25():
    from elasticdl_b200.common.tensor_utils import Tensor

    group, client, _ = make_pair(1, "sgd")
    client.partition_dense_parameters(["t1", "t2"])
    client.push_dense_parameters([Tensor("t1", np.array([[1, 2, 3], [4, 5, 6]], dtype=F), None),
                                  Tensor("t2", np.array([[1, 2], [1.1, 2.2]], dtype=F), None)], 0, 0)
    g1, g2 = np.ones((2, 3), dtype=F), np.ones((2, 2), dtype=F)
    client.push_gradients([Tensor("t1", g1, None), Tensor("t2", g2, None)], [], 0.05, [0])
    d = group.pull_dense(["t1", "t2"])
    assert close(d["t1"].cpu().numpy().ravel(), [0.95, 1.95, 2.95, 3.95, 4.95, 5.95], 1e-4)
    assert close(d["t2"].cpu().numpy().ravel(), [0.95, 1.95, 1.05, 2.15], 1e-4)
    with pytest.raises(KeyError):
        client.push_gradients([Tensor("t3", g2, None)], [], 0.1, [1])
    client.push_embedding_table_infos([info("t3", 2, capacity=16)])
    client.push_gradients([Tensor("t1", g1, None), Tensor("t2", g2, None)],
                          [Tensor("t3", np.ones((2, 2), dtype=F), np.array([1, 3]))], 0.1, [1])
    d = group.pull_dense(["t1", "t2"])
    assert close(d["t1"].cpu().numpy().ravel(), [0.85, 1.85, 2.85, 3.85, 4.85, 5.85], 1e-4)
    assert close(client.pull_embedding_vectors("t3", [1, 3]).ravel(), [-0.1] * 4, 1e-4)
    # ids [1,3,3,5]: the raw Go kernel applies duplicates sequentially, the PSClient sums
    # them first (ps_client.py:255-257) -- identical for SGD: -0.2, -0.3, -0.1
    client.push_gradients([], [Tensor("t3", np.ones((4, 2), dtype=F), np.array([1, 3, 3, 5]))], 0.1, [2])
    assert close(client.pull_embedding_vectors("t3", [1, 3, 5]).ravel(), [-0.2, -0.2, -0.3, -0.3, -0.1, -0.1], 1e-4)
    group.close()


def test_gpu_adam_global_step_optimizer_test_go_118():
    from elasticdl_b200.common.tensor_utils import Tensor

    ot, oa = "Adam", "learning_rate=0.1;beta_1=0.9;beta_2=0.999;epsilon=1e-08;amsgrad=false;"
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient

    group = PSGroup(1, ot, oa, device=0)
    client = PSClient(group)
    client.partition_dense_parameters(["t1", "t2"])
    client.push_dense_parameters([Tensor("t1", np.array([[1, 2, 3], [4, 5, 6]], dtype=F), None),
                                  Tensor("t2", np.array([[1, 2], [1.1, 2.2]], dtype=F), None)], 0, 0)
    client.push_embedding_table_infos([info("t3", 2, capacity=16)])
    group.set_shard_state(0, step=1)  # optimizer_test.go:150 opt.step = 1
    g1, g2 = np.ones((2, 3), dtype=F), np.ones((2, 2), dtype=F)
    client.push_gradients([Tensor("t1", g1, None), Tensor("t2", g2, None)], [], 0.0, [0])  # step 2
    off = np.arange(6)
    assert close(group.pull_dense(["t1"])["t1"].cpu().numpy().ravel(), 0.9255863187 + off, 1e-4)
    with pytest.raises(KeyError):  # failed call still bumps the step (quirk Q2) -> 3
        client.push_gradients([], [Tensor("nope", g2, np.array([0, 1]))], 0.0, [1])
    client.push_gradients([Tensor("t1", g1, None), Tensor("t2", g2, None)],
                          [Tensor("t3", np.ones((2, 2), dtype=F), np.array([1, 3]))], 0.0, [1])  # step 4
    assert group.snapshot()[0][1] == 4
    assert close(group.pull_dense(["t1"])["t1"].cpu().numpy().ravel(), 0.8474920307 + off, 1e-4)
    assert close(group.pull_dense(["t2"])["t2"].cpu().numpy().ravel(),
                 [0.8474920307, 1.8474920307, 0.9474920307, 2.0474920307], 1e-4)
    assert close(client.pull_embedding_vectors("t3", [1, 3]).ravel(), [-0.058112835] * 4, 1e-4)
    client.push_gradients([], [Tensor("t3", np.ones((3, 2), dtype=F), np.array([1, 3, 5]))], 0.0, [2])  # step 5
    assert close(client.pull_embedding_vectors("t3", [1, 3, 5]).ravel(),
                 [-0.1314178004] * 4 + [-0.0545489238] * 2, 1e-4)
    group.close()


def test_gpu_push_model_handshake_server_test_go_107():
    from elasticdl_b200.common.tensor_utils import Tensor

    group, client, _ = make_pair(2, "sgd")
    rng = np.random.RandomState(9)
    a, b = rng.rand(2, 5).astype(F), rng.rand(2, 5).astype(F)
    client.partition_dense_parameters(["t1", "t2"])
    versions = [-1, -1]
    params, uninit = client.pull_dense_parameters([0, 1], versions)
    assert params == {} and sorted(uninit) == sorted(client.ps_to_parameter.keys())
    for ps_id in uninit:
        client.push_dense_parameters([Tensor("t1", a, None), Tensor("t2", b, None)], ps_id, 0)
    params, uninit = client.pull_dense_parameters([0, 1], versions)
    assert uninit == [] and np.array_equal(params["t1"], a) and np.array_equal(params["t2"], b)
    assert all(versions[p] == 0 for p in client.ps_to_parameter)
    # first writer wins: a second push_model is ignored
    for ps_id in client.ps_to_parameter:
        client.push_dense_parameters([Tensor("t1", a * 0, None), Tensor("t2", b * 0, None)], ps_id, 0)
    params, _ = client.pull_dense_parameters([0, 1], versions)
    assert np.array_equal(params["t1"], a)
    # PushGradients{LearningRate: 0.2} with grads == params (server_test.go:305-331)
    client.push_embedding_table_infos([info("e1", 10, capacity=8)])
    c = rng.rand(1, 10).astype(F)
    group.set_rows([("e1", [1], c)])
    acc, ver = client.push_gradients([Tensor("t1", a, None), Tensor("t2", b, None)],
                                     [Tensor("e1", c, np.array([1]))], 0.2, versions)
    assert acc and ver == 1
    params, _ = client.pull_dense_parameters([0, 1], versions)
    assert np.array_equal(params["t1"], a - F(0.2) * a) and np.array_equal(params["t2"], b - F(0.2) * b)
    assert np.array_equal(client.pull_embedding_vectors("e1", [1]), c - F(0.2) * c)
    assert versions == [1, 1] or all(versions[p] == 1 for p in client.ps_to_parameter)
    group.close()


def test_gpu_staleness_modulation_server_go_178():
    from elasticdl_b200.common.tensor_utils import Tensor

    group, client, oc = make_pair(1, "sgd", lr_staleness_modulation=True)
    for c, T in ((client, Tensor), (oc, O.Tensor)):
        c.partition_dense_parameters(["w"])
        c.push_dense_parameters([T("w", np.ones(4, dtype=F), None)], 0, 0)
    group.set_shard_state(0, version=5)
    oc.servers[0].version = 5
    for lr, ver in ((0.1, 1), (0.0, 6), (0.3, 2)):
        client.push_gradients([Tensor("w", np.ones(4, dtype=F), None)], [], lr, [ver])
        oc.push_gradients([O.Tensor("w", np.ones(4, dtype=F), None)], [], lr, [ver])
        assert np.array_equal(group.pull_dense(["w"])["w"].cpu().numpy(), oc.servers[0].dense["w"])
    group.close()


def test_gpu_amsgrad_dense_quirk_q1():
    from elasticdl_b200.common.tensor_utils import Tensor

    for q1 in (False, True):
        group, client, oc = make_pair(1, "amsgrad", reproduce_q1=q1)
        for c, T in ((client, Tensor), (oc, O.Tensor)):
            c.partition_dense_parameters(["w"])
            c.push_dense_parameters([T("w", np.linspace(-1, 1, 12).astype(F), None)], 0, 0)
        for _ in range(3):
            g = np.linspace(0.5, -0.5, 12).astype(F)
            client.push_gradients([Tensor("w", g, None)], [], 0.0, [0])
            oc.push_gradients([O.Tensor("w", g, None)], [], 0.0, [0])
        assert np.array_equal(group.pull_dense(["w"])["w"].cpu().numpy(), oc.servers[0].dense["w"])
        group.close()


def test_gpu_errors():
    from elasticdl_b200._lib import PSNotFound, PSRangeError
    from elasticdl_b200.common.tensor_utils import Tensor

    group, client, _ = make_pair(2, "sgd")
    client.push_embedding_table_infos([info("e", 4, capacity=100)])
    with pytest.raises(KeyError):
        client.pull_embedding_vectors("missing", [1])
    with pytest.raises(ValueError):
        client.pull_embedding_vectors("e", [])
    with pytest.raises(ValueError):  # id beyond capacity (embedding_delegate.py:254-264)
        client.pull_embedding_vectors("e", [5, 100000])
    with pytest.raises(ValueError):  # width mismatch (kernel.go:36-38)
        client.push_gradients([], [Tensor("e", np.ones((2, 3), dtype=F), np.array([1, 2]))], 0.1, [0, 0])
    assert [s[1] for s in group.snapshot()] == [1, 1]  # the failed ApplyGradients bumped step (Q2)
    assert [s[0] for s in group.snapshot()] == [0, 0]  # ... but not the version
    with pytest.raises(ValueError):
        from elasticdl_b200.ps import PSGroup

        PSGroup(1, "SGD", "learning_rate=0.1;momentum=0.0;nesterov=true;redundant_arg=1;", device=0)
    with pytest.raises(ValueError):
        PSGroup(1, "RMSprop", "learning_rate=0.1;", device=0)
    group.close()


def test_gpu_table_ids_and_len():
    group, client, _ = make_pair(3, "sgd")
    client.push_embedding_table_infos([info("e", 2, capacity=64)])
    client.pull_embedding_vectors("e", [1, 3, 5, 7, 9, 3])
    assert group.table_size("e") == 5
    got = sorted(sum((group.table_ids("e", s).cpu().tolist() for s in range(3)), []))
    assert got == [1, 3, 5, 7, 9]
    for s in range(3):
        assert all(i % 3 == s for i in group.table_ids("e", s).cpu().tolist())
    group.close()


# ------------------------------------------------------------------ full-size properties (BASELINE config 2 sizes)
def test_full_size_roundtrip_and_linearity():
    """5.5 M-row deep table (dac_ctr C3+C4+... after the 1e6 cap), 8 shards:
    set -> pull round trip, SGD push(+g) then push(-g) returns bit-exactly (values on a
    binary grid), pulls are idempotent, checksum of checksums."""
    from elasticdl_b200.common.tensor_utils import Tensor

    group, client, _ = make_pair(8, "sgd")
    rows = 5_549_416
    client.push_embedding_table_infos([info("deep", 8, capacity=rows), info("wide", 1, capacity=rows)])
    gen = torch.Generator(device="cuda").manual_seed(3)
    k = 1 << 20
    ids = torch.randperm(rows, device="cuda", generator=gen)[:k]
    vals = torch.randint(-64, 64, (k, 8), device="cuda", generator=gen).float() / 8
    group.set_rows([("deep", ids, vals)])
    (got,) = group.pull_rows([("deep", ids)])
    assert torch.equal(got, vals)
    (again,) = group.pull_rows([("deep", ids)])
    assert torch.equal(again, got)
    g = torch.randint(-8, 8, (k, 8), device="cuda", generator=gen).float()
    client.push_gradients([], [Tensor("deep", g, ids)], 0.5, [0] * 8)
    (mid,) = group.pull_rows([("deep", ids)])
    assert torch.equal(mid, vals - 0.5 * g)
    client.push_gradients([], [Tensor("deep", -g, ids)], 0.5, [1] * 8)
    (back,) = group.pull_rows([("deep", ids)])
    assert torch.equal(back, vals)
    assert float(back.double().sum()) == float(vals.double().sum())
    assert group.table_size("deep") == k
    # duplicates: pushing each id twice with g/2 equals pushing g once (exact on the grid)
    ids2 = torch.cat([ids, ids])
    g2 = torch.cat([g / 2, g / 2])
    client.push_gradients([], [Tensor("deep", g2, ids2)], 0.5, [2] * 8)
    (dup,) = group.pull_rows([("deep", ids)])
    assert torch.equal(dup, vals - 0.5 * g)
    assert [s[0] for s in group.snapshot()] == [3] * 8
    group.close()


# ------------------------------------------------------------------ config 2: census wide&deep, async SGD, 4 workers
def test_four_concurrent_workers_async_sgd_census_shapes():
    """BASELINE.json configs[2]: 3 wide (dim 1) + 3 deep (dim 8) small tables, async SGD, 4 workers,
    batch 64 (scripts/client_test.sh:38).  Workers are threads with their own view + stream
    (worker_ps_interaction_test.py:136-151 drives workers as threads against shared PS instances).
    Sparse ids are disjoint per worker so the racy interleaving cannot change the result."""
    import threading

    from elasticdl_b200.common.tensor_utils import Tensor
    from elasticdl_b200.worker.ps_client import PSClient

    n_shards, n_workers, steps, rows = 2, 4, 6, 4000
    group, client, oc = make_pair(n_shards, "sgd")
    names = [("wide%d" % i, 1) for i in range(3)] + [("deep%d" % i, 8) for i in range(3)]
    client.push_embedding_table_infos([info(n, d, capacity=rows) for n, d in names])
    oc.push_embedding_table_infos([oinfo(n, d) for n, d in names])
    for c, T in ((client, Tensor), (oc, O.Tensor)):
        c.partition_dense_parameters(["mlp/w"])
        for ps_id in set(c.parameter_to_ps.values()):
            c.push_dense_parameters([T("mlp/w", np.zeros((24, 16), dtype=F), None)], ps_id, 0)
    plans = []
    for w in range(n_workers):
        rng = np.random.RandomState(100 + w)  # seed per worker = 100 + rank (SURVEY 8d config 3)
        plan = []
        for s in range(steps):
            step_grads = []
            for n, d in names:
                ids = (rng.randint(0, rows // n_workers, 64) * n_workers + w).astype(np.int64)  # ids == w (mod 4)
                step_grads.append((n, rng.randn(64, d).astype(F), ids))
            plan.append(step_grads)
        plans.append(plan)
    errors = []

    def worker(w):
        try:
            view = group.clone_view()
            wc = PSClient(view)
            wc.parameter_to_ps, wc.ps_to_parameter = client.parameter_to_ps, client.ps_to_parameter
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                versions = [0] * n_shards
                for step_grads in plans[w]:
                    acc, v = wc.push_gradients([], [Tensor(n, g, i) for n, g, i in step_grads], 0.1, versions)
                    assert acc
                    versions = [v] * n_shards
                    wc.pull_embedding_vectors(names[3][0], step_grads[3][2])
            stream.synchronize()
            view.close()
        except Exception as e:  # noqa: BLE001
            errors.append((w, repr(e)))

    threads = [threading.Thread(target=worker, args=(w,)) for w in range(n_workers)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors
    for w in range(n_workers):
        for step_grads in plans[w]:
            oc.push_gradients([], [O.Tensor(n, g.copy(), i) for n, g, i in step_grads], 0.1, [0] * n_shards)
    state = group.snapshot()
    assert [s[0] for s in state] == [n_workers * steps] * n_shards  # one version per push per worker
    all_ids = np.arange(rows, dtype=np.int64)
    for n, d in names:
        got = client.pull_embedding_vectors(n, all_ids)
        want = np.zeros_like(got)
        for s in oc.servers:
            keys = s.tables[n].keys()
            want[keys] = s.tables[n].get(keys)
        assert np.allclose(got, want, rtol=1e-5, atol=1e-6), n
    group.close()


# ------------------------------------------------------------------ sync-SGD (SURVEY 8f-1)
def test_sync_sgd_pserver_servicer_test_py_366():
    """grads_to_wait 2: dense averaged / sparse summed, third push with version 0 -> rejected."""
    from elasticdl_b200.common.tensor_utils import Tensor
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient

    group = PSGroup(1, "SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", device=0,
                    use_async=False, grads_to_wait=2)
    client = PSClient(group)
    rng = np.random.RandomState(3)
    var = {"v0": rng.rand(3, 2).astype(F), "v1": rng.rand(3).astype(F)}
    g0 = {"v0": rng.rand(3, 2).astype(F), "v1": rng.rand(3).astype(F)}
    g1 = {"v0": rng.rand(3, 2).astype(F), "v1": rng.rand(3).astype(F)}
    client.partition_dense_parameters(var.keys())
    client.push_dense_parameters([Tensor(n, v, None) for n, v in var.items()], 0, 0)
    client.push_embedding_table_infos([info("emb", 8, capacity=16)])
    table = rng.rand(10, 8).astype(F)
    group.set_rows([("emb", np.arange(10), table)])
    e0 = (rng.rand(3, 8).astype(F), np.array([3, 1, 3]))
    e1 = (rng.rand(2, 8).astype(F), np.array([1, 9]))
    lr = 0.1
    acc, ver = client.push_gradients([Tensor(n, v, None) for n, v in g0.items()], [Tensor("emb", *e0)], lr, [0])
    assert (acc, ver) == (True, 0)
    acc, ver = client.push_gradients([Tensor(n, v, None) for n, v in g1.items()], [Tensor("emb", *e1)], lr, [0])
    assert (acc, ver) == (True, 1)
    acc, ver = client.push_gradients([Tensor(n, v, None) for n, v in g1.items()], [], lr, [0])
    assert (acc, ver) == (False, 1)
    d = group.pull_dense(list(var))
    for n in var:
        assert np.allclose(d[n].cpu().numpy(), var[n] - lr * (g0[n] + g1[n]) / 2, atol=1e-6)
    want = table.copy()
    for vals, ids in (e0, e1):
        for gv, gi in zip(vals, ids):
            want[gi] -= lr * gv
    assert np.allclose(client.pull_embedding_vectors("emb", np.arange(10)), want, atol=1e-6)
    # tolerance lets one-version-stale pushes in
    group2 = PSGroup(1, "SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", device=0,
                     use_async=False, grads_to_wait=1, sync_version_tolerance=1)
    c2 = PSClient(group2)
    c2.partition_dense_parameters(["w"])
    c2.push_dense_parameters([Tensor("w", np.ones(4, dtype=F), None)], 0, 0)
    assert c2.push_gradients([Tensor("w", np.ones(4, dtype=F), None)], [], lr, [0]) == (True, 1)
    assert c2.push_gradients([Tensor("w", np.ones(4, dtype=F), None)], [], lr, [0]) == (True, 2)  # stale by 1: ok
    assert c2.push_gradients([Tensor("w", np.ones(4, dtype=F), None)], [], lr, [0]) == (False, 2)  # stale by 2
    group.close()
    group2.close()


# ------------------------------------------------------------------ hashed tables: unbounded ids (embedding_table.go:22-58)
HASHED_CASES = [(opt, d) for opt in OPTS for d in (1, 8)] + [(opt, d) for opt in ("adam", "ftrl") for d in (4, 10, 64)]


@pytest.mark.parametrize("n_shards", [1, 3])
@pytest.mark.parametrize("opt,dim", HASHED_CASES)
def test_hashed_table_unbounded_ids(opt, dim, n_shards):
    """An ElasticDL Embedding without input_dim: ids are arbitrary int64, rows are created lazily on
    first pull OR push (kernel_test.go:56-66), len(table) counts the created rows.  Two hashed tables of the same
    dim share every push launch (k_push_rows: 4 / 8 floats per thread in 1..8 chunks per row, or scalars); a push
    without duplicate ids matches the oracle bit for bit, pushes with duplicates (summed in another order) to 1e-5."""
    from elasticdl_b200.common.tensor_utils import EmbeddingTableInfo, Tensor

    group, client, oc = make_pair(n_shards, opt)
    tabs = ("h", "h2")
    client.push_embedding_table_infos([EmbeddingTableInfo(t, dim, "zero", 1) for t in tabs])  # no capacity -> hashed
    oc.push_embedding_table_infos([oinfo(t, dim) for t in tabs])
    import zlib
    rng = np.random.RandomState(zlib.crc32(repr((opt, dim, n_shards)).encode()))
    ids = np.unique(rng.randint(0, 2 ** 40, size=3000).astype(np.int64))
    rng.shuffle(ids)
    ids2 = np.unique(rng.randint(0, 2 ** 40, size=2000).astype(np.int64))
    vals = rng.randn(len(ids), dim).astype(F)
    half = len(ids) // 2
    group.set_rows([("h", ids[:half], vals[:half])])
    for s in oc.servers:
        m = ids[:half] % n_shards == s.id
        s.tables["h"].set(ids[:half][m], vals[:half][m])
    q = rng.choice(ids[:half], 2000)
    assert np.array_equal(client.pull_embedding_vectors("h", q), oc.pull_embedding_vectors("h", q))
    assert group.table_size("h") == half

    # the duplicated rounds sum repeated ids in another order than the oracle (and from run to run): Momentum's
    # velocity carries those last-bit differences past 1e-7 absolute (test_push_gradients_all_optimizers: 1e-6), and
    # FTRL's linear slot, a running sum of O(1) terms that cancel, to a few 1e-6 (measured on an H100: 2.5e-6)
    slot_atol = {"adam": 1e-7, "amsgrad": 1e-7, "ftrl": 1e-5, "ftrl_shrink": 1e-5}.get(opt, 1e-6)

    def compare(exact):
        for t in tabs:
            created = np.sort(np.concatenate([s.tables[t].keys() for s in oc.servers]))
            assert group.table_size(t) == len(created), t
            got_ids = np.sort(np.concatenate([group.table_ids(t, s).cpu().numpy() for s in range(n_shards)]))
            assert np.array_equal(got_ids, created), t
            got, want = client.pull_embedding_vectors(t, created), oc.pull_embedding_vectors(t, created)
            assert np.array_equal(got, want) if exact else np.allclose(got, want, rtol=1e-5, atol=1e-6), t
            for k, sn in enumerate(oc.servers[0].opt.slot_names):
                gs = group.slot_rows(t, created, k + 1).cpu().numpy()
                ws = np.zeros_like(gs)
                for s in oc.servers:
                    m = created % n_shards == s.id
                    ws[m] = s.opt.table_slots[sn][t].get(created[m])
                assert np.array_equal(gs, ws) if exact else np.allclose(gs, ws, rtol=1e-5, atol=slot_atol), (t, sn)

    # pushes create the second half lazily (zero rows) and update the first half; the first has no duplicate ids
    versions, oversions = [0] * n_shards, [0] * n_shards
    for step in range(4):
        if step == 0:
            pid, pid2 = rng.permutation(ids)[:1500], rng.permutation(ids2)[:700]
        else:
            pid, pid2 = rng.choice(ids, 1500), rng.choice(ids2, 700)  # with duplicates
        g, g2 = rng.randn(len(pid), dim).astype(F), rng.randn(len(pid2), dim).astype(F)
        a1 = client.push_gradients([], [Tensor("h", g, pid), Tensor("h2", g2, pid2)], 0.05 if step == 1 else 0.0, versions)
        a2 = oc.push_gradients([], [O.Tensor("h", g.copy(), pid.copy()), O.Tensor("h2", g2.copy(), pid2.copy())],
                               0.05 if step == 1 else 0.0, oversions)
        assert a1 == a2
        versions, oversions = [a1[1]] * n_shards, [a2[1]] * n_shards
        if step == 0:
            compare(exact=True)
    compare(exact=False)
    group.close()


def test_hashed_table_uniform_and_full():
    from elasticdl_b200.common.tensor_utils import EmbeddingTableInfo

    group, client, _ = make_pair(2, "sgd")
    group.register_table("u", 8, "uniform", None, expected_rows=600)
    group.commit()
    ids = np.arange(0, 400, dtype=np.int64) * 7919 + 2 ** 35
    a = client.pull_embedding_vectors("u", ids)
    assert a.min() >= -0.05 and a.max() < 0.05 and a.std() > 0.01
    assert np.array_equal(client.pull_embedding_vectors("u", ids), a)  # stable once created
    assert group.table_size("u") == 400
    # 2 shards x 1024 slots: the 2049th distinct id on some shard cannot be placed
    with pytest.raises(ValueError, match="full"):
        client.pull_embedding_vectors("u", np.arange(5000, dtype=np.int64) * 2 + 1)
    group.close()


# ------------------------------------------------------------------ checkpoint save / re-sharded restore (SURVEY 8f-2)
def test_checkpoint_resharding_2_to_3_checkpoint_test_go_25(tmp_path):
    """Save with 2 shards, restore with 3: ids {0,2,4} U {1,3,5} land on shards {0,3} {1,4} {2,5}
    (checkpoint_test.go:25-82); dense parameters re-hash by name; slots are not checkpointed (Q9)."""
    from elasticdl_b200.common.tensor_utils import Tensor
    from elasticdl_b200.ps import checkpoint as ck

    group, client, _ = make_pair(2, "adam")
    client.push_embedding_table_infos([info("e1", 2, capacity=64), info("hashed", 4, capacity=None)])
    ids = np.array([0, 2, 4, 1, 3, 5], dtype=np.int64)
    vals = np.arange(12, dtype=F).reshape(6, 2)
    group.set_rows([("e1", ids, vals)])
    hid = np.array([7, 2 ** 33 + 1, 12], dtype=np.int64)
    hval = np.arange(12, dtype=F).reshape(3, 4) + 100
    group.set_rows([("hashed", hid, hval)])
    dense = {"dense/kernel:0": np.arange(6, dtype=F).reshape(2, 3), "dense/bias:0": np.array([9, 8, 7], dtype=F)}
    client.partition_dense_parameters(dense.keys())
    for ps_id in set(client.parameter_to_ps.values()):
        client.push_dense_parameters([Tensor(n, v, None) for n, v in dense.items()], ps_id, 0)
    for _ in range(3):  # move the version to 3 and dirty the optimizer slots
        client.push_gradients([Tensor(n, np.ones_like(v), None) for n, v in dense.items()],
                              [Tensor("e1", np.ones((2, 2), dtype=F), np.array([0, 1]))], 0.0, [0, 0])
    want_rows = client.pull_embedding_vectors("e1", ids)
    want_dense = {n: group.pull_dense([n])[n].cpu().numpy() for n in dense}
    vdir = ck.save(group, str(tmp_path), keep_checkpoint_max=2)
    assert vdir.endswith("version-3") and ck.is_valid_version_dir(vdir)
    assert sorted(__import__("os").listdir(vdir)) == ["variables-0-of-2.ckpt", "variables-1-of-2.ckpt"]
    # the files parse back: per-shard contents follow id % 2
    _, infos, d0, t0 = ck.decode_model(open(vdir + "/variables-0-of-2.ckpt", "rb").read())
    assert sorted(t0["e1"][0].tolist()) == [0, 2, 4] and {i[0] for i in infos} == {"e1", "hashed"}
    group.close()

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient

    g3 = PSGroup(3, *OPTS["adam"], device=0)
    c3 = PSClient(g3)
    c3.push_embedding_table_infos([info("e1", 2, capacity=64)])  # "hashed" is created from the checkpoint's infos
    assert ck.load(g3, c3, ck.latest_version_dir(str(tmp_path))) == 3
    assert [sorted(g3.table_ids("e1", s).cpu().tolist()) for s in range(3)] == [[0, 3], [1, 4], [2, 5]]
    assert np.array_equal(c3.pull_embedding_vectors("e1", ids), want_rows)
    assert np.array_equal(c3.pull_embedding_vectors("hashed", hid), hval)
    versions = [-1] * 3
    params, uninit = c3.pull_dense_parameters([0, 1, 2], versions)
    assert uninit == [] and all(np.array_equal(params[n], want_dense[n]) for n in dense)
    assert all(versions[p] == 3 for p in c3.ps_to_parameter)
    assert not g3.slot_rows("e1", ids, 1).any()  # slots start from zero again (quirk Q9)
    g3.close()


def test_unique_bounded_direct_address_segments():
    """b200ps_unique_bounded: segments whose id range fits the table dedup by direct address;
    results must equal the hashed path / tf.unique exactly."""
    import ctypes

    from elasticdl_b200 import _lib

    group, _, _ = make_pair(1)
    rng = np.random.RandomState(11)
    T, k = 5, 6000
    bounds = [7, 300, 0, 5000, 10 ** 6]  # 0 = unknown, 1e6 > table capacity -> hashed
    ids = np.stack([rng.randint(0, b if b else 10 ** 5, size=k) for b in bounds]).astype(np.int64)
    d_ids = torch.from_numpy(ids).cuda().view(-1)
    lib = _lib.lib()
    arr = (ctypes.c_int64 * T)(*bounds)
    need = lib.b200ps_unique_bounded_workspace(T, k, arr)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    uniq = torch.empty(T * k, dtype=torch.int64, device="cuda")
    inv = torch.empty(T * k, dtype=torch.int32, device="cuda")
    n = torch.empty(T, dtype=torch.int32, device="cuda")
    for _ in range(2):  # twice: the workspace is reused dirty
        _lib.check(lib.b200ps_unique_bounded(group._h, d_ids.data_ptr(), T, k, arr, uniq.data_ptr(), inv.data_ptr(),
                                             n.data_ptr(), ws.data_ptr(), ws.numel(), group._stream()))
        u, i, c = uniq.cpu().numpy().reshape(T, k), inv.cpu().numpy().reshape(T, k), n.cpu().numpy()
        for t in range(T):
            wu, wi = O.unique_first_occurrence(ids[t])
            assert c[t] == len(wu) and np.array_equal(u[t, : c[t]], wu) and np.array_equal(i[t], wi), t
    group.close()


def test_unique_bounded_epoch_tags_survive_reuse_and_wraparound():
    """Direct-address segments are not cleared between calls (epoch-prefixed positions, a real
    clear every 2047 calls): 2100 calls on one dirty workspace with fresh ids each time, and a
    workspace full of garbage, all equal tf.unique."""
    import ctypes

    from elasticdl_b200 import _lib

    group, _, _ = make_pair(1)
    lib = _lib.lib()
    T, k = 3, 700
    bounds = [5, 900, 40000]
    arr = (ctypes.c_int64 * T)(*bounds)
    need = lib.b200ps_unique_bounded_workspace(T, k, arr)
    ws = torch.randint(0, 255, (need,), dtype=torch.uint8, device="cuda")  # garbage, not zeros
    uniq = torch.empty(T * k, dtype=torch.int64, device="cuda")
    inv = torch.empty(T * k, dtype=torch.int32, device="cuda")
    n = torch.empty(T, dtype=torch.int32, device="cuda")
    rng = np.random.RandomState(3)
    pool = [np.stack([rng.randint(0, b, size=k) for b in bounds]).astype(np.int64) for _ in range(7)]
    d_pool = [torch.from_numpy(p).cuda().view(-1) for p in pool]
    for call in range(2100):
        j = call % len(pool)
        if call % 3 == 2 or call in (2046, 2047):  # calls without bounds share the workspace and its epoch counter
            _lib.check(lib.b200ps_unique(group._h, d_pool[j].data_ptr(), T, k, uniq.data_ptr(), inv.data_ptr(),
                                         n.data_ptr(), ws.data_ptr(), ws.numel(), group._stream()))
        else:
            _lib.check(lib.b200ps_unique_bounded(group._h, d_pool[j].data_ptr(), T, k, arr, uniq.data_ptr(), inv.data_ptr(),
                                                 n.data_ptr(), ws.data_ptr(), ws.numel(), group._stream()))
        if call < 5 or call % 211 == 0 or 2040 <= call <= 2055 or call == 2099:
            u, i, c = uniq.cpu().numpy().reshape(T, k), inv.cpu().numpy().reshape(T, k), n.cpu().numpy()
            for t in range(T):
                wu, wi = O.unique_first_occurrence(pool[j][t])
                assert c[t] == len(wu) and np.array_equal(u[t, : c[t]], wu) and np.array_equal(i[t], wi), (call, t)
    group.close()


# ------------------------------------------------------------------ kernel_api.h drop-ins on raw device arrays
@pytest.mark.parametrize("n", [10, 1001, 4096 * 33])
def test_raw_kernel_api_matches_oracle_bit_exact(n):
    """b200ps_kernel_{sgd,momentum,adam,adagrad} == kernel_api.cc via the oracle, bit for bit
    (kernel_test.go:25-47 asserts exact equality for SGD)."""
    import ctypes

    from elasticdl_b200 import _lib

    lib = _lib.lib()
    rng = np.random.RandomState(n)
    g, p, m, v, ms = [rng.rand(n).astype(F) for _ in range(5)]
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def dev(*arrs):
        return [torch.from_numpy(a.copy()).cuda() for a in arrs]

    # SGD
    dg, dp = dev(g, p)
    _lib.check(lib.b200ps_kernel_sgd(dg.data_ptr(), dp.data_ptr(), 0.1, n, st))
    want = p.copy()
    O.lib.oracle_sgd(O._f32(g), O._f32(want), 0.1, n)
    assert np.array_equal(dp.cpu().numpy(), want)
    # Momentum / Nesterov
    for nesterov in (0, 1):
        dg, dp, dv = dev(g, p, v)
        _lib.check(lib.b200ps_kernel_momentum(dg.data_ptr(), dp.data_ptr(), dv.data_ptr(), 0.9, nesterov, 0.05, n, st))
        wp, wv = p.copy(), v.copy()
        O.lib.oracle_momentum(O._f32(g), O._f32(wp), O._f32(wv), 0.9, nesterov, 0.05, n)
        assert np.array_equal(dp.cpu().numpy(), wp) and np.array_equal(dv.cpu().numpy(), wv)
    # Adam / AMSGrad (kernel_test.go:69-180: step 5, lr .1, betas .9/.999, eps 1e-8)
    for ams in (False, True):
        dg, dp, dm, dv, dms = dev(g, p, m, v, ms)
        _lib.check(lib.b200ps_kernel_adam(dg.data_ptr(), dp.data_ptr(), dm.data_ptr(), dv.data_ptr(), 0.1, n, 5, 0.9,
                                          0.999, 1e-8, dms.data_ptr() if ams else None, st))
        wp, wm, wv, wms = p.copy(), m.copy(), v.copy(), ms.copy()
        O.lib.oracle_adam(O._f32(g), O._f32(wp), O._f32(wm), O._f32(wv), 0.1, n, 5, 0.9, 0.999, 1e-8,
                          O._f32(wms) if ams else O._null_f32())
        assert np.array_equal(dp.cpu().numpy(), wp) and np.array_equal(dm.cpu().numpy(), wm)
        assert np.array_equal(dv.cpu().numpy(), wv)
        if ams:
            assert np.array_equal(dms.cpu().numpy(), wms)
    # Adagrad
    dg, dp, dm = dev(g, p, m)
    _lib.check(lib.b200ps_kernel_adagrad(dg.data_ptr(), dp.data_ptr(), dm.data_ptr(), 0.05, n, 1e-7, st))
    wp, wm = p.copy(), m.copy()
    O.lib.oracle_adagrad(O._f32(g), O._f32(wp), O._f32(wm), 0.05, n, 1e-7)
    assert np.array_equal(dp.cpu().numpy(), wp) and np.array_equal(dm.cpu().numpy(), wm)


# ------------------------------------------------------------------ round 2: persistent unique, flat row kernels
@pytest.mark.parametrize("k,hi,T,bounded", [(300_000, 1 << 40, 2, False), (70_001, 50_000, 3, True), (2049, 7, 2, True),
                                            (33, 1000, 5, False)])
def test_unique_many_tiles_lookback_int32_and_negative_ids(k, hi, T, bounded):
    """The single persistent unique kernel: hundreds of tiles per segment (decoupled look-back over more than one
    32-tile window), a ragged last chunk / tile, negative ids on the hashed path, and the int32 entry point --
    all equal tf.unique (first-occurrence order, inverse) exactly; int32 and int64 inputs give identical outputs."""
    import ctypes

    from elasticdl_b200 import _lib

    group, _, _ = make_pair(1)
    lib = _lib.lib()
    rng = np.random.RandomState(k % 1000 + T)
    ids = rng.randint(0, min(hi, 2 ** 62), size=(T, k)).astype(np.int64)
    if not bounded:
        ids[:, ::7] *= -1  # negative ids are legal for tf.unique (hashed segments)
        ids[0, -5:] = [-1, -2, -1, -31, -2]  # collide with nothing: dead lanes of the ragged tail never match
    d_ids = torch.from_numpy(ids).cuda().view(-1)
    bounds = (ctypes.c_int64 * T)(*([hi] * T if bounded else [0] * T))
    need = lib.b200ps_unique_bounded_workspace(T, k, bounds)
    ws = torch.randint(0, 255, (need,), dtype=torch.uint8, device="cuda")
    outs = []
    for narrow in ((False, True) if bounded else (False,)):
        uniq = torch.empty(T * k, dtype=torch.int64, device="cuda")
        inv = torch.empty(T * k, dtype=torch.int32, device="cuda")
        n = torch.empty(T, dtype=torch.int32, device="cuda")
        src = d_ids.to(torch.int32) if narrow else d_ids
        fn = lib.b200ps_unique_bounded_i32 if narrow else lib.b200ps_unique_bounded
        for _ in range(2):
            _lib.check(fn(group._h, src.data_ptr(), T, k, bounds, uniq.data_ptr(), inv.data_ptr(), n.data_ptr(),
                          ws.data_ptr(), ws.numel(), group._stream()))
        group.check()
        u, i, c = uniq.cpu().numpy().reshape(T, k), inv.cpu().numpy().reshape(T, k), n.cpu().numpy()
        for t in range(T):
            wu, wi = O.unique_first_occurrence(ids[t])
            assert c[t] == len(wu) and np.array_equal(u[t, : c[t]], wu) and np.array_equal(i[t], wi), (t, narrow)
        outs.append((u, i, c))
    group.close()


def _flat_launch_case(opt, n_shards, large, make_pair=make_pair):
    """ONE b200ps_pull_rows / b200ps_push_rows call over segments of mixed dims, a dense parameter addressed by rows
    (Indexed* kernels, kernel.go:48-55) and device-side live counts (n_dev < n), pushed twice so that the second
    push reads nonzero slots: the flat kernels (csrc/ps_flat.cuh) must equal the oracle bit for bit -- params and
    every slot -- and must not touch rows beyond the live counts.  large: the host-side item bound reaches
    8 x 6 x 256 x #SM, which selects the instances with two rows in flight per thread (U = 2).  make_pair: the
    (group, client, oracle client) maker of the optimizer family `opt` belongs to."""
    from elasticdl_b200 import _lib
    from elasticdl_b200.common.hash_utils import string_to_id

    group, client, oc = make_pair(n_shards, opt)
    rng = np.random.RandomState(5 if not large else 6)
    dn = "dense/w:0"
    if not large:
        dims = [8, 1, 64, 10, 4, 1, 8]
        caps = [5000, 37, 900, 411, 64, 20000, 3]
        dshape = (50, 12)
    else:
        dims = [64, 8, 1, 10, 4]
        caps = [40_000, 250_000, 100_000, 30_000, 5000]
        dshape = (5000, 12)
    names = ["t%d" % i for i in range(len(dims))]
    client.push_embedding_table_infos([info(n, d, capacity=c) for n, d, c in zip(names, dims, caps)])
    oc.push_embedding_table_infos([oinfo(n, d) for n, d in zip(names, dims)])
    group.register_dense(dn, dshape, string_to_id(dn, n_shards))
    group.commit()
    dense0 = rng.randn(*dshape).astype(F)
    group.set_dense([(dn, dense0)])
    dim_of = dict(zip(names + [dn], dims + [dshape[1]]))
    cap_of = dict(zip(names + [dn], caps + [dshape[0]]))
    if not large:  # (table, rows, live rows); live 0 = an empty segment; table 0 twice
        spec = []
        for n_ in names + [dn, names[0]]:
            m = min(cap_of[n_], 700)
            spec.append((n_, m, 0 if n_ == names[4] else int(rng.randint(1, m + 1))))
    else:  # small and large live counts, ragged against every warp / unroll boundary
        spec = [(names[0], 32_000, 32_000 - 7), (names[1], 200_000, 13), (names[2], 90_000, 90_000 - 9),
                (names[3], 25_000, 24_991), (names[4], 5000, 3), (dn, 4000, 3999)]
    segs, used = [], {}
    for n_, m, nl in spec:
        ids = rng.permutation(cap_of[n_]).astype(np.int64)
        ids = ids[~np.isin(ids, used.get(n_, []))][:m]  # a push applies each row once per launch
        nl = min(nl, len(ids))
        used[n_] = np.concatenate([used.get(n_, np.zeros(0, np.int64)), ids[:nl]])
        segs.append((n_, dim_of[n_], ids, nl))
    if large:  # the same bound split_segs computes: rows a segment may hold x lanes per row
        bound = sum(min(len(ids), -(-cap_of[n_] // n_shards) * n_shards if n_ != dn else cap_of[n_]) * d
                    for n_, d, ids, _ in segs)
        assert bound >= 8 * 6 * 256 * torch.cuda.get_device_properties(0).multi_processor_count
    # initial rows everywhere
    for n_, d, c in zip(names, dims, caps):
        all_ids = np.arange(c, dtype=np.int64)
        vals = rng.randn(c, d).astype(F)
        group.set_rows([(n_, all_ids, vals)])
        for s_ in oc.servers:
            m = all_ids % n_shards == s_.id
            s_.tables[n_].set(all_ids[m], vals[m])
    lib, h = group.lib, group._h
    items, keep = [], []
    for n_, d, ids, nl in segs:
        tid = group.lookup(n_)[0]
        t_ids = torch.from_numpy(ids).cuda()
        n_dev = torch.tensor([nl], dtype=torch.int32, device="cuda")
        rows = torch.full((len(ids), d), -7.0, dtype=torch.float32, device="cuda")
        keep.append((t_ids, n_dev, rows))
        items.append((tid, len(ids), t_ids, n_dev, rows))
    arr, n = group.make_segs(items)
    _lib.check(lib.b200ps_pull_rows(h, arr, n, group._stream()))
    group.check()
    for (n_, d, ids, nl), (_, _, rows) in zip(segs, keep):
        got = rows.cpu().numpy()
        if n_ == dn:
            want = dense0[ids[:nl]]
        else:
            want = oc.pull_embedding_vectors(n_, ids[:nl]) if nl else np.zeros((0, d), F)
        assert np.array_equal(got[:nl], want), n_
        assert (got[nl:] == -7.0).all(), n_  # nothing beyond the live count
    # the oracle: the same ApplyGradients on every shard (dense-by-rows = Indexed kernels)
    owner = string_to_id(dn, n_shards)
    oc.servers[owner].dense[dn] = dense0.copy()
    oc.servers[owner].opt.init_dense(dn, dshape)
    oc.partition_dense_parameters([dn])
    for lr in (0.05, 0.0):
        # push: gradients for the live rows, one launch
        t_grads = []
        for (n_, d, ids, nl), (_, _, rows) in zip(segs, keep):
            g = (rng.randn(len(ids), d) * 0.1).astype(F)
            rows.copy_(torch.from_numpy(g))
            if nl:
                t_grads.append(O.Tensor(n_, g[:nl].copy(), ids[:nl].copy()))
        group.push_begin(lr, [0] * n_shards)
        _lib.check(lib.b200ps_push_rows(h, arr, n, group._stream()))
        group.push_end()
        group.check()
        oc.push_gradients([t for t in t_grads if t.name == dn], [t for t in t_grads if t.name != dn], lr, [0] * n_shards)
    for n_, d, c in zip(names, dims, caps):
        all_ids = np.arange(c, dtype=np.int64)
        assert np.array_equal(client.pull_embedding_vectors(n_, all_ids), oc.pull_embedding_vectors(n_, all_ids)), n_
        for k, sn in enumerate(oc.servers[0].opt.slot_names):
            got = group.slot_rows(n_, all_ids, k + 1).cpu().numpy()
            for s_ in oc.servers:
                m = all_ids % n_shards == s_.id
                assert np.array_equal(got[m], s_.opt.table_slots[sn][n_].get(all_ids[m])), (n_, sn)
    srv = oc.servers[owner]
    assert np.array_equal(group.pull_dense([dn])[dn].cpu().numpy(), srv.dense[dn]), "indexed rows of a dense parameter"
    for k, sn in enumerate(srv.opt.slot_names):
        assert np.array_equal(group.slot_dense(dn, k + 1).cpu().numpy(), srv.opt.dense_slots[sn][dn]), (dn, sn)
    group.close()


@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("n_shards", [1, 3])
def test_flat_launch_mixed_tables_device_counts(opt, n_shards):
    """Nine segments of dims 1, 4, 8, 10, 64, a dense row view, an empty segment, one table twice."""
    _flat_launch_case(opt, n_shards, large=False)


@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("n_shards", [1, 3])
def test_flat_launch_unrolled_large_device_counts(opt, n_shards):
    """The push every DeepFM benchmark step runs: millions of lane-items, two rows in flight per thread."""
    _flat_launch_case(opt, n_shards, large=True)


def test_unique_packed_per_segment_id_widths():
    """b200ps_unique_packed: every segment of the ids buffer at its own width (1 / 2 / 4 / 8 bytes, unsigned,
    16 B padded segments) == the int64 dedup of the same ids, bit for bit."""
    import ctypes

    from elasticdl_b200 import _lib

    group, _, _ = make_pair(1)
    lib = _lib.lib()
    rng = np.random.RandomState(21)
    T, k = 6, 5001
    bounds_l = [200, 256, 65536, 40000, 10 ** 6, 3]
    widths_l = [1, 1, 2, 2, 4, 8]
    ids = np.stack([rng.randint(0, b, size=k) for b in bounds_l]).astype(np.int64)
    ids[1, :3] = [255, 0, 255]
    ids[2, :3] = [65535, 32768, 32767]
    widths = (ctypes.c_int32 * T)(*widths_l)
    bounds = (ctypes.c_int64 * T)(*bounds_l)
    nbytes = lib.b200ps_packed_ids_bytes(widths, T, k)
    buf = np.zeros(nbytes, dtype=np.uint8)
    off = 0
    for t, w in enumerate(widths_l):
        seg = ids[t].astype({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.int64}[w])
        buf[off:off + k * w] = seg.view(np.uint8)
        off += (k * w + 15) // 16 * 16
    assert off == nbytes
    d_buf = torch.from_numpy(buf).cuda()
    need = lib.b200ps_unique_bounded_workspace(T, k, bounds)
    ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    uniq = torch.empty(T * k, dtype=torch.int64, device="cuda")
    inv = torch.empty(T * k, dtype=torch.int32, device="cuda")
    n = torch.empty(T, dtype=torch.int32, device="cuda")
    for bps in (0, 1):
        _lib.check(lib.b200ps_unique_packed(group._h, d_buf.data_ptr(), widths, T, k, bounds, uniq.data_ptr(), inv.data_ptr(),
                                            n.data_ptr(), ws.data_ptr(), ws.numel(), bps, group._stream()))
        group.check()
        u, i, c = uniq.cpu().numpy().reshape(T, k), inv.cpu().numpy().reshape(T, k), n.cpu().numpy()
        for t in range(T):
            wu, wi = O.unique_first_occurrence(ids[t])
            assert c[t] == len(wu) and np.array_equal(u[t, : c[t]], wu) and np.array_equal(i[t], wi), (t, bps)
    group.close()


@pytest.mark.parametrize("n_shards", [1, 2])
def test_large_mixed_dim_pull_bit_exact(n_shards):
    """A large flat pull (k_copy_flat) returns exactly the table rows: mixed dims (8, 64 in 16 B chunks; 1, 10 in
    floats) in one launch, ragged warp tails, device-side counts, and an out-of-range id (every other row still
    arrives, the error is raised)."""
    from elasticdl_b200 import _lib

    group, client, _ = make_pair(n_shards, "adam")
    rng = np.random.RandomState(9)
    dims, caps = [8, 64, 1, 10], [300_000, 200_000, 50_000, 5_000]
    names = ["s%d" % i for i in range(4)]
    client.push_embedding_table_infos([info(n, d, capacity=c) for n, d, c in zip(names, dims, caps)])
    tabs = {}
    for n_, d, c in zip(names, dims, caps):
        vals = rng.randn(c, d).astype(F)
        group.set_rows([(n_, np.arange(c), vals)])
        tabs[n_] = vals
    lib, h = group.lib, group._h
    items, keep = [], []
    for n_, d, c in zip(names, dims, caps):
        m = c - 7
        ids = rng.permutation(c)[:m].astype(np.int64)
        nl = m - 13
        t_ids = torch.from_numpy(ids).cuda()
        n_dev = torch.tensor([nl], dtype=torch.int32, device="cuda")
        rows = torch.full((m, d), -3.0, dtype=torch.float32, device="cuda")
        keep.append((ids, nl, rows, t_ids, n_dev))
        items.append((group.lookup(n_)[0], m, t_ids, n_dev, rows))
    arr, nseg = group.make_segs(items)
    _lib.check(lib.b200ps_pull_rows(h, arr, nseg, group._stream()))  # 0.6 M + 3.2 M + ... lane-items
    group.check()
    for (ids, nl, rows, _, _), n_ in zip(keep, names):
        got = rows.cpu().numpy()
        assert np.array_equal(got[:nl], tabs[n_][ids[:nl]]), n_
        assert (got[nl:] == -3.0).all(), n_
    # one id out of range in the middle of the dim-8 segment: every other row still arrives, the error is reported
    ids0, nl0, rows0, t_ids0, _ = keep[0]
    t_ids0[1234] = caps[0] + 5
    rows0.fill_(-3.0)
    _lib.check(lib.b200ps_pull_rows(h, arr, nseg, group._stream()))
    with pytest.raises(ValueError):
        group.check()
    got = rows0.cpu().numpy()
    ok = np.ones(nl0, dtype=bool)
    ok[1234] = False
    assert np.array_equal(got[:nl0][ok], tabs[names[0]][ids0[:nl0]][ok])
    assert (got[1234] == -3.0).all()
    group.close()


@pytest.mark.parametrize("n_shards", [1, 2])
def test_wide_rows_big_gather(n_shards):
    """A big gather / set of wide rows (5.1 M lane-items: the persistent grid loops ~8 times with two rows in
    flight per thread): 320 K dim-64 rows set, pulled back in random order with a device-side count and a
    ragged tail -- bit-exact (embedding_table.go:61-77)."""
    group, client, _ = make_pair(n_shards, "sgd")
    rng = np.random.RandomState(21)
    rows, dim = 320_000, 64
    client.push_embedding_table_infos([info("w64", dim, capacity=rows)])
    vals = rng.randn(rows, dim).astype(F)
    group.set_rows([("w64", np.arange(rows), vals)])  # 5.1 M lane-items
    ids = rng.permutation(rows).astype(np.int64)
    m = rows - 3
    live = m - 11
    t_ids = torch.from_numpy(ids[:m]).cuda()
    n_dev = torch.tensor([live], dtype=torch.int32, device="cuda")
    out = torch.full((m, dim), -7.0, dtype=torch.float32, device="cuda")
    group._run_segs(group.lib.b200ps_pull_rows, [(group.lookup("w64")[0], m, t_ids, n_dev, out)])
    group.check()
    got = out.cpu().numpy()
    assert np.array_equal(got[:live], vals[ids[:live]])
    assert (got[live:] == -7.0).all()
    group.close()


@pytest.mark.parametrize("k", [700, 9000, 32768])
def test_unique_small_segments_in_shared_memory(k):
    """Segments whose id range fits a shared-memory position array (kUSmallMax = 16384) are deduplicated by one
    block each (k_unique_small, ids in registers: 8 / 16 / 32 per thread), the others by the grid-wide kernel --
    same first-occurrence order, inverse index and counts as tf.unique, over several calls (epochs of the
    grid-wide kernel) and with out-of-range ids (counted as id 0 AND reported through the group's error word)."""
    import ctypes

    from elasticdl_b200 import _lib

    group, _, _ = make_pair(1)
    lib = _lib.lib()
    rng = np.random.RandomState(33)
    bounds_l = [3, 27, 16384, 16385, 1000, 2_000_000, 1, 5000]
    T = len(bounds_l)
    bounds = (ctypes.c_int64 * T)(*bounds_l)
    need = lib.b200ps_unique_bounded_workspace(T, k, bounds)
    ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
    uniq = torch.empty(T * k, dtype=torch.int64, device="cuda")
    inv = torch.empty(T * k, dtype=torch.int32, device="cuda")
    n = torch.empty(T, dtype=torch.int32, device="cuda")
    for call in range(3):
        ids = np.stack([rng.randint(0, b, size=k) for b in bounds_l]).astype(np.int64)
        if call == 1:
            ids[1, 5] = 10 ** 9   # out of range: counted as id 0, and b200ps_check raises
            ids[4, 0] = -7
        d_ids = torch.from_numpy(ids).cuda()
        _lib.check(lib.b200ps_unique_bounded(group._h, d_ids.data_ptr(), T, k, bounds, uniq.data_ptr(), inv.data_ptr(),
                                             n.data_ptr(), ws.data_ptr(), ws.numel(), group._stream()))
        if call == 1:
            with pytest.raises(_lib.PSRangeError):
                group.check()
        group.check()
        u, i, c = uniq.cpu().numpy().reshape(T, k), inv.cpu().numpy().reshape(T, k), n.cpu().numpy()
        for t in range(T):
            seen = ids[t].copy()
            seen[(seen < 0) | (seen >= bounds_l[t])] = 0
            wu, wi = O.unique_first_occurrence(seen)
            assert c[t] == len(wu) and np.array_equal(u[t, : c[t]], wu) and np.array_equal(i[t], wi), (t, call)
    group.close()


# ------------------------------------------------------------------ golden vectors produced by the reference's own kernels
def _ref_kernel_cases():
    import os
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import gen_kernel_vectors as G

    return G.cases()


@pytest.mark.parametrize("name,kind,hp,n", _ref_kernel_cases(), ids=[c[0] for c in _ref_kernel_cases()])
def test_raw_kernels_reproduce_reference_kernel_vectors(name, kind, hp, n):
    """tests/golden/ref_kernel_vectors.npz = outputs of /root/reference's kernel_api.cc compiled unmodified
    (oracle/_ref, tests/golden/gen_kernel_vectors.py).  The kernel_api.h drop-ins on the GPU reproduce them bit for
    bit over three successive applications (slots feed back; Adam's double bias correction at steps 1..100002)."""
    import ctypes
    import os

    from elasticdl_b200 import _lib

    lib = _lib.lib()
    vec = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_kernel_vectors.npz"))
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    g3 = torch.from_numpy(vec[name + "/g"]).cuda()
    p, s0, s1, s2 = [torch.from_numpy(vec[name + "/in_" + k].copy()).cuda() for k in ("p", "s0", "s1", "s2")]
    for k in range(3):
        g = g3[k].contiguous()
        if kind == "sgd":
            rc = lib.b200ps_kernel_sgd(g.data_ptr(), p.data_ptr(), hp["lr"], n, st)
        elif kind == "momentum":
            rc = lib.b200ps_kernel_momentum(g.data_ptr(), p.data_ptr(), s0.data_ptr(), hp["mu"], hp["nesterov"], hp["lr"],
                                            n, st)
        elif kind == "adam":
            rc = lib.b200ps_kernel_adam(g.data_ptr(), p.data_ptr(), s0.data_ptr(), s1.data_ptr(), hp["lr"], n,
                                        hp["step"] + k, hp["beta1"], hp["beta2"], hp["eps"],
                                        s2.data_ptr() if hp["ams"] else None, st)
        else:
            rc = lib.b200ps_kernel_adagrad(g.data_ptr(), p.data_ptr(), s0.data_ptr(), hp["lr"], n, hp["eps"], st)
        _lib.check(rc)
    for k, t in (("p", p), ("s0", s0), ("s1", s1), ("s2", s2)):
        got = t.cpu().numpy().view(np.uint32)
        want = vec[name + "/out_" + k].view(np.uint32)
        assert np.array_equal(got, want), (name, k, int((got != want).sum()))
