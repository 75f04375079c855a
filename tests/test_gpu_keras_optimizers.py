"""The Keras optimizers the PS applies besides the Go four and FTRL (RMSprop and its momentum / centered variants,
Adadelta, Adamax, Nadam) on the device, bit for bit against oracle/keras_optim_oracle.py.

Gradients are multiples of 1/64 in [-4, 4], so a duplicated id's gradient sum is exact in any order and every
comparison is bitwise, duplicates included.  Several pushes run before the comparison, so every slot and every
per-push scalar (Adamax's bias correction, Nadam's schedule) is non-zero."""
import zlib

import numpy as np
import pytest
import torch

from oracle import keras_optim_oracle as K
from oracle import ps_oracle as O
from tests.test_gpu_parity import _setup_model, info, oinfo

pytestmark = pytest.mark.gpu
F = np.float32

KERAS_OPTS = {
    "rmsprop": ("RMSprop", "learning_rate=0.01;rho=0.9;momentum=0.0;epsilon=1e-07;centered=false;"),
    "rmsprop_momentum": ("RMSprop", "learning_rate=0.01;rho=0.9;momentum=0.5;epsilon=1e-07;centered=false;"),
    "rmsprop_centered": ("RMSprop", "learning_rate=0.01;rho=0.9;momentum=0.0;epsilon=1e-07;centered=true;"),
    "rmsprop_centered_momentum": ("RMSprop", "learning_rate=0.01;rho=0.8;momentum=0.9;epsilon=1e-07;centered=true;"),
    "adadelta": ("Adadelta", "learning_rate=1.0;rho=0.95;epsilon=1e-07;"),
    "adamax": ("Adamax", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;"),
    "nadam": ("Nadam", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;"),
}


def make_pair(n_shards, opt):
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient

    ot, oa = KERAS_OPTS[opt]
    group = PSGroup(n_shards, ot, oa, device=0)
    servers = [K.KerasOracleServer(i, ot, oa, num_ps=n_shards) for i in range(n_shards)]
    return group, PSClient(group), O.OraclePSClient(servers)


def _q(rng, *shape):
    """Gradients whose sums are exact: multiples of 1/64 in [-4, 4]."""
    return (rng.randint(-256, 257, shape) / 64.0).astype(F)


def _grads(rng, dims, step, dup):
    from elasticdl_b200.common.tensor_utils import Tensor

    dense = [("t1", _q(rng, 2, 3)), ("t2", _q(rng, 64, 8) if step % 2 else None), ("bias", _q(rng, 7)),
             ("big", _q(rng, 1000, 16))]
    sparse_dense = ("t2", _q(rng, 20, 8), (rng.randint(0, 64, 20) if dup else rng.permutation(64)[:20]).astype(np.int64))
    edl = []
    for d in dims:
        ids = (rng.randint(0, 200, 300) if dup else rng.permutation(500)[:300]).astype(np.int64)
        edl.append(("e%d" % d, _q(rng, 300, d), ids))

    def build(T):
        grads = [T(n, v.copy(), None) for n, v in dense if v is not None]
        if not step % 2:
            grads.append(T(sparse_dense[0], sparse_dense[1].copy(), sparse_dense[2].copy()))
        return grads, [T(n, v.copy(), i.copy()) for n, v, i in edl]
    return build(Tensor), build(O.Tensor)


def _check_state(group, client, oc, dense, dims, n_shards):
    for name in dense:
        srv = oc.servers[oc.parameter_to_ps[name]]
        assert np.array_equal(group.pull_dense([name])[name].cpu().numpy(), srv.dense[name]), name
        for k, sn in enumerate(srv.opt.slot_names):
            got = group.slot_dense(name, k + 1).cpu().numpy()
            assert np.array_equal(got, srv.opt.dense_slots[sn][name]), (name, sn)
            assert got.any(), (name, sn)
    all_ids = np.arange(500, dtype=np.int64)
    for d in dims:
        name = "e%d" % d
        got = client.pull_embedding_vectors(name, all_ids)
        for s in oc.servers:
            m = all_ids % n_shards == s.id
            touched = np.isin(all_ids[m], s.tables[name].keys())
            ids_t = all_ids[m][touched]
            assert np.array_equal(got[m][touched], s.tables[name].get(ids_t)), name
            assert not got[m][~touched].any()  # rows outside every push stay untouched
            for k, sn in enumerate(s.opt.slot_names):  # slot_rows reads each slot under its index
                gs = group.slot_rows(name, ids_t, k + 1).cpu().numpy()
                assert np.array_equal(gs, s.opt.table_slots[sn][name].get(ids_t)), (name, sn)
                assert not group.slot_rows(name, all_ids[m][~touched], k + 1).cpu().numpy().any()


@pytest.mark.parametrize("opt", list(KERAS_OPTS))
@pytest.mark.parametrize("n_shards", [1, 2, 3])
@pytest.mark.parametrize("dup", [False, True])
def test_push_gradients_match_oracle_bitwise(opt, n_shards, dup):
    group, client, oc = make_pair(n_shards, opt)
    rng = np.random.RandomState(zlib.crc32(repr((opt, n_shards, dup)).encode()))
    dims = (1, 8, 10)
    dense = _setup_model(client, oc, rng, dims)
    versions = [0] * n_shards
    for step in range(5):
        (grads, edl), (ograds, oedl) = _grads(rng, dims, step, dup)
        lr = 0.5 * float(KERAS_OPTS[opt][1].split(";")[0].split("=")[1]) if step == 2 else 0.0
        acc, v = client.push_gradients(grads, edl, lr, versions)
        oacc, ov = oc.push_gradients(ograds, oedl, lr, list(versions))
        assert (acc, v) == (oacc, ov) == (True, step + 1)
        versions = [v] * n_shards
    assert len(oc.servers[0].opt.slot_names) == len(K.KINDS[opt][1])
    _check_state(group, client, oc, dense, dims, n_shards)
    group.close()


@pytest.mark.parametrize("opt", list(KERAS_OPTS))
@pytest.mark.parametrize("dim", [1, 8])
def test_hashed_table_matches_oracle_bitwise(opt, dim):
    from elasticdl_b200.common.tensor_utils import Tensor

    n_shards = 2
    group, client, oc = make_pair(n_shards, opt)
    client.push_embedding_table_infos([info("h", dim, capacity=None)])
    oc.push_embedding_table_infos([oinfo("h", dim)])
    rng = np.random.RandomState(zlib.crc32(repr((opt, dim)).encode()))
    pool = np.unique(rng.randint(0, 2 ** 40, 400)).astype(np.int64)
    versions = [0] * n_shards
    for step in range(4):
        ids = rng.choice(pool, 300)
        g = _q(rng, 300, dim)
        acc, v = client.push_gradients([], [Tensor("h", g.copy(), ids.copy())], 0.0, versions)
        oacc, ov = oc.push_gradients([], [O.Tensor("h", g.copy(), ids.copy())], 0.0, list(versions))
        assert (acc, v) == (oacc, ov)
        versions = [v] * n_shards
    for s in oc.servers:
        keys = s.tables["h"].keys()
        assert np.array_equal(client.pull_embedding_vectors("h", keys), s.tables["h"].get(keys))
        for k, sn in enumerate(s.opt.slot_names):
            assert np.array_equal(group.slot_rows("h", keys, k + 1).cpu().numpy(),
                                  s.opt.table_slots[sn]["h"].get(keys)), sn
    group.close()


@pytest.mark.parametrize("opt", list(KERAS_OPTS))
def test_push_rows_direct_equals_oracle_rows_update(opt):
    """b200ps_push_rows with a step bumped per push, on unique ids of several tables in one launch: each row is
    the oracle's apply_rows of its gradient at that step."""
    group, client, oc = make_pair(1, opt)
    kind, hp = K.hyper_params(*KERAS_OPTS[opt])
    dims = (4, 16, 64)
    client.push_embedding_table_infos([info("r%d" % d, d, capacity=4096) for d in dims])
    rng = np.random.RandomState(zlib.crc32(opt.encode()))
    dev = torch.device("cuda", 0)
    state = {}
    for d in dims:
        ids = rng.permutation(4096)[:1500].astype(np.int64)
        rows = rng.randn(1500, d).astype(F)
        group.set_rows([("r%d" % d, ids, rows)])
        state[d] = (ids, rows, [np.zeros((1500, d), dtype=F) for _ in K.KINDS[kind][1]])
    keep = []
    for t in range(1, 6):
        segs = []
        for d in dims:
            ids, rows, slots = state[d]
            g = _q(rng, 1500, d)
            ids_d, g_d = torch.from_numpy(ids).to(dev), torch.from_numpy(g).to(dev)
            keep += [ids_d, g_d]
            segs.append((group.lookup("r%d" % d)[0], 1500, ids_d, None, g_d))
            rows, slots = K.apply_rows(kind, hp, rows, slots, g, hp["lr"], t)
            state[d] = (ids, rows, slots)
        group.push_begin(0.0, [0])
        group.push_rows(segs)
        group.push_end()
    for d in dims:
        ids, rows, slots = state[d]
        assert np.array_equal(client.pull_embedding_vectors("r%d" % d, ids), rows), d
        for k, want in enumerate(slots):
            assert np.array_equal(group.slot_rows("r%d" % d, ids, k + 1).cpu().numpy(), want), (d, k)
    group.close()


@pytest.mark.parametrize("opt", ["rmsprop_centered_momentum", "adadelta", "nadam"])
def test_checkpoint_restore_restarts_every_slot_at_zero(opt, tmp_path):
    from elasticdl_b200.common.tensor_utils import Tensor
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.ps import checkpoint as ck
    from elasticdl_b200.worker.ps_client import PSClient

    group, client, _ = make_pair(2, opt)
    client.push_embedding_table_infos([info("e1", 2, capacity=64)])
    ids = np.arange(6, dtype=np.int64)
    group.set_rows([("e1", ids, np.arange(12, dtype=F).reshape(6, 2))])
    dense = {"w": np.arange(6, dtype=F).reshape(2, 3)}
    client.partition_dense_parameters(dense.keys())
    for ps_id in set(client.parameter_to_ps.values()):
        client.push_dense_parameters([Tensor(n, v, None) for n, v in dense.items()], ps_id, 0)
    for _ in range(3):
        client.push_gradients([Tensor("w", np.ones((2, 3), dtype=F), None)],
                              [Tensor("e1", np.ones((6, 2), dtype=F), ids)], 0.0, [0, 0])
    n_slots = len(K.KINDS[opt][1])
    assert all(group.slot_rows("e1", ids, k + 1).cpu().numpy().all() for k in range(n_slots))
    want_rows = client.pull_embedding_vectors("e1", ids)
    vdir = ck.save(group, str(tmp_path), keep_checkpoint_max=1)
    group.close()

    g3 = PSGroup(3, *KERAS_OPTS[opt], device=0)
    c3 = PSClient(g3)
    c3.push_embedding_table_infos([info("e1", 2, capacity=64)])
    assert ck.load(g3, c3, vdir) == 3
    assert np.array_equal(c3.pull_embedding_vectors("e1", ids), want_rows)
    for k in range(n_slots):
        assert not g3.slot_rows("e1", ids, k + 1).cpu().numpy().any(), k
        assert not g3.slot_dense("w", k + 1).cpu().numpy().any(), k
    g3.close()


@pytest.mark.parametrize("opt", list(KERAS_OPTS))
def test_dense_reduce_average_matches_oracle_bitwise(opt):
    """The sync-SGD dense reduce (grads_to_wait = 2: two replicas summed, the sum divided by 2) then the update."""
    from elasticdl_b200.common.tensor_utils import Tensor

    group, client, _ = make_pair(1, opt)
    kind, hp = K.hyper_params(*KERAS_OPTS[opt])
    rng = np.random.RandomState(zlib.crc32(("reduce", opt).__repr__().encode()))
    p = rng.randn(257, 12).astype(F)
    client.partition_dense_parameters(["w"])
    client.push_dense_parameters([Tensor("w", p.copy(), None)], 0, 0)
    slots = [np.zeros_like(p) for _ in K.KINDS[kind][1]]
    dev = torch.device("cuda", 0)
    for t in range(1, 5):
        g1, g2 = _q(rng, 257, 12), _q(rng, 257, 12)
        group.push_begin(0.0, [0])
        group.push_dense_reduce("w", [torch.from_numpy(g1).to(dev), torch.from_numpy(g2).to(dev)], 2.0, divide=True)
        group.push_end()
        K.update(kind, hp, (g1 + g2) / F(2), p, slots, *K.push_scalars(kind, hp, hp["lr"], t))
    assert np.array_equal(group.pull_dense(["w"])["w"].cpu().numpy(), p)
    for k, want in enumerate(slots):
        assert np.array_equal(group.slot_dense("w", k + 1).cpu().numpy(), want), k
    group.close()


@pytest.mark.parametrize("opt", list(KERAS_OPTS))
@pytest.mark.parametrize("n_shards", [1, 3])
def test_paired_records_match_oracle_bitwise(opt, n_shards):
    """k_pair_push<OPT>: three pairs (dim-8 A + dim-1 B in one record per id, the per-slot-count lane layouts) in
    one b200ps_push_rows_pair launch per round, device-side live counts that are not multiples of the rows per warp,
    an explicit and the optimizer's own lr.  Params and every slot of both halves equal the oracle (each pair = two
    ordinary tables) after every round; a row no push reached keeps zero slots."""
    group, client, oc = make_pair(n_shards, opt)
    lib = group.lib
    caps = (7, 3000, 50_003)
    names = [("pa%d" % i, "pb%d" % i) for i in range(len(caps))]
    tids = [group.register_pair(a, b, c) for (a, b), c in zip(names, caps)]
    group.commit()
    oc.push_embedding_table_infos([oinfo(n, d) for a, b in names for n, d in ((a, 8), (b, 1))])
    n_slots = len(K.KINDS[opt][1])
    rng = np.random.RandomState(zlib.crc32(repr(("pair", opt, n_shards)).encode()))
    seg_n, live_n = [7, 2000, 30_000], [5, 1997, 29_995]
    seen = [np.zeros(0, dtype=np.int64) for _ in caps]
    for lr in (0.0, 0.5 * float(KERAS_OPTS[opt][1].split(";")[0].split("=")[1]), 0.0, 0.0):
        items, rows_b, keep, ograds = [], [], [], []
        for (ta, _), cap, n, live, (a, b), i in zip(tids, caps, seg_n, live_n, names, range(3)):
            ids = rng.permutation(cap)[:n].astype(np.int64)
            ga, gb = _q(rng, n, 8), _q(rng, n)
            t_ids = torch.from_numpy(ids).cuda()
            n_dev = torch.tensor([live], dtype=torch.int32, device="cuda")
            t_ga, t_gb = torch.from_numpy(ga).cuda(), torch.from_numpy(gb).cuda()
            keep.append((t_ids, n_dev, t_ga, t_gb))
            items.append((ta, n, t_ids, n_dev, t_ga))
            rows_b.append(t_gb)
            ograds += [O.Tensor(a, ga[:live].copy(), ids[:live].copy()),
                       O.Tensor(b, gb[:live].reshape(-1, 1).copy(), ids[:live].copy())]
            seen[i] = np.union1d(seen[i], ids[:live])
        group.push_begin(lr, [0] * n_shards)
        group.pair_call(lib.b200ps_push_rows_pair, items, rows_b)
        group.push_end()
        group.check()
        oc.push_gradients([], ograds, lr, [0] * n_shards)
        for (a, b), ids in zip(names, seen):
            for name in (a, b):
                for k in range(n_slots + 1):
                    got = group.slot_rows(name, ids, k).cpu().numpy()
                    want = np.empty_like(got)
                    for s in oc.servers:
                        m = ids % n_shards == s.id
                        t = s.tables[name] if k == 0 else s.opt.table_slots[s.opt.slot_names[k - 1]][name]
                        want[m] = t.get(ids[m])
                    assert np.array_equal(got, want), (name, k)
    untouched = np.setdiff1d(np.arange(caps[2]), seen[2])[:100]
    for k in range(1, n_slots + 1):
        assert not group.slot_rows(names[2][0], untouched, k).cpu().numpy().any(), k
    group.close()


@pytest.mark.parametrize("opt", ["adamax", "nadam"])
def test_per_push_scalars_match_oracle_over_a_long_range_of_steps(opt):
    """Adamax's lr / (1 - b1^t) and Nadam's folded scalars come from device double pow / sqrt in k_push_begin and from
    the host's in the oracle.  At shard steps from 1 to 10^7 (past the end of Nadam's schedule table), one push of a
    known row state gives the same row and slots, bit for bit, as the oracle's update at that step."""
    group, client, _ = make_pair(1, opt)
    kind, hp = K.hyper_params(*KERAS_OPTS[opt])
    dim, n = 16, 64
    client.push_embedding_table_infos([info("s", dim, capacity=n)])
    rng = np.random.RandomState(zlib.crc32(("steps", opt).__repr__().encode()))
    steps = np.unique(np.concatenate([np.arange(1, 400), rng.randint(400, 10 ** 7, 200)]))
    ids = np.arange(n, dtype=np.int64)
    ids_d = torch.from_numpy(ids).cuda()
    p0 = rng.randn(n, dim).astype(F)
    s0 = [np.abs(rng.randn(n, dim)).astype(F) * F(0.1) for _ in K.KINDS[kind][1]]
    tid = group.lookup("s")[0]
    for t in steps:
        g = (rng.randn(n, dim)).astype(F)
        group.set_rows([("s", ids, p0)])
        for k, x in enumerate(s0):
            group.slot_rows("s", ids, k + 1, values=x)
        group.set_shard_state(0, step=int(t) - 1)
        g_d = torch.from_numpy(g).cuda()
        group.push_begin(0.0, [0])
        group.push_rows([(tid, n, ids_d, None, g_d)])
        group.push_end()
        want_p, want_s = K.apply_rows(kind, hp, p0, s0, g, hp["lr"], int(t))
        assert np.array_equal(group.pull_rows([("s", ids)])[0].cpu().numpy(), want_p), t
        for k, w in enumerate(want_s):
            assert np.array_equal(group.slot_rows("s", ids, k + 1).cpu().numpy(), w), (t, k)
    group.close()


ENGINE_OPTS = {
    "rmsprop_momentum": KERAS_OPTS["rmsprop_momentum"],
    "rmsprop_centered": KERAS_OPTS["rmsprop_centered"],
    "rmsprop_centered_momentum": KERAS_OPTS["rmsprop_centered_momentum"],
    "nadam": KERAS_OPTS["nadam"],
}


@pytest.mark.parametrize("opt", list(ENGINE_OPTS))
def test_deepfm_engine_graph_steps_push_the_oracle_update(opt):
    """DeepFMPSEngine trained by graph replays: after every step the batch's unique rows of every table and the dense
    parameters (params and every slot) equal the oracle's update of the gradients the engine pushed, from the
    pre-step state, at that step and the engine's lr (it pushes with an explicit learning rate); rows outside the
    batch keep their values."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch, synthetic_batch

    ot, oa = ENGINE_OPTS[opt]
    kind, hp = K.hyper_params(ot, oa)
    n_slots = len(K.KINDS[kind][1])
    rows, B = [7, 11, 1000, 50_000], 4096
    dev = torch.device("cuda", 0)
    group = PSGroup(1, ot, oa, device=0)
    try:
        eng = DeepFMPSEngine(group, B, group_rows=rows)
        eng.capture()
        tables = [(n, g, "wide") for g, n in enumerate(eng.wide_names)] + [(n, g, "deep") for g, n in enumerate(eng.deep_names)]

        def state(name, ids):  # pull_rows creates (initializes) a row as the engine's own pull would
            t = torch.from_numpy(np.ascontiguousarray(ids, dtype=np.int64))
            return [group.pull_rows([(name, t)])[0].cpu().numpy()] + [
                group.slot_rows(name, t, k).cpu().numpy() for k in range(1, n_slots + 1)]

        def dense_state():
            return {name: [group.pull_dense([name])[name].cpu().numpy().reshape(-1)] +
                    [group.slot_dense(name, k).cpu().numpy().reshape(-1) for k in range(1, n_slots + 1)]
                    for name, _ in eng.params}

        sample = [np.arange(min(r, 2048)) for r in rows]
        for t in range(1, 5):
            ids, dense, labels = synthetic_batch(B, t, dev, "zipf", group_rows=rows)
            dedup = [O.unique_first_occurrence(row) for row in ids.cpu().numpy()]
            pre = {name: (state(name, dedup[g][0]), state(name, sample[g])) for name, g, _ in tables}
            dense0 = dense_state()
            eng.step_graph(pack_batch(ids, dense, labels, widths=eng.widths))
            torch.cuda.synchronize()
            group.check()
            gsum = {"wide": eng.gsum_w.view(eng.G, B, 1).cpu().numpy(), "deep": eng.gsum_d.view(eng.G, B, eng.D).cpu().numpy()}
            for name, g, fam in tables:
                u = dedup[g][0]
                (before, sample0) = pre[name]
                want_p, want_s = K.apply_rows(kind, hp, before[0], before[1:], gsum[fam][g, :len(u)], eng.lr, t)
                for k, (a, b) in enumerate(zip(state(name, u), [want_p] + want_s)):
                    assert np.array_equal(a, b), (opt, t, name, k, float(np.abs(a - b).max()))
                outside = ~np.isin(sample[g], u)
                for k, (a, b) in enumerate(zip(state(name, sample[g]), sample0)):
                    assert np.array_equal(a[outside], b[outside]), (opt, t, name, k)
            flat_g = eng.flat_grads.cpu().numpy()
            dense1 = dense_state()
            for (name, _), (off, n) in zip(eng.params, eng.flat_views):
                want_p, want_s = K.apply_rows(kind, hp, dense0[name][0], dense0[name][1:], flat_g[off:off + n],
                                              eng.lr, t)
                for k, (a, b) in enumerate(zip(dense1[name], [want_p] + want_s)):
                    assert np.array_equal(a, b), (opt, t, name, k)
            assert group.snapshot() == [(t, t, True)], t
    finally:
        group.close()
