"""The PRODUCT's worker-side client (elasticdl_b200/worker/ps_client.py) on CPU: its host logic -- name -> PS routing,
merge / dedup / validation of gradients, versions, return values -- driven against a host-memory stand-in of PSGroup
and compared with what the reference's own PSClient did when it was EXECUTED against fake stubs
(tests/golden `ps_client`, written by tests/golden/gen_from_reference.py).

The stand-in replaces only the device: every method PSClient calls on a PSGroup (register_*, commit, lookup, pull_rows,
unique, segment_sum, push_begin / push_dense / push_rows / push_end, snapshot, try_init / set_dense / finish_init,
check) with host tensors and a record of what was asked.  The reference sends one request per PS; here all shards are
addressed by ONE call (`id % N` inside the kernels), so the comparison is on the union over PS of the reference's
requests: the same dense gradients by name, the same (id -> summed gradient row) per table, the same learning rate,
pulled rows in the caller's id order, the same uninitialised-PS list and versions written back."""
import json
import os

import numpy as np
import pytest
import torch

from elasticdl_b200.common.tensor_utils import EmbeddingTableInfo, Tensor
from elasticdl_b200.ps.group import PSGroup
from elasticdl_b200.worker.ps_client import PSClient

F = np.float32
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_python_vectors.json")


class HostGroup(PSGroup):
    """PSGroup's interface over host memory (no CUDA, no library): a test double for the product's host logic."""

    def __init__(self, n_shards, fake):  # noqa: super().__init__ needs a device
        self._h = None
        self.n_shards = n_shards
        self.local_shards = list(range(n_shards))
        self.device = torch.device("cpu")
        self.use_async = True
        self.tables, self.dense_owner, self.table_initializers = {}, {}, {}
        self.fake = fake  # the FakeStub script of the golden generator: initialized / version0 per PS
        self.versions = [f["version0"] for f in fake]
        self.initialized = [f["initialized"] for f in fake]
        self.dense_values = {}
        self.calls = []

    def close(self):
        pass

    # definition
    def register_table(self, name, dim, initializer="uniform", capacity=None, expected_rows=None):
        if name not in self.tables:
            self.tables[name] = (len(self.tables), int(dim), False, (capacity, int(dim)))
            self.table_initializers[name] = str(initializer)
            self.calls.append(["register_table", name, int(dim), str(initializer)])
        return self.tables[name][0]

    def register_dense(self, name, shape, shard):
        if name not in self.tables:
            shape = tuple(int(x) for x in shape)
            numel = int(np.prod(shape)) if len(shape) else 1
            rows = shape[0] if len(shape) >= 2 else numel
            self.tables[name] = (len(self.tables), numel // rows if rows else 1, True, shape)
            self.dense_owner[name] = int(shard)
        return self.tables[name][0]

    def commit(self):
        pass

    def check(self):
        pass

    def _ids(self, ids):
        return torch.as_tensor(np.asarray(ids) if not isinstance(ids, torch.Tensor) else ids).to(torch.int64).reshape(-1)

    def _f32(self, v):
        return torch.as_tensor(np.asarray(v) if not isinstance(v, torch.Tensor) else v).to(torch.float32).contiguous()

    def _name_of(self, tid):
        return next(n for n, t in self.tables.items() if t[0] == tid)

    # data path
    def pull_rows(self, requests):
        outs = []
        for name, ids in requests:
            ids = self._ids(ids).tolist()
            self.calls.append(["pull_rows", name, ids])
            dim = self.lookup(name)[1]
            outs.append(torch.tensor([[i + 0.25 * c for c in range(dim)] for i in ids], dtype=torch.float32))
        return outs

    def unique(self, ids, T=1, bounds=None):
        assert T == 1
        ids = self._ids(ids)
        first, uniq, inv = {}, [], []
        for i in ids.tolist():  # tf.unique: first-occurrence order
            if i not in first:
                first[i] = len(uniq)
                uniq.append(i)
            inv.append(first[i])
        pad = uniq + [0] * (ids.numel() - len(uniq))
        return (torch.tensor(pad, dtype=torch.int64), torch.tensor(inv, dtype=torch.int32),
                torch.tensor([len(uniq)], dtype=torch.int32))

    def segment_sum(self, values, inv, T, k, dim, out=None):
        values = self._f32(values).reshape(k, dim).numpy()
        out = np.zeros((k, dim), F)
        seen = set()
        for pos, j in enumerate(inv.tolist()):  # occurrence order, first occurrence assigns (tensor_utils.py:53-58)
            if j in seen:
                out[j] += values[pos]
            else:
                out[j] = values[pos]
                seen.add(j)
        return torch.from_numpy(out)

    def snapshot(self):
        return [(self.versions[s], 0, self.initialized[s]) for s in range(self.n_shards)]

    def pull_dense(self, names, into=None):
        self.calls.append(["pull_dense", list(names)])
        return {n: torch.zeros(self.lookup(n)[3]) for n in names}

    def try_init(self, shard):
        won = not self.initialized[shard]
        self.calls.append(["try_init", shard, won])
        return won

    def set_dense(self, named_values):
        for name, v in named_values:
            t = self._f32(v)
            assert tuple(t.shape) == tuple(self.lookup(name)[3]), name
            self.calls.append(["set_dense", name, t.reshape(-1).tolist()])

    def finish_init(self, shard, version):
        self.calls.append(["finish_init", shard, int(version)])

    def push_begin(self, learning_rate, model_versions):
        self.calls.append(["push_begin", float(learning_rate), [int(v) for v in model_versions]])

    def bump_step(self):
        self.calls.append(["bump_step"])

    def push_dense(self, items):
        for tid, _, _, _, t in items:
            self.calls.append(["push_dense", self._name_of(tid), list(t.shape), t.reshape(-1).tolist()])

    def push_rows(self, items):
        for tid, n, ids, n_dev, grads in items:
            live = int(n_dev[0]) if n_dev is not None else n
            dim = self.lookup(self._name_of(tid))[1]
            g = grads.reshape(-1, dim)[:live]
            self.calls.append(["push_rows", self._name_of(tid),
                               {int(i): row.tolist() for i, row in zip(ids[:live].tolist(), g)}])

    def push_dense_reduce(self, name, grads, scale=1.0, divide=False):
        self.calls.append(["push_dense_reduce", name, [g.reshape(-1).tolist() for g in grads], float(scale), divide])

    def push_end(self, sync=True):
        self.versions = [v + 1 for v in self.versions]  # every shard, every push (quirk Q7)
        self.calls.append(["push_end"])
        return list(self.versions) if sync else None


def _reference_union(case):
    """Union over PS of the reference's recorded push_gradients requests."""
    dense, tables, lrs, versions = {}, {}, set(), {}
    for method, ps, payload in case["log"]:
        if method != "push_gradients":
            continue
        lrs.add(payload["learning_rate"])
        g = payload["gradients"]
        versions[ps] = g["version"]
        for name, t in g["dense"].items():
            assert name not in dense
            dense[name] = (t["shape"], t["data"])
        for name, t in g["tables"].items():
            rows = np.asarray(t["data"], F).reshape(t["shape"])
            for i, row in zip(t["ids"], rows):
                assert i not in tables.setdefault(name, {})  # an id reaches exactly one PS
                tables[name][i] = row.tolist()
    return dense, tables, lrs, versions


@pytest.mark.parametrize("idx", [0, 1, 2], ids=["1ps", "2ps", "3ps"])
def test_product_ps_client_host_logic_matches_the_executed_reference(idx):
    case = json.load(open(GOLD))["ps_client"][idx]
    n = case["ps_num"]
    group = HostGroup(n, case["fake"])
    client = PSClient(group)
    shapes = {"dense/kernel:0": (3, 2), "dense/bias:0": (3,), "dense_1/kernel:0": (3, 2),
              "emb_keras/embeddings:0": (10, 2), "scalar:0": ()}
    client.partition_dense_parameters(case["param_names"], shapes=shapes)
    assert client.parameter_to_ps == case["parameter_to_ps"]
    assert {str(k): v for k, v in client.ps_to_parameter.items()} == case["ps_to_parameter"]
    client.push_embedding_table_infos([EmbeddingTableInfo(*i) for i in case["infos"]])
    assert [c[1:] for c in group.calls if c[0] == "register_table"] == [i[:3] for i in case["infos"]]

    # push_dense_parameters: each PS gets the parameters that hash to it, first writer wins (only uninitialised PS)
    params = [Tensor(name, np.asarray(v, F), None) for name, v in case["params"]]
    for p in range(n):
        client.push_dense_parameters(params, p, 3)
    want_sets = {}
    for method, ps, payload in case["log"]:
        if method == "push_model":
            want_sets[ps] = {k: v["data"] for k, v in payload["dense"].items()}
    got_sets = {}
    for c in group.calls:
        if c[0] == "try_init":
            cur = c[1] if c[2] else None
            if c[2]:
                got_sets[cur] = {}
        elif c[0] == "set_dense" and cur is not None:
            got_sets[cur][c[1]] = c[2]
    for ps in range(n):
        if not case["fake"][ps]["initialized"]:  # the reference's PS ignores push_model once initialised (server.go:209-221)
            assert got_sets[ps] == want_sets[ps], ps
        else:
            assert ps not in got_sets

    # pull_dense_parameters: same uninitialised list, same versions written back
    versions = list(case["pull_dense"]["versions_in"])
    _, uninit = client.pull_dense_parameters(list(range(n)), versions)
    assert uninit == case["pull_dense"]["uninit"] and versions == case["pull_dense"]["versions_out"]

    # pull_embedding_vectors: rows in the caller's id order (numpy in -> numpy out)
    rows = client.pull_embedding_vectors("edl_emb", np.asarray(case["pull_ids"], np.int64))
    assert isinstance(rows, np.ndarray) and rows.tolist() == case["pull_rows"]

    # push_gradients
    grads = [Tensor(name, np.asarray(v, F), None if i is None else np.asarray(i, np.int64)) for name, v, i in case["grads"]]
    edl = [Tensor(name, np.asarray(v, F), np.asarray(i, np.int64)) for name, v, i in case["edl_grads"]]
    group.calls.clear()
    accepted, max_version = client.push_gradients(grads, edl, case["learning_rate"], list(case["push_versions"]))
    assert [bool(accepted), int(max_version)] == case["push_result"]
    want_dense, want_tables, want_lr, want_versions = _reference_union(case)
    begin = [c for c in group.calls if c[0] == "push_begin"]
    assert len(begin) == 1 and {begin[0][1]} == want_lr and begin[0][2] == [want_versions[p] for p in range(n)]
    got_dense = {c[1]: (c[2], c[3]) for c in group.calls if c[0] == "push_dense"}
    assert got_dense == {k: (list(v[0]), v[1]) for k, v in want_dense.items()}
    got_tables = {c[1]: c[2] for c in group.calls if c[0] == "push_rows"}
    assert set(got_tables) == set(want_tables)
    for name in want_tables:
        assert got_tables[name] == want_tables[name], name
    assert [c[0] for c in group.calls][-1] == "push_end"


def test_product_ps_client_errors_before_any_update():
    """Unknown gradient names and wrong widths fail the whole push after step++ (quirk Q2: optimizer.go:44-59,
    kernel.go:36-38) and before any table is touched."""
    fake = [{"initialized": True, "version0": 0, "accept": True, "dense": {}}]
    group = HostGroup(1, fake)
    client = PSClient(group)
    client.partition_dense_parameters(["w"], shapes={"w": (2, 2)})
    client.push_embedding_table_infos([EmbeddingTableInfo("e", 4, "zeros", 1)])
    with pytest.raises(KeyError):
        client.push_gradients([Tensor("nope", np.zeros((2, 2), F), None)], [], 0.1, [0])
    for bad in ([Tensor("w", np.zeros((3, 2), F), None)], ):
        group.calls.clear()
        with pytest.raises(ValueError):
            client.push_gradients(bad, [], 0.1, [0])
        assert [c[0] for c in group.calls] == ["bump_step"]
    group.calls.clear()
    with pytest.raises(ValueError):
        client.push_gradients([], [Tensor("e", np.zeros((2, 3), F), np.array([1, 2]))], 0.1, [0])
    assert [c[0] for c in group.calls] == ["bump_step"]
    with pytest.raises(ValueError):  # the reference np.concatenate()s an empty list (ps_client.py:123)
        client.pull_embedding_vectors("e", [])


def test_product_sync_sgd_host_logic_divides_pserver_servicer_test_py_366():
    """Sync-SGD as the Python PS does it (python/ps/servicer.py:168-238; vector of pserver_servicer_test.py:366-432):
    grads_to_wait = 2 -> the first push is buffered (accepted, version unchanged), the second applies ONE update with
    the dense gradients averaged (the fused reduce kernel gets both parts and divides their sum by 2) and the sparse gradients
    concatenated then summed per id, version 0 -> 1; a third push that still carries version 0 is rejected."""
    import threading

    fake = [{"initialized": True, "version0": 0, "accept": True, "dense": {}}]
    group = HostGroup(1, fake)
    group.use_async, group.grads_to_wait, group.sync_version_tolerance = False, 2, 0
    group._sync_lock, group._sync_buffer = threading.Lock(), {"n": 0, "dense": {}, "sparse": {}}
    client = PSClient(group)
    rng = np.random.RandomState(3)
    g0 = {"v0": rng.rand(3, 2).astype(F), "v1": rng.rand(3).astype(F)}
    g1 = {"v0": rng.rand(3, 2).astype(F), "v1": rng.rand(3).astype(F)}
    client.partition_dense_parameters(["v0", "v1"], shapes={"v0": (3, 2), "v1": (3,)})
    client.push_embedding_table_infos([EmbeddingTableInfo("emb", 8, "zeros", 1, 16)])
    e0 = (rng.rand(3, 8).astype(F), np.array([3, 1, 3]))
    e1 = (rng.rand(2, 8).astype(F), np.array([1, 9]))
    group.calls.clear()
    assert client.push_gradients([Tensor(n, v, None) for n, v in g0.items()], [Tensor("emb", *e0)], 0.1, [0]) == (True, 0)
    assert [c[0] for c in group.calls] == []  # buffered: nothing reaches the tables
    assert client.push_gradients([Tensor(n, v, None) for n, v in g1.items()], [Tensor("emb", *e1)], 0.1, [0]) == (True, 1)
    kinds = [c[0] for c in group.calls]
    assert kinds == ["push_begin", "push_dense_reduce", "push_dense_reduce", "push_rows", "push_end"]
    assert group.calls[0][1:] == [0.1, [0]]
    for c in group.calls[1:3]:
        name, parts, scale, divide = c[1], c[2], c[3], c[4]
        assert scale == 2 and divide is True and parts == [g0[name].reshape(-1).tolist(), g1[name].reshape(-1).tolist()]
    rows = group.calls[3][2]
    assert group.calls[3][1] == "emb" and list(rows) == [3, 1, 9]  # first-occurrence order over e0 ++ e1
    assert np.array_equal(np.asarray(rows[3], F), e0[0][0] + e0[0][2])
    assert np.array_equal(np.asarray(rows[1], F), e0[0][1] + e1[0][0])
    assert np.array_equal(np.asarray(rows[9], F), e1[0][1])
    group.calls.clear()
    assert client.push_gradients([Tensor(n, v, None) for n, v in g1.items()], [], 0.1, [0]) == (False, 1)
    assert group.calls == []


class StoreGroup(HostGroup):
    """HostGroup that keeps table rows, dense values and per-shard state: enough for ps/checkpoint.py save / load."""

    def __init__(self, n_shards, opt_type="Adam", opt_args=""):
        super().__init__(n_shards, [{"initialized": False, "version0": 0} for _ in range(n_shards)])
        self.opt_type, self.opt_args = opt_type, opt_args
        self.rows, self.dense_store, self.slot_writes = {}, {}, []

    def set_rows(self, requests):
        for name, ids, values in requests:
            dim = self.lookup(name)[1]
            vals = np.asarray(values, F).reshape(len(np.asarray(ids).reshape(-1)), dim)
            for i, v in zip(np.asarray(ids).reshape(-1).tolist(), vals):
                self.rows.setdefault(name, {})[int(i)] = v.copy()

    def slot_rows(self, name, ids, slot, values=None):
        if slot > 2:
            raise ValueError("Adam has two slots")
        self.slot_writes.append((name, sorted(np.asarray(ids).tolist()), slot, float(np.asarray(values).max())))

    def table_ids(self, name, shard):
        return torch.tensor(sorted(i for i in self.rows.get(name, {}) if i % self.n_shards == shard), dtype=torch.int64)

    def pull_rows(self, requests):
        return [torch.from_numpy(np.stack([self.rows[name][int(i)] for i in self._ids(ids).tolist()]))
                for name, ids in requests]

    def set_dense(self, named_values):
        for name, v in named_values:
            t = self._f32(v)
            assert tuple(t.shape) == tuple(self.lookup(name)[3]), name
            self.dense_store[name] = t.numpy().copy()

    def pull_dense(self, names, into=None):
        return {n: torch.from_numpy(self.dense_store[n]) for n in names}

    def set_shard_state(self, shard, version=-1, step=-1, initialized=-1):
        if version >= 0:
            self.versions[shard] = version
        if initialized >= 0:
            self.initialized[shard] = bool(initialized)


def test_checkpoint_save_load_resharding_host_logic_checkpoint_test_go_25(tmp_path):
    """ps/checkpoint.py save -> load over host memory: 2 shards saved, 3 shards restored -- ids {0,2,4} U {1,3,5} land
    on {0,3} {1,4} {2,5} (checkpoint_test.go:25-82), dense parameters re-hash by name, the version is adopted, the
    optimizer slots of restored rows are reset (quirk Q9), and the files are proto.Model messages the protobuf library
    reads (elasticdl.proto:24-29)."""
    import sys

    from elasticdl_b200.common.hash_utils import string_to_id
    from elasticdl_b200.ps import checkpoint as ck

    g2 = StoreGroup(2)
    c2 = PSClient(g2)
    c2.push_embedding_table_infos([EmbeddingTableInfo("e1", 2, "uniform", 1, 64)])
    ids = np.array([0, 2, 4, 1, 3, 5], dtype=np.int64)
    vals = np.arange(12, dtype=F).reshape(6, 2)
    g2.set_rows([("e1", ids, vals)])
    dense = {"dense/kernel:0": np.arange(6, dtype=F).reshape(2, 3), "dense/bias:0": np.array([9, 8, 7], dtype=F)}
    c2.partition_dense_parameters(dense.keys(), shapes={k: v.shape for k, v in dense.items()})
    g2.set_dense(list(dense.items()))
    g2.versions = [3, 3]
    vdir = ck.save(g2, str(tmp_path))
    assert vdir.endswith("version-3") and sorted(os.listdir(vdir)) == ["variables-0-of-2.ckpt", "variables-1-of-2.ckpt"]

    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_cpu_checkpoint_format import _pb_classes  # Model built at runtime from the .proto field numbers

    Model, _ = _pb_classes()
    seen_dense = {}
    for shard in range(2):
        m = Model()
        m.ParseFromString(open(os.path.join(vdir, "variables-%d-of-2.ckpt" % shard), "rb").read())
        assert m.version == 3 and [(i.name, i.dim, i.initializer) for i in m.embedding_table_infos] == [("e1", 2, "uniform")]
        assert sorted(m.embedding_tables["e1"].ids) == [i for i in range(6) if i % 2 == shard]
        for name in m.dense_parameters:
            assert string_to_id(name, 2) == shard  # a dense parameter is saved by the shard that owns it
            seen_dense[name] = np.frombuffer(m.dense_parameters[name].tensor_content, "<f4")
    assert set(seen_dense) == set(dense) and all(np.array_equal(seen_dense[k], dense[k].reshape(-1)) for k in dense)

    g3 = StoreGroup(3)
    c3 = PSClient(g3)
    assert ck.load(g3, c3, ck.latest_version_dir(str(tmp_path))) == 3
    assert [g3.table_ids("e1", s).tolist() for s in range(3)] == [[0, 3], [1, 4], [2, 5]]
    assert np.array_equal(c3.pull_embedding_vectors("e1", ids), vals)
    assert g3.versions == [3, 3, 3] and g3.initialized == [True, True, True]
    assert {k: c3.parameter_to_ps[k] for k in dense} == {k: string_to_id(k, 3) for k in dense}
    assert all(np.array_equal(g3.dense_store[k], dense[k]) for k in dense)
    assert [(w[0], w[1], w[2], w[3]) for w in g3.slot_writes] == [("e1", [0, 1, 2, 3, 4, 5], 1, 0.0), ("e1", [0, 1, 2, 3, 4, 5], 2, 0.0)]
