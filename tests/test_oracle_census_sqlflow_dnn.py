"""census_model_sqlflow's DNNClassifier (workloads/fc_dnn.py CENSUS_SQLFLOW_DNN) on the CPU: its layout and column
order, its ids from raw strings against oracle/feature_oracle.py, the truncated-normal initialiser of its kept-dense
tables, the float64 Indexed Adam of oracle/census_sqlflow_dnn_oracle.py against the PS restatement of
oracle/ps_oracle.py and on the rows it must not touch, and ParameterServerModelHandler keeping the twin's 64 x 16
tables as dense parameters under the engine's names (DESIGN.md section 4, Q36)."""
import numpy as np
import pytest
import torch

from elasticdl_b200.common.model_handler import ParameterServerModelHandler, need_partition_embedding
from elasticdl_b200.layers.dense_table import DenseTableEmbedding
from elasticdl_b200.layers.embedding import Embedding
from elasticdl_b200.workloads import fc_dnn as M
from oracle import census_sqlflow_dnn_oracle as CO
from oracle import feature_oracle as FO
from oracle.ps_oracle import OracleServer

L = M.CENSUS_SQLFLOW_DNN
ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")


def test_layout():
    assert M.layout_of("census_model_sqlflow_dnn") is L
    assert (L.F, L.n_mlp) == (4 + 8 * 16, 16 * 132 + 305)
    # Q17: DenseFeatures sorts its columns by name
    assert [c for c, _, _ in L.columns] == [
        "age", "capital-gain", "capital-loss", "education_embedding", "hours-per-week", "marital-status_embedding",
        "native-country_embedding", "occupation_embedding", "race_embedding", "relationship_embedding",
        "sex_embedding", "workclass_embedding"]
    assert [o for _, _, _, o in L.blocks] == [0, 1, 2, 3, 19, 20, 36, 52, 68, 84, 100, 116]
    assert [(r, d) for _, r, d in L.tables] == [(64, 16)] * 8
    assert L.table_names[0] == "dense_features/workclass_embedding/embedding_weights:0"
    assert L.table_kinds == [M.DENSE_TABLE] * 8
    assert L.spec()["table_kinds"] == ["dense"] * 8
    assert not L.loss_mean  # census_functional.py:51-53: per-sample losses, batch sums (Q16)
    assert L.optimizer == ("Adam", ADAM[1], 1e-3)  # census_functional.py:56-57: Adam() defaults
    assert [n for n, _ in L.mlp] == M.MLP_NAMES
    # the tower reads the same layout as census_dnn_model's: only the tables' kind differs
    assert bytes(L.c) == bytes(M.CENSUS_DNN.c)
    assert {k: v for k, v in L.spec().items() if k != "table_kinds"} == \
        {k: v for k, v in M.CENSUS_DNN.spec().items() if k != "table_kinds"}
    # the two earlier layouts keep hashed PS tables
    assert M.CENSUS_DNN.table_kinds == [M.PS_TABLE] * 8 and M.HEART.table_kinds == [M.PS_TABLE]
    assert M.CENSUS_DNN.initial_tables(0) == {} and M.HEART.initial_tables(0) == {}
    with pytest.raises(ValueError, match="table_kinds"):
        M.Layout("bad", ["a"], ["s"], tables=[("s", 8, 4)], buckets=[],
                 columns=[("a", M.NUMERIC, "a"), ("s_embedding", M.EMBEDDING, "s")], loss_mean=False,
                 optimizer=None, table_kinds=["sparse"])


def test_ids_from_raw_strings():
    """categorical_column_with_hash_bucket(key, 64) over each string column: Fingerprint64 % 64, "" to id 0."""
    gs = L.groups()
    assert gs == M.CENSUS_DNN.groups()
    for k, (key, rows, _) in enumerate(L.tables):
        assert gs[k] == {"kind": "hash", "column": L.string_keys.index(key), "num_bins": 64}
    raw = ["Private", "", "Self-emp-not-inc", "Bachelors", "", "United-States", "?", "x" * 32]
    want = FO.hashing([s for s in raw], 64)
    got = CO.ids_from_strings(raw, 64)
    assert got.dtype == np.int64 and got.tolist() == [0 if s == "" else int(w) for s, w in zip(raw, want)]
    assert all(0 <= int(i) < 64 for i in got)
    assert FO.hashing(["A", "B", "C", "D", "E"], 3).tolist() == [1, 0, 1, 1, 2]  # hashing.py:35-39


def test_truncated_normal_initialiser():
    t0 = L.initial_tables(0)
    assert list(t0) == L.table_names
    x = torch.stack(list(t0.values()))
    assert x.dtype == torch.float32 and x.shape == (8, 64, 16)
    std = 1.0 / np.sqrt(16)
    assert float(x.abs().max()) <= 2 * std  # redrawn outside two stddevs
    assert float((x.abs() > 1.8 * std).float().mean()) > 0.005  # and not rescaled into a narrower range
    # a normal truncated at two stddevs has stddev 0.8796 sigma; 8192 draws
    assert abs(float(x.double().std()) - 0.87962566 * std) < 0.02 * std
    assert abs(float(x.double().mean())) < 0.01
    again = L.initial_tables(0)
    assert all(torch.equal(t0[n], again[n]) for n in t0)
    other = L.initial_tables(1)
    assert not any(torch.equal(t0[n], other[n]) for n in t0)
    assert len({x[k].sum().item() for k in range(8)}) == 8  # every table its own draws


def _state(seed, rows=64, dim=16):
    g = torch.Generator().manual_seed(seed)
    p = (torch.rand((rows, dim), generator=g) * 2 - 1) * 0.5
    m = (torch.rand((rows, dim), generator=g) * 2 - 1) * 1e-2
    v = torch.rand((rows, dim), generator=g) * 1e-4
    return p, m, v


def test_indexed_adam_touches_the_pushed_rows_only():
    p, m, v = _state(1)
    ids = torch.tensor([0, 5, 17, 63, 40])
    g = (torch.rand((5, 16), generator=torch.Generator().manual_seed(2)) * 2 - 1) * 0.1
    g[0] = 0  # the fill id of empty strings: a zero row, still pushed (Q36)
    step, lr = 3, 1e-3
    p2, m2, v2 = CO.indexed_adam(p, m, v, ids, g, lr, step)
    others = torch.ones(64, dtype=torch.bool)
    others[ids] = False
    for before, after in ((p, p2), (m, m2), (v, v2)):
        assert after.dtype == torch.float64
        assert torch.equal(after[others].float(), before[others])  # bit for bit
        assert not torch.equal(after[ids].float(), before[ids])
    # row 0: zero gradient, nonzero m -> m and v decay and the row moves by lr_t m / (sqrt(v) + eps)
    assert torch.allclose(m2[0], 0.9 * m[0].double()) and torch.allclose(v2[0], 0.999 * v[0].double())
    assert float((p2[0] - p[0].double()).abs().min()) > 0
    # the same update as the PS restatement (float32 C, kernel_api.cc:40-77) on a dense parameter
    srv = OracleServer(0, *ADAM)
    name = L.table_names[0]
    srv.push_model(dense={name: p.numpy()})
    srv.opt.dense_slots["m"][name][...] = m.numpy()
    srv.opt.dense_slots["v"][name][...] = v.numpy()
    srv.opt.step = step - 1  # push_gradients bumps it to `step`
    ok, _ = srv.push_gradients({}, {name: (ids.numpy(), g.numpy())}, lr, 0)
    assert ok
    np.testing.assert_allclose(srv.dense[name], p2.numpy(), rtol=1e-6, atol=1e-8)
    # float32 rounding: half an ulp of the slots' magnitudes (m ~ 1e-2, v ~ 1e-4) per operation
    np.testing.assert_allclose(srv.opt.dense_slots["m"][name], m2.numpy(), rtol=1e-6, atol=2e-9)
    np.testing.assert_allclose(srv.opt.dense_slots["v"][name], v2.numpy(), rtol=1e-6, atol=2e-11)
    with pytest.raises(ValueError, match="unique ids"):
        CO.indexed_adam(p, m, v, torch.tensor([1, 1]), torch.zeros((2, 16)), lr, step)
    spec = L.spec()
    out = CO.apply_dense_tables(spec, {k: (p, m, v) for k in range(8)}, [ids] * 8, [g] * 8, lr, step)
    assert sorted(out) == list(range(8)) and torch.equal(out[3][0], p2)
    assert CO.apply_dense_tables(M.CENSUS_DNN.spec(), {}, [], [], lr, step) == {}


def test_model_handler_keeps_the_twin_tables_dense():
    assert not need_partition_embedding(64, 16)  # 4 KB: at most 2 MB stays a Keras variable
    twin = M.FeatureColumnDNN(L)
    weights = [t.weight for t in twin.tables]
    init = L.initial_tables(0)
    for n, w in zip(L.table_names, weights):
        assert getattr(twin, n) is w and torch.equal(w.detach(), init[n])
    ParameterServerModelHandler().get_model_to_train(twin)
    names = {id(p): n for n, p in twin.named_parameters()}
    for k, (t, w) in enumerate(zip(twin.tables, weights)):
        assert isinstance(t, DenseTableEmbedding) and (t.input_dim, t.output_dim) == (64, 16)
        assert t.weight is w  # the twin's values are what the first writer pushes
        assert names[id(t.weight)] == L.table_names[k]  # the trainer's PS name for the kept table
    assert [n for n, _ in twin.named_parameters()] == L.table_names + M.MLP_NAMES
    # census_dnn_model's twin keeps ElasticDL tables under the same names (hashed PS tables)
    c = M.FeatureColumnDNN(M.CENSUS_DNN)
    ParameterServerModelHandler().get_model_to_train(c)
    assert all(type(t) is Embedding for t in c.tables)
    assert [t.embedding_weight_name for t in c.tables] == M.CENSUS_DNN.table_names
    assert [n for n, _ in c.named_parameters()] == M.MLP_NAMES


def test_twin_forward_matches_the_oracle_on_cpu():
    """The twin's DenseFeatures and MLP before any swap (plain nn.Embedding lookups) against fc_dnn_oracle."""
    from oracle import fc_dnn_oracle as FD

    twin = M.FeatureColumnDNN(L).double()
    B = 50
    g = torch.Generator().manual_seed(4)
    numeric = torch.randn((4, B), generator=g, dtype=torch.float64)
    ids = torch.randint(0, 64, (8, B), generator=g)
    empty = torch.rand((8, B), generator=g) < 0.3
    ids[empty] = 0
    feats = {"numeric": numeric, "buckets": torch.zeros((0, B), dtype=torch.int64),
             "present": (~empty).double()}
    for k, (key, _, _) in enumerate(L.tables):
        feats[key] = ids[k]
    p = twin(feats)
    inv, nu, rows = [], [], []
    for k, n in enumerate(L.table_names):
        u, iv = torch.unique(ids[k], return_inverse=True)
        inv.append(iv.to(torch.int32))
        nu.append(u.numel())
        rows.append(getattr(twin, n).detach()[u])
    flat = torch.cat([getattr(twin, n).detach().reshape(-1) for n in M.MLP_NAMES])
    ref = FD.fc_dnn_reference(L.spec(), numeric, ids.to(torch.int32), empty, torch.stack(inv), nu, rows,
                              torch.zeros(B, dtype=torch.float64), flat)
    torch.testing.assert_close(p.detach(), torch.sigmoid(ref["logits"]), rtol=1e-12, atol=1e-12)
