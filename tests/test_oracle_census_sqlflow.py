"""The census_model_sqlflow oracle (oracle/census_sqlflow_oracle.py) and configuration on the CPU: the tower oracle
against float64 autograd with absent ids and empty groups in both reshape modes; the offsets, dims and sizes against
feature_configs.py's literal numbers; hand-written raw rows for every dropping and aliasing case of both id rules;
the feature-transform specs; the five model files' reshape modes and names; the zoo's schedule against its literal
_schedule; every mutation moving the outputs."""
import numpy as np
import pytest
import torch

from elasticdl_b200.workloads import census_sqlflow as M
from elasticdl_b200.workloads import census_sqlflow_features as F
from oracle import census_sqlflow_oracle as O


def _ids(B, gen, absent=0.3, empty_group=None):
    rows = []
    for g, r in enumerate(O.GROUP_ROWS):
        v = torch.randint(0, r, (4, B), generator=gen)
        v[torch.rand((4, B), generator=gen) < absent] = -1
        if empty_group == g:
            v[:, ::2] = -1  # every other sample has no id in this group
        rows.append(v)
    return torch.cat(rows)


def _batch(B, seed, empty_group=None):
    gen = torch.Generator().manual_seed(seed)
    ids = _ids(B, gen, empty_group=empty_group)
    labels = (torch.rand(B, generator=gen) < 0.3).double()
    flat = O.random_params(gen, "cpu", dtype=torch.float64)
    return ids, labels, flat


def _autograd(ids, labels, flat, q11):
    """The model in torch float64 autograd: mean pooling by embedding_bag over the present ids."""
    flat = flat.clone().requires_grad_(True)
    p = O.unflatten(flat)
    B = ids.shape[1]

    def pool(table, gi):
        present = gi >= 0
        idx = gi.t()[present.t()]
        offsets = torch.cat([torch.zeros(1, dtype=torch.long), present.t().sum(1).cumsum(0)[:-1]])
        return torch.nn.functional.embedding_bag(idx, table, offsets, mode="mean")  # an empty bag is zero

    wide = [pool(p[6 + g], ids[4 * g:4 * g + 4])[:, 0] for g in range(2)]
    e = torch.stack([pool(p[8 + g], ids[4 * g:4 * g + 4]) for g in range(3)])
    x = e.reshape(B, 24) if q11 else e.permute(1, 0, 2).reshape(B, 24)
    h = x
    for i in range(3):
        h = h @ p[2 * i] + p[2 * i + 1]
    z = wide[0] + wide[1] + h.sum(1)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(z, labels)
    (g,) = torch.autograd.grad(loss, [flat])
    return z.detach(), loss.detach(), g


@pytest.mark.parametrize("empty_group", [None, 0, 2])
@pytest.mark.parametrize("q11", [False, True])
@pytest.mark.parametrize("B", [1, 7, 130])
def test_oracle_matches_autograd(B, q11, empty_group):
    ids, labels, flat = _batch(B, seed=B + 10 * q11, empty_group=empty_group)
    ref = O.csql_reference(ids, labels, flat, q11)
    z, loss, g = _autograd(ids, labels, flat, q11)
    torch.testing.assert_close(ref["logits"], z, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["loss"], loss, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["grads"], g[:O.N_MLP], rtol=1e-10, atol=1e-14)
    for t in range(5):
        gt = g[O.OFFS[6 + t]:O.OFFS[7 + t]].view(O.SHAPES[6 + t])
        torch.testing.assert_close(ref["gsum"][t], gt, rtol=1e-10, atol=1e-14)
        # a row no present id names has a zero gradient and is not listed
        assert torch.equal(ref["touched"][t], ref["occ"][t] > 0)
        assert not gt[~ref["touched"][t]].any()


def test_offsets_dims_and_sizes():
    # feature_configs.py:137-205 -- offsets from the bucket counts [8, 7, 6, 6], [30, 7, 6, 30], [6, 2, 5, 100]
    assert [F.id_offsets(g) for g in ("group1", "group2", "group3")] == [[0, 8, 15, 21], [0, 30, 37, 43],
                                                                         [0, 6, 8, 13]]
    assert F.GROUP_DIMS == (27, 73, 113) == O.GROUP_ROWS
    assert [F.FEATURES[n][1] for n in ("education", "occupation", "native_country")] == [30, 30, 100]
    assert list(F.FEATURE_GROUPS.values()) == [["workclass", "hours_per_week", "capital_gain", "capital_loss"],
                                               ["education", "marital_status", "relationship", "occupation"],
                                               ["age", "sex", "race", "native_country"]]
    assert (M.N_PARAMS, M.N_MLP, M.N_UNIQ, M.N_GSUM) == (2376, 572, 313, 1804)
    assert M.N_PARAMS == 572 + 100 + 1704 and M.N_UNIQ == 27 + 73 + 27 + 73 + 113
    assert M.N_GSUM == 27 + 73 + (27 + 73 + 113) * 8
    assert M.UNIQ_OFF == (0, 27, 100, 127, 200) and M.GSUM_OFF == (0, 27, 100, 316, 900)


def _rows(variant, numeric_rows, string_rows):
    """ids [12, n] of hand-written rows: numeric_rows [(age, gain, loss, hours)], string_rows [{key: value}]."""
    num = np.array(numeric_rows, dtype=np.float32).T
    base = {k: "" for k in F.STRING_KEYS}
    strs = [[dict(base, **r)[k] for r in string_rows] for k in F.STRING_KEYS]
    return O.sqlflow_ids(num, strs, variant, F.FEATURES, list(F.FEATURE_GROUPS.values()), F.NUMERIC_KEYS,
                         F.STRING_KEYS)


KNOWN = {"workclass": "Private", "marital_status": "Divorced", "relationship": "Husband", "race": "Black",
         "sex": "Male", "education": "Bachelors", "occupation": "Sales", "native_country": "Peru"}


def test_keras_rule_rows():
    ids = _rows("keras", [(39.0, 0.0, 2000.0, 40.0), (0.0, 6000.0, 0.0, 0.0)],
                [KNOWN, dict(KNOWN, workclass="?", marital_status="Unknown", relationship="?", race="?", sex="X",
                             education="", occupation="", native_country="")])
    a, b = ids[:, 0].tolist(), ids[:, 1].tolist()
    # group1: workclass 0; hours 40 -> bucket 4 + 8; gain 0.0 dropped by ToSparse; loss 2000 -> bucket 1 + 21
    assert a[0:4] == [0, 12, -1, 22]
    # an unknown workclass is len(vocabulary) + 0 = 8: hours_per_week's bucket 0 (Q22); 0.0 hours dropped
    assert b[0:4] == [8, -1, 15 + 1, -1]
    # group2: Divorced 1 + 30, Husband 2 + 37; unknown marital -> 7 + 30 = 37 (relationship's 0), unknown
    # relationship -> 6 + 37 = 43 (occupation's bucket 0); "" hashes dropped
    assert a[5:7] == [31, 39] and b[4:8] == [-1, 37, 43, -1]
    # group3: age 39 -> bucket 2; Male 1 + 6; Black 4 + 8; age 0.0 dropped; unknown sex -> 2 + 6 = 8 (race's 0),
    # unknown race -> 5 + 8 = 13 (native_country's bucket 0)
    assert a[8:11] == [2, 7, 12] and b[8:12] == [-1, 8, 13, -1]
    assert 0 <= a[4] < 30 and 43 <= a[7] < 73 and 13 <= a[11] < 113


def test_fc_rule_rows():
    ids = _rows("fc", [(39.0, 0.0, 2000.0, 40.0), (0.0, 6000.0, 0.0, 0.0)],
                [KNOWN, dict(KNOWN, workclass="?", marital_status="Unknown", relationship="?", race="?", sex="X",
                             education="", occupation="", native_country="")])
    a, b = ids[:, 0].tolist(), ids[:, 1].tolist()
    # bucketized columns are dense: gain 0.0 keeps bucket 0 (+15); hours 0.0 bucket 0 (+8), age 0.0 bucket 1
    assert a[0:4] == [0, 12, 15, 22]
    # an unknown workclass is -1 + 0 = -1: pruned (Q23, Q24)
    assert b[0:4] == [-1, 8, 16, 21]
    # unknown marital -> -1 + 30 = 29 (education's last bucket), unknown relationship -> -1 + 37 = 36
    # (marital_status's last id); "" hashes dropped (Q21)
    assert b[4:8] == [-1, 29, 36, -1]
    # unknown sex -> -1 + 6 = 5 (age's last bucket), unknown race -> -1 + 8 = 7 (sex's last id)
    assert b[8:12] == [1, 5, 7, -1]
    # "" in a vocabulary column is dropped, not looked up (Q21)
    assert _rows("fc", [(39.0, 1.0, 1.0, 1.0)], [dict(KNOWN, race="")])[10, 0] == -1
    assert _rows("keras", [(39.0, 1.0, 1.0, 1.0)], [dict(KNOWN, race="")])[10, 0] == -1


def test_id_mutations_change_ids():
    rows = [(39.0, 0.0, 2000.0, 40.0), (0.0, 6000.0, 0.0, 0.0)]
    strs = [KNOWN, dict(KNOWN, workclass="?", marital_status="", sex="X")]
    for v in F.VARIANTS:
        base = _rows(v, rows, strs)
        num = np.array(rows, dtype=np.float32).T
        raw = [[r.get(k, "") for r in [dict({kk: "" for kk in F.STRING_KEYS}, **s) for s in strs]]
               for k in F.STRING_KEYS]
        for m in O.ID_MUTATIONS:
            mut = O.sqlflow_ids(num, raw, v, F.FEATURES, list(F.FEATURE_GROUPS.values()), F.NUMERIC_KEYS,
                                F.STRING_KEYS, mutate=m)
            assert not np.array_equal(mut, base), (v, m)


def test_transform_specs():
    for v in F.VARIANTS:
        gs = F.groups(v)
        assert [g["offset"] for g in gs] == [0, 8, 15, 21, 0, 30, 37, 43, 0, 6, 8, 13]
        for spec, name in zip(gs, sum(F.FEATURE_GROUPS.values(), [])):
            op = F.FEATURES[name][0]
            assert spec["absent"] == (op != "bucketize" or v == "keras"), (v, name)
            if op == "lookup":
                assert spec["num_oov_tokens"] == (1 if v == "keras" else 0)
    with pytest.raises(ValueError, match="variant"):
        F.groups("tf")


def test_models_and_names():
    assert {m: M.model_of(m) for m in M.MODELS} == {
        "wide_deep_functional_keras": ("keras", True), "wide_deep_functional_tensor_interface_keras": ("keras", False),
        "wide_deep_subclass_keras": ("keras", False), "wide_deep_functional_fc": ("fc", True),
        "wide_deep_functional_tensor_interface_fc": ("fc", False)}
    assert M.param_names("keras")[6:] == ["sparse_embedding/embeddings:0", "sparse_embedding_1/embeddings:0",
                                          "sparse_embedding_2/embeddings:0", "sparse_embedding_3/embeddings:0",
                                          "sparse_embedding_4/embeddings:0"]
    fc = M.param_names("fc")[6:]
    assert fc[0] == ("dense_features/capital_gain_bucketized_C_capital_loss_bucketized_C_hours_per_week_bucketized"
                     "_C_workclass_embedding/embedding_weights:0")
    assert fc[4].startswith("dense_features_4/age_bucketized_C_native_country_C_race_C_sex_embedding/")
    # Q26: one DenseFeatures sorts its three deep columns by name, group 3 first
    assert sorted(M.FC_COLUMNS) == [M.FC_COLUMNS[2], M.FC_COLUMNS[0], M.FC_COLUMNS[1]]
    with pytest.raises(ValueError, match="unknown model"):
        M.model_of("census_model_sqlflow")


def test_zoo_schedule_matches_its_literal():
    def _schedule(model_version):  # wide_deep_functional_keras.py:280-286
        if model_version < 5000:
            return 0.0003
        elif model_version < 12000:
            return 0.0002
        else:
            return 0.0001

    sched = M.callbacks()[0].schedule
    for v in [0, 1, 4998, 4999, 5000, 5001, 11998, 11999, 12000, 12001, 10 ** 6]:
        assert sched(v) == float(np.float32(_schedule(v))), v
    assert M.optimizer()[2] == 1e-3


@pytest.mark.parametrize("q11", [False, True])
def test_mutations_move_their_outputs(q11):
    ids, labels, flat = _batch(600, seed=21 + q11, empty_group=1)
    ref = O.csql_reference(ids, labels, flat, q11)
    assert not O.caught_by(ref, ref)
    muts = O.mutations(ref, (ids, labels, flat, q11))
    assert set(muts) == set(O.TOWER_MUTATIONS)
    for name, mut in muts.items():
        assert O.caught_by(mut, ref), name
