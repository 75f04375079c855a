"""The float64 feature-column DNN oracle (oracle/fc_dnn_oracle.py) on the CPU: against torch float64 autograd of
the same model for both layouts and both reductions, with empty strings and clipped probabilities; the layouts'
column order, widths, parameter counts and feature transform specs; and every mutation moving the outputs it
should."""
import numpy as np
import pytest
import torch

from elasticdl_b200.workloads import fc_dnn as M
from oracle import fc_dnn_oracle as O
from oracle import feature_oracle as FO


def _batch(L, B, seed, b3=None, empty_fraction=0.2):
    g = torch.Generator().manual_seed(seed)
    T = len(L.tables)
    numeric = torch.randn((len(L.numeric_keys), B), generator=g)
    ids = torch.zeros((T + len(L.buckets), B), dtype=torch.int32)
    for i, (_, bins) in enumerate(L.buckets):
        ids[T + i] = torch.randint(0, len(bins) + 1, (B,), generator=g, dtype=torch.int32)
    empty = torch.rand((T, B), generator=g) < empty_fraction
    inv, n_unique, rows = [], [], []
    for k, (_, r, d) in enumerate(L.tables):
        bucket = torch.randint(0, r, (B,), generator=g)
        bucket[empty[k]] = 0  # the fill id
        u, iv = torch.unique(bucket, return_inverse=True)
        inv.append(iv.to(torch.int32))
        n_unique.append(u.numel())
        rows.append((torch.rand((u.numel(), d), generator=g, dtype=torch.float64) * 2 - 1) * 0.5)
    labels = (torch.rand(B, generator=g) < 0.3).to(torch.float64)
    flat = torch.cat([(torch.rand(int(np.prod(s)), generator=g, dtype=torch.float64) * 2 - 1) * 0.4
                      for _, s in L.mlp])
    if b3 is not None:
        flat[-1] = b3
    return numeric.double(), ids, empty, torch.stack(inv), n_unique, rows, labels, flat


def _autograd(spec, numeric, ids, empty, inv, n_unique, rows, labels, flat):
    rows = [r.clone().requires_grad_(True) for r in rows]
    flat = flat.clone().requires_grad_(True)
    W1, b1, W2, b2, W3, b3 = O.unflatten(spec["F"], flat)
    x = O.dense_features(spec, numeric, ids, empty, inv, rows)
    h = torch.relu(x @ W1 + b1)
    h = torch.relu(h @ W2 + b2)
    z = (h @ W3 + b3)[:, 0]
    loss = M.keras_bce(labels, torch.sigmoid(z), spec["loss_mean"])
    gs = torch.autograd.grad(loss, [flat] + rows)
    return z.detach(), loss.detach(), gs[0], list(gs[1:])


@pytest.mark.parametrize("b3", [None, 20.0, -20.0])
@pytest.mark.parametrize("loss_mean", [False, True])
@pytest.mark.parametrize("model", ["census_dnn_model", "heart_functional_api"])
@pytest.mark.parametrize("B", [1, 7, 130])
def test_oracle_matches_autograd(B, model, loss_mean, b3):
    L = M.layout_of(model)
    spec = dict(L.spec(), loss_mean=loss_mean)
    inputs = _batch(L, B, seed=B + 3 * loss_mean, b3=b3)
    ref = O.fc_dnn_reference(spec, *inputs)
    z, loss, grads, gsum = _autograd(spec, *inputs)
    torch.testing.assert_close(ref["logits"], z, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["loss"], loss, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["grads"], grads, rtol=1e-10, atol=1e-14)
    for a, b in zip(ref["gsum"], gsum):
        torch.testing.assert_close(a, b, rtol=1e-10, atol=1e-14)
    if b3 is not None:  # every probability is clipped: no gradient at all (Q19)
        assert torch.count_nonzero(ref["grads"]) == 0
        assert all(torch.count_nonzero(g) == 0 for g in ref["gsum"])


def test_layouts():
    C, Hh = M.CENSUS_DNN, M.HEART
    assert (C.F, C.n_mlp, Hh.F, Hh.n_mlp) == (4 + 8 * 16, 2417, 11 + 6 + 8, 705)
    # Q17: DenseFeatures sorts its columns by name
    assert [c for c, _, _ in C.columns] == [
        "age", "capital-gain", "capital-loss", "education_embedding", "hours-per-week", "marital-status_embedding",
        "native-country_embedding", "occupation_embedding", "race_embedding", "relationship_embedding",
        "sex_embedding", "workclass_embedding"]
    assert [c for c, _, _ in Hh.columns] == ["age_bucketized", "ca", "chol", "oldpeak", "slope", "thal_embedding",
                                             "thalach", "trestbps"]
    assert [o for _, _, _, o in Hh.blocks] == [0, 11, 12, 13, 14, 15, 23, 24]
    assert C.table_names[1] == "dense_features/education_embedding/embedding_weights:0"
    assert [(r, d) for _, r, d in C.tables] == [(64, 16)] * 8 and [(r, d) for _, r, d in Hh.tables] == [(100, 8)]
    assert not C.loss_mean and Hh.loss_mean
    assert [n for n, _ in C.mlp] == ["dense/kernel:0", "dense/bias:0", "dense_1/kernel:0", "dense_1/bias:0",
                                     "dense_2/kernel:0", "dense_2/bias:0"]
    with pytest.raises(ValueError, match="unknown model"):
        M.layout_of("census_model_sqlflow")


def test_transform_specs_hash_like_the_reference():
    """Each table is categorical_column_with_hash_bucket over its own string column: Fingerprint64 mod the bucket
    count (feature_oracle restates FarmHash); heart's age is bucketized left-closed at its ten boundaries."""
    for L in (M.CENSUS_DNN, M.HEART):
        gs = L.groups()
        for k, (key, rows, _) in enumerate(L.tables):
            assert gs[k] == {"kind": "hash", "column": L.string_keys.index(key), "num_bins": rows}
    assert M.HEART.groups()[1] == {"kind": "discretize", "column": 0, "bins": [float(b) for b in M.HEART_AGE_BOUNDARIES]}
    assert FO.hashing(["A", "B", "C", "D", "E"], 3).tolist() == [1, 0, 1, 1, 2]  # hashing.py:35-39
    assert FO.discretize(np.array([17.0, 18.0, 64.9, 65.0]), M.HEART_AGE_BOUNDARIES).tolist() == [0, 1, 9, 10]


@pytest.mark.parametrize("model", ["census_dnn_model", "heart_functional_api"])
def test_mutations_move_their_outputs(model):
    L = M.layout_of(model)
    spec = L.spec()
    inputs = _batch(L, 300, seed=11)
    ref = O.fc_dnn_reference(spec, *inputs)
    assert not O.caught_by(ref, ref)
    muts = O.mutations(spec, inputs)
    assert set(muts) == set(O.MUTATIONS)
    for name, mut in muts.items():
        caught = O.caught_by(mut, ref)
        if name == "clip_grad_kept":  # no probability of this batch is clipped: checked below
            continue
        assert caught, name
        if name in ("no_relu_mask", "swap_reduction", "tile_missing"):
            assert "grads" in caught, (name, caught)
        if name in ("unsorted", "empty_not_zeroed"):
            assert "logits" in caught, (name, caught)
    clipped = _batch(L, 300, seed=12, b3=20.0)
    ref = O.fc_dnn_reference(spec, *clipped)
    assert "grads" in O.caught_by(O.mutations(spec, clipped, ("clip_grad_kept",))["clip_grad_kept"], ref)
