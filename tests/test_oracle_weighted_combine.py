"""tests/weighted_oracle.py (the float64 weighted lookup) against the reference's literal vectors
(feature_column_test.py:75-111 forward, :172-270 gradients), against torch's own float64 F.embedding_bag with
per_sample_weights, and at the edges where the reference raises (DESIGN.md §4, Q14).  CPU only."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sparse_oracle as so
from tests import weighted_oracle as wo

COMBINERS = ["sum", "mean", "sqrtn"]


def _one_hot(dim):  # feature_column_test.py:30-40: the row of id i is one-hot at i % dim
    return lambda ids: (np.arange(dim)[None, :] == (np.asarray(ids)[:, None] % dim)).astype(np.float64)


def _dense_coo(ids):
    ids = np.asarray(ids)
    rows = np.repeat(np.arange(ids.shape[0]), ids.shape[1])
    return rows, ids.reshape(-1)


def test_feature_column_weighted_output():
    rows, vals = _dense_coo([[2, 6, 5], [3, 1, 1]])
    # the weights are cast to float32 before they multiply (embedding_delegate.py:141-142)
    w = np.array([0.33, 5.0, 1.024, 2.048, 0.5, 1.0], dtype=np.float32).astype(np.float64)
    out, uniq, _ = wo.lookup_weighted(rows, vals, w, 2, _one_hot(8), "sum")
    want = np.array([[0.0, 0.0, 0.33, 0.0, 0.0, 1.024, 5.0, 0.0],
                     [0.0, 1.5, 0.0, 2.048, 0.0, 0.0, 0.0, 0.0]], dtype=np.float32)
    np.testing.assert_array_equal(uniq, [2, 6, 5, 3, 1])
    assert np.array_equal(out.astype(np.float32), want)


# feature_column_test.py:172-230: per-occurrence gradients of the output's sum, in the order of the flat ids
GRAD_IDS = [[1, 2], [10, 10], [6, 3], [10, 2]]
GRAD_W = [0.3, 0.6, 0.1, 0.2, 0.8, 0.1, 0.9, 0.6]
GRAD_OCC = {
    "sum": [0.3, 0.6, 0.1, 0.2, 0.8, 0.1, 0.9, 0.6],
    "mean": [0.3 / 0.9, 0.6 / 0.9, 0.1 / 0.3, 0.2 / 0.3, 0.8 / 0.9, 0.1 / 0.9, 0.9 / 1.5, 0.6 / 1.5],
    "sqrtn": [w / np.sqrt(a * a + b * b)
              for (a, b) in [(0.3, 0.6), (0.1, 0.2), (0.8, 0.1), (0.9, 0.6)] for w in (a, b)],
}


@pytest.mark.parametrize("combiner", COMBINERS)
def test_feature_column_weighted_gradients(combiner):
    """The reference's BET gradient is per occurrence (an IndexedSlices over the flat ids); ours is per unique id
    (layers/embedding.py), so the occurrences of each id are summed: tf.unique's idx maps them."""
    rows, vals = _dense_coo(GRAD_IDS)
    fill_by_id = lambda ids: np.repeat(np.asarray(ids, dtype=np.float64)[:, None], 8, axis=1)
    _, uniq, _ = wo.lookup_weighted(rows, vals, GRAD_W, 4, fill_by_id, combiner)
    np.testing.assert_array_equal(uniq, [1, 2, 10, 6, 3])
    _, idx = so.unique_first(vals)
    want = np.zeros(5)
    np.add.at(want, idx, GRAD_OCC[combiner])
    g = wo.grad_bet_weighted(rows, vals, GRAD_W, 4, 5, np.ones((4, 8)), combiner)
    np.testing.assert_allclose(g, np.repeat(want[:, None], 8, axis=1), rtol=1e-14)


@pytest.mark.parametrize("combiner", COMBINERS)
def test_unit_weights_give_the_unweighted_lookup_exactly(combiner):
    rng = np.random.default_rng(11)
    B, dim = 50, 6
    lens = rng.integers(0, 9, B)
    rows = np.repeat(np.arange(B), lens)
    vals = rng.integers(-3, 40, rows.size)
    table = rng.standard_normal((40, dim))
    out, uniq, bet = so.lookup(rows, vals, B, lambda u: table[u], combiner)
    wout, wuniq, wbet = wo.lookup_weighted(rows, vals, np.ones(rows.size), B, lambda u: table[u], combiner)
    assert np.array_equal(out, wout) and np.array_equal(uniq, wuniq) and np.array_equal(bet, wbet)
    G = rng.standard_normal((B, dim))
    g = so.grad_bet(rows, vals, B, len(uniq), G, combiner)
    assert np.array_equal(g, wo.grad_bet_weighted(rows, vals, np.ones(rows.size), B, len(uniq), G, combiner))


def _bags(rng, B, N, pad):
    lens = rng.poisson(4, B)
    lens[rng.random(B) < 0.1] = 0
    ids = rng.integers(0, N, int(lens.sum()))
    if pad is not None:
        ids[rng.random(ids.size) < 0.2] = pad
    offsets = np.concatenate([[0], np.cumsum(lens)[:-1]])
    return lens, ids, offsets


@pytest.mark.parametrize("pad", [None, 3])
def test_against_torch_embedding_bag_float64(pad):
    rng = np.random.default_rng(7)
    B, N, dim = 40, 12, 5
    lens, ids, offsets = _bags(rng, B, N, pad)
    w = rng.uniform(-1.0, 2.0, ids.size)
    table = torch.tensor(rng.standard_normal((N, dim)), dtype=torch.float64, requires_grad=True)
    psw = torch.tensor(w, requires_grad=True)
    out = F.embedding_bag(torch.tensor(ids), table, torch.tensor(offsets), mode="sum", per_sample_weights=psw,
                          padding_idx=pad)
    G = rng.standard_normal((B, dim))
    out.backward(torch.tensor(G))

    rows = np.repeat(np.arange(B), lens)
    vals = ids if pad is None else np.where(ids == pad, -1, ids)  # padding entries are dropped, as torch drops them
    tab = table.detach().numpy()
    got, uniq, bet = wo.lookup_weighted(rows, vals, w, B, lambda u: tab[u], "sum")
    np.testing.assert_allclose(got, out.detach().numpy(), rtol=1e-12, atol=1e-14)
    gbet = wo.grad_bet_weighted(rows, vals, w, B, len(uniq), G, "sum")
    dense = np.zeros((N, dim))
    np.add.at(dense, uniq, gbet)
    np.testing.assert_allclose(dense, table.grad.numpy(), rtol=1e-12, atol=1e-14)
    gw = wo.grad_weights(rows, vals, B, bet, G)
    np.testing.assert_allclose(gw, psw.grad.numpy(), rtol=1e-12, atol=1e-14)
    if pad is not None:
        assert (gw[ids == pad] == 0).all() and (psw.grad.numpy()[ids == pad] == 0).all()


def test_pruned_weights_empty_rows_and_signs():
    # row 0: a negative id whose weight goes with it; row 1: only negative ids (empty: 0, fill id 0 gets nothing);
    # row 2: a negative weight is kept under mean (never pruned by sign)
    rows = [0, 0, 1, 2, 2]
    vals = [4, -1, -2, 5, 6]
    w = [2.0, 100.0, 7.0, -1.0, 3.0]
    fake = lambda ids: np.repeat(np.asarray(ids, dtype=np.float64)[:, None], 2, axis=1)
    out, uniq, bet = wo.lookup_weighted(rows, vals, w, 3, fake, "mean")
    np.testing.assert_array_equal(uniq, [4, 0, 5, 6])
    np.testing.assert_allclose(out[:, 0], [4.0, 0.0, (-5.0 + 18.0) / 2.0], rtol=1e-15)
    g = wo.grad_bet_weighted(rows, vals, w, 3, 4, np.ones((3, 2)), "mean")
    np.testing.assert_allclose(g[:, 0], [1.0, 0.0, -0.5, 1.5], rtol=1e-15)
    gw = wo.grad_weights(rows, vals, 3, bet, np.ones((3, 2)))
    np.testing.assert_array_equal(gw, [8.0, 0.0, 0.0, 10.0, 12.0])


def test_zero_weight_sum_divides_by_zero():
    rows, vals = [0, 0, 1], [1, 2, 3]
    fake = lambda ids: np.repeat(np.asarray(ids, dtype=np.float64)[:, None], 2, axis=1)
    out, _, _ = wo.lookup_weighted(rows, vals, [1.0, -1.0, 0.0], 2, fake, "mean")
    assert np.isinf(out[0]).all() and np.isnan(out[1]).all()  # -1 / 0 and 0 / 0
    out, _, _ = wo.lookup_weighted(rows, vals, [1.0, -1.0, 0.0], 2, fake, "sqrtn")
    assert np.isfinite(out[0]).all() and np.isnan(out[1]).all()


def test_bounds_cover_float32_arithmetic():
    rng = np.random.default_rng(3)
    B, dim = 64, 5
    lens = rng.integers(0, 40, B)
    rows = np.repeat(np.arange(B), lens)
    vals = rng.integers(-3, 50, rows.size)
    w = rng.uniform(0.1, 2.0, rows.size).astype(np.float32)
    table = rng.standard_normal((50, dim)).astype(np.float32)
    G = rng.standard_normal((B, dim)).astype(np.float32)
    frows, src, cnt = wo.fill_src(rows, vals, B)
    _, fids, _ = so.fill(rows, vals, B)
    _, inv = so.unique_first(fids)
    for combiner in COMBINERS:
        out, uniq, bet = wo.lookup_weighted(rows, vals, w, B, lambda u: table[u], combiner)
        acc = np.zeros((B, dim), dtype=np.float32)
        den = np.zeros(B, dtype=np.float32)
        for j in range(len(fids)):  # float32 in entry order, then the combiner's one operation
            if src[j] >= 0:
                acc[frows[j]] += w[src[j]] * table[fids[j]]
                den[frows[j]] += w[src[j]] if combiner == "mean" else w[src[j]] * w[src[j]]
        d = {"sum": np.ones(B, np.float32), "mean": den, "sqrtn": np.sqrt(den)}[combiner]
        got = np.where(cnt[:, None] > 0, acc / np.where(cnt > 0, d, 1)[:, None], 0)
        assert (np.abs(got - out) <= wo.bound_weighted(rows, vals, w, B, np.abs(bet), combiner)).all()
        gw = np.zeros((len(uniq), dim), dtype=np.float32)
        for j in range(len(fids)):
            if src[j] >= 0:
                gw[inv[j]] += G[frows[j]] * w[src[j]] / d[frows[j]]
        want = wo.grad_bet_weighted(rows, vals, w, B, len(uniq), G, combiner)
        gb = wo.grad_bound_weighted(rows, vals, w, B, len(uniq), np.abs(G.astype(np.float64)), combiner)
        assert (np.abs(gw - want) <= gb).all()
    _, uniq, bet = wo.lookup_weighted(rows, vals, w, B, lambda u: table[u], "sum")
    g32 = np.zeros(rows.size, dtype=np.float32)
    for j in range(len(fids)):
        if src[j] >= 0:
            g32[src[j]] = np.dot(table[fids[j]], G[frows[j]])
    want = wo.grad_weights(rows, vals, B, bet, G)
    assert (np.abs(g32 - want) <= wo.grad_weights_bound(rows, vals, B, np.abs(bet), np.abs(G.astype(np.float64)))).all()
