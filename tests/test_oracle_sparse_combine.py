"""oracle/sparse_oracle.py against the reference's literal vectors (layer_test.py:188-215 forward, :294-370
BET gradients) and at its edges: all-empty rows, all-negative rows, nnz = 0.  CPU only."""
import numpy as np
import pytest

from oracle import sparse_oracle as so

# layer_test.py:191-193: a [4, 6] input, rows 0: [1], 1: [1, 3], 2: [2], 3: [0, 2, 6]
ROWS = [0, 1, 1, 2, 3, 3, 3]
VALS = [1, 1, 3, 2, 0, 2, 6]
DIM = 8
FWD = {
    "sum": [1.0, 4.0, 2.0, 8.0],
    "mean": [1.0, 2.0, 2.0, 8.0 / 3.0],
    "sqrtn": [1.0, 4.0 / np.sqrt(2.0), 2.0, 8.0 / np.sqrt(3.0)],
}
GRADS = {  # layer_test.py:307-319, for the unique ids (1, 3, 2, 0, 6)
    "sum": [0 + 1, 1, 2 + 3, 3, 3],
    "mean": [1 / 2.0, 1 / 2.0, 2 + 3 / 3.0, 3 / 3.0, 3 / 3.0],
    "sqrtn": [1 / np.sqrt(2.0), 1 / np.sqrt(2.0), 2 + 3 / np.sqrt(3.0), 3 / np.sqrt(3.0), 3 / np.sqrt(3.0)],
}


def _fake(ids):  # the reference test's lookup: row of id i is [i] * dim
    return np.repeat(np.asarray(ids, dtype=np.float64)[:, None], DIM, axis=1)


def _mult():  # layer_test.py:303-305: output row i multiplied by i
    return np.repeat(np.arange(4, dtype=np.float64)[:, None], DIM, axis=1)


@pytest.mark.parametrize("combiner", ["sum", "mean", "sqrtn"])
def test_layer_test_py_forward(combiner):
    out, uniq, _ = so.lookup(ROWS, VALS, 4, _fake, combiner)
    np.testing.assert_array_equal(uniq, [1, 3, 2, 0, 6])
    np.testing.assert_allclose(out, np.repeat(np.array(FWD[combiner])[:, None], DIM, axis=1), rtol=1e-15)


@pytest.mark.parametrize("combiner", ["sum", "mean", "sqrtn"])
def test_layer_test_py_bet_gradients(combiner):
    # two calls record two entries with the same ids and gradients
    for _ in range(2):
        _, uniq, _ = so.lookup(ROWS, VALS, 4, _fake, combiner)
        g = so.grad_bet(ROWS, VALS, 4, len(uniq), _mult(), combiner)
        np.testing.assert_array_equal(uniq, [1, 3, 2, 0, 6])
        np.testing.assert_allclose(g[:, 0], GRADS[combiner], rtol=1e-15)
        assert (g == g[:, :1]).all()


@pytest.mark.parametrize("combiner", ["sum", "mean", "sqrtn"])
def test_all_empty_rows(combiner):
    out, uniq, bet = so.lookup([], [], 5, _fake, combiner)
    np.testing.assert_array_equal(uniq, [0])
    assert bet.shape == (1, DIM) and (out == 0).all() and out.shape == (5, DIM)
    g = so.grad_bet([], [], 5, 1, np.ones((5, DIM)), combiner)
    assert (g == 0).all()


@pytest.mark.parametrize("combiner", ["sum", "mean", "sqrtn"])
def test_all_negative_rows(combiner):
    # row 1 holds only negative ids: it is empty after pruning, gets id 0 and a zero output row
    rows, vals = [0, 1, 1, 2], [4, -1, -7, 4]
    out, uniq, _ = so.lookup(rows, vals, 3, _fake, combiner)
    np.testing.assert_array_equal(uniq, [4, 0])
    assert (out[1] == 0).all() and (out[0] == 4).all() and (out[2] == 4).all()
    g = so.grad_bet(rows, vals, 3, 2, np.ones((3, DIM)), combiner)
    np.testing.assert_array_equal(g[:, 0], [2.0, 0.0])  # the fill id gets nothing unless it also occurs for real


def test_fill_id_zero_that_also_occurs():
    rows, vals = [1, 1], [0, 5]
    _, uniq, _ = so.lookup(rows, vals, 2, _fake, "sum")
    np.testing.assert_array_equal(uniq, [0, 5])  # row 0's fill id first, then row 1's real 0 maps onto it
    g = so.grad_bet(rows, vals, 2, 2, np.ones((2, DIM)), "sum")
    np.testing.assert_array_equal(g[:, 0], [1.0, 1.0])


def test_bound_covers_float32_sums():
    rng = np.random.default_rng(3)
    B, dim = 64, 5
    lens = rng.integers(0, 40, B)
    rows = np.repeat(np.arange(B), lens)
    vals = rng.integers(-3, 50, rows.size)
    table = rng.standard_normal((50, dim)).astype(np.float32)
    for combiner in ("sum", "mean", "sqrtn"):
        out, uniq, bet = so.lookup(rows, vals, B, lambda u: table[u], combiner)
        frows, fids, cnt = so.fill(rows, vals, B)
        _, inv = so.unique_first(fids)
        got = np.zeros((B, dim), dtype=np.float32)
        for j in range(len(fids)):  # float32 sum in entry order, then the combiner's one operation
            got[frows[j]] += table[fids[j]]
        c = np.maximum(cnt, 1).astype(np.float32)[:, None]
        got = {"sum": got, "mean": got / c, "sqrtn": got / np.sqrt(c)}[combiner]
        got[cnt == 0] = 0
        bd = so.bound(rows, vals, B, np.abs(bet), combiner)
        assert (np.abs(got - out) <= bd).all()
