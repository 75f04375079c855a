"""Float64 restatement of the reference's pooled lookup of a sparse input without weights
(safe_embedding_lookup_sparse, embedding_delegate.py:108-230; TF's SparseEmbedding layer computes the same):
prune ids < 0, give each empty row the id 0 (sparse_fill_empty_rows), tf.unique in first-occurrence order,
sparse_segment_{sum,mean,sqrt_n}, then zero the rows that were empty.

Test infrastructure only: the product never imports it."""
import numpy as np


def fill(rows, vals, batch):
    """Row-major COO (rows, vals) of a [batch, L] input -> (filled rows, filled ids, kept count per row)."""
    rows = np.asarray(rows, dtype=np.int64).reshape(-1)
    vals = np.asarray(vals, dtype=np.int64).reshape(-1)
    keep = vals >= 0
    rows, vals = rows[keep], vals[keep]
    cnt = np.bincount(rows, minlength=batch).astype(np.int64)
    empty = np.nonzero(cnt == 0)[0]
    rows = np.concatenate([rows, empty])
    vals = np.concatenate([vals, np.zeros_like(empty)])
    order = np.argsort(rows, kind="stable")
    return rows[order], vals[order], cnt


def unique_first(ids):
    """tf.unique: distinct ids in first-occurrence order and the inverse."""
    _, first, inv = np.unique(ids, return_index=True, return_inverse=True)
    rank = np.empty(len(first), dtype=np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(len(first))
    return ids[np.sort(first)], rank[inv.reshape(-1)]


def _scale(cnt, combiner):
    c = np.maximum(cnt, 1).astype(np.float64)
    return {"sum": np.ones_like(c), "mean": 1.0 / c, "sqrtn": 1.0 / np.sqrt(c)}[combiner] * (cnt > 0)


def lookup(rows, vals, batch, bet_of, combiner):
    """Returns (out [batch, dim] float64, unique ids, BET float64 [U, dim]); bet_of(unique_ids) -> rows."""
    frows, fids, cnt = fill(rows, vals, batch)
    uniq, inv = unique_first(fids)
    bet = np.asarray(bet_of(uniq), dtype=np.float64)
    out = np.zeros((batch, bet.shape[1]), dtype=np.float64)
    np.add.at(out, frows, bet[inv])
    return out * _scale(cnt, combiner)[:, None], uniq, bet


def grad_bet(rows, vals, batch, n_unique, G, combiner):
    """d(sum(out * G)) / d BET, [U, dim] float64."""
    frows, fids, cnt = fill(rows, vals, batch)
    _, inv = unique_first(fids)
    G = np.asarray(G, dtype=np.float64)
    g = np.zeros((n_unique, G.shape[1]), dtype=np.float64)
    np.add.at(g, inv, G[frows] * _scale(cnt, combiner)[frows, None])
    return g


def bound(rows, vals, batch, absrows, combiner):
    """Per-row rounding bound of the fp32 combine, in the tower oracles' form: a sum of m addends in any order is
    within (m - 1) 2^-24 sum|x| of the exact one, the scale adds one rounding of the result (and sqrtn one of the
    square root).  absrows = |BET| rows per filled entry's id ([U, dim] float64 of |bet|)."""
    frows, fids, cnt = fill(rows, vals, batch)
    _, inv = unique_first(fids)
    mag = np.zeros((batch, absrows.shape[1]), dtype=np.float64)
    np.add.at(mag, frows, absrows[inv])
    m = np.maximum(cnt, 1).astype(np.float64)[:, None]
    u = 2.0 ** -24
    return ((m - 1) * u + 3 * u) * mag * _scale(cnt, combiner)[:, None] + 2.0 ** -149


def grad_bound(rows, vals, batch, n_unique, absG, combiner):
    """Bound of the fp32 backward: each addend is G / d (one rounding, and one of the square root for sqrtn),
    summed by multiplicity per unique id; flushed subnormal addends lose at most 2^-126 each."""
    frows, fids, cnt = fill(rows, vals, batch)
    _, inv = unique_first(fids)
    live = cnt[frows] > 0
    mag = np.zeros((n_unique, absG.shape[1]), dtype=np.float64)
    np.add.at(mag, inv[live], absG[frows[live]] * _scale(cnt, combiner)[frows[live], None])
    mult = np.bincount(inv[live], minlength=n_unique).astype(np.float64)[:, None]
    u = 2.0 ** -24
    return (np.maximum(mult - 1, 0) * u + 3 * u) * mag + (mult + 1) * 2.0 ** -126
