"""Float64 restatement of the reference's weighted pooled lookup of a sparse input (safe_embedding_lookup_sparse
with sparse_weights, embedding_delegate.py:134-194; nn.EmbeddingBag's per_sample_weights), on top of
oracle/sparse_oracle.py's fill and unique_first, with the rounding bounds of the fp32 kernels.

A weight is pruned with its id; the fill entry of an empty row has weight 0 and the row gives 0; weights are never
pruned by sign (DESIGN.md §4, Q14).  weights are in the input's entry order, as rows and vals.

Test infrastructure only: the product never imports it."""
import numpy as np

from oracle.sparse_oracle import fill, unique_first


def fill_src(rows, vals, batch):
    """fill() of the input entry indices: (filled rows, input entry of each filled entry (-1 for the fill of an empty
    row), kept count per row), in the order fill() gives."""
    vals = np.asarray(vals, dtype=np.int64).reshape(-1)
    tag = np.where(vals >= 0, np.arange(vals.size) + 1, -1)
    frows, fsrc, cnt = fill(rows, tag, batch)
    return frows, fsrc - 1, cnt


def _weighted_fill(rows, vals, weights, batch):
    frows, src, cnt = fill_src(rows, vals, batch)
    vals = np.asarray(vals, dtype=np.int64).reshape(-1)
    weights = np.asarray(weights, dtype=np.float64).reshape(-1)
    live = src >= 0
    fids = np.where(live, vals[np.maximum(src, 0)], 0)
    w = np.where(live, weights[np.maximum(src, 0)] if weights.size else 0.0, 0.0)
    return frows, src, cnt, fids, w


def weighted_scale(rows, vals, weights, batch, combiner):
    """1 / the row's divisor (1 for sum, 1 / sum w for mean, 1 / sqrt(sum w^2) for sqrtn), 0 for an empty row; a
    non-empty row whose divisor is 0 gets inf, so its output is inf or NaN as IEEE division gives."""
    frows, _, cnt, _, w = _weighted_fill(rows, vals, weights, batch)
    den = {"sum": np.ones(batch),
           "mean": np.bincount(frows, weights=w, minlength=batch),
           "sqrtn": np.sqrt(np.bincount(frows, weights=w * w, minlength=batch))}[combiner]
    with np.errstate(divide="ignore"):
        s = 1.0 / den
    return np.where(cnt > 0, s, 0.0)


def lookup_weighted(rows, vals, weights, batch, bet_of, combiner):
    """Returns (out [batch, dim] float64, unique ids, BET float64 [U, dim]); unit weights give lookup()'s values
    exactly."""
    frows, _, cnt, fids, w = _weighted_fill(rows, vals, weights, batch)
    uniq, inv = unique_first(fids)
    bet = np.asarray(bet_of(uniq), dtype=np.float64)
    out = np.zeros((batch, bet.shape[1]), dtype=np.float64)
    np.add.at(out, frows, w[:, None] * bet[inv])
    with np.errstate(invalid="ignore"):
        out = out * weighted_scale(rows, vals, weights, batch, combiner)[:, None]
    out[cnt == 0] = 0.0
    return out, uniq, bet


def grad_bet_weighted(rows, vals, weights, batch, n_unique, G, combiner):
    """d(sum(out * G)) / d BET, [U, dim] float64."""
    frows, src, _, fids, w = _weighted_fill(rows, vals, weights, batch)
    _, inv = unique_first(fids)
    G = np.asarray(G, dtype=np.float64)
    s = weighted_scale(rows, vals, weights, batch, combiner)
    live = src >= 0
    g = np.zeros((n_unique, G.shape[1]), dtype=np.float64)
    np.add.at(g, inv[live], G[frows[live]] * (w[live] * s[frows[live]])[:, None])
    return g


def grad_weights(rows, vals, batch, bet, G):
    """d(sum(out * G)) / d weights of the sum combiner, float64 [nnz]: dot(BET row of the entry's id, G of its row)
    for a kept entry, 0 for a dropped one.  bet: lookup_weighted's [U, dim] BET."""
    frows, src, _ = fill_src(rows, vals, batch)
    _, fids, _ = fill(rows, vals, batch)
    _, inv = unique_first(fids)
    G = np.asarray(G, dtype=np.float64)
    gw = np.zeros(np.asarray(vals).size, dtype=np.float64)
    live = src >= 0
    gw[src[live]] = np.einsum("jd,jd->j", np.asarray(bet, dtype=np.float64)[inv[live]], G[frows[live]])
    return gw


def bound_weighted(rows, vals, weights, batch, absbet, combiner):
    """Per-row bound of the fp32 weighted combine: the m products are rounded once each and summed in some order
    (m u sum|w e|); the divisor, summed the same way and for sqrtn square-rooted, and the division add (m + 2) u more
    relative error.  Flushed subnormal products lose at most 2^-126 each."""
    frows, _, cnt, fids, w = _weighted_fill(rows, vals, weights, batch)
    _, inv = unique_first(fids)
    mag = np.zeros((batch, absbet.shape[1]), dtype=np.float64)
    np.add.at(mag, frows, np.abs(w)[:, None] * absbet[inv])
    m = np.maximum(cnt, 1).astype(np.float64)[:, None]
    s = np.abs(weighted_scale(rows, vals, weights, batch, combiner))[:, None]
    u = 2.0 ** -24
    return ((2 * m + 4) * u * mag + m * 2.0 ** -126) * s + 2.0 ** -149


def grad_bound_weighted(rows, vals, weights, batch, n_unique, absG, combiner):
    """Bound of the fp32 weighted backward: each addend G w / d carries the product's and the division's roundings and
    the divisor's error ((m_row + 3) u relative), and the addends of one unique id are summed in some order."""
    frows, src, cnt, fids, w = _weighted_fill(rows, vals, weights, batch)
    _, inv = unique_first(fids)
    s = np.abs(weighted_scale(rows, vals, weights, batch, combiner))
    live = src >= 0
    a = absG[frows[live]] * (np.abs(w[live]) * s[frows[live]])[:, None]
    u = 2.0 ** -24
    mag = np.zeros((n_unique, absG.shape[1]), dtype=np.float64)
    own = np.zeros_like(mag)
    np.add.at(mag, inv[live], a)
    np.add.at(own, inv[live], a * (cnt[frows[live]] + 3)[:, None] * u)
    mult = np.bincount(inv[live], minlength=n_unique).astype(np.float64)[:, None]
    return np.maximum(mult - 1, 0) * u * mag + own + (mult + 1) * 2.0 ** -126


def grad_weights_bound(rows, vals, batch, absbet, absG):
    """Bound of the fp32 weight gradient: a dot product of dim terms, each rounded once, summed in some order."""
    frows, src, _ = fill_src(rows, vals, batch)
    _, fids, _ = fill(rows, vals, batch)
    _, inv = unique_first(fids)
    dim = absbet.shape[1]
    gb = np.zeros(np.asarray(vals).size, dtype=np.float64)
    live = src >= 0
    gb[src[live]] = dim * 2.0 ** -24 * np.einsum("jd,jd->j", absbet[inv[live]], absG[frows[live]]) + dim * 2.0 ** -126
    return gb
