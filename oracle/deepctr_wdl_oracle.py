"""Float64 reference of the deepctr WDL tower (include/b200_deepctr_wdl.h) -- TEST INFRASTRUCTURE.

deepctr's WDL of model_zoo/deepctr/wdl.py:19-75, from raw rows: ids = FarmHash Fingerprint64 % 10000 of the 26
string columns (oracle/feature_oracle.py; "" is an ordinary bucket), x = [E_1[id_1] .. E_26[id_26] | I] (F = 117),
three relu layers 256 -> 128 -> 64, z = h3 wd + sum_j L_j[id_j] + I w_lin + global_bias, the Keras clipped
binary cross-entropy on p = sigmoid(z) (DESIGN.md section 4, Q19), its batch mean, plus 1e-5 (sum |E_j|^2 +
sum |L_j|^2 + |w_lin|^2) over whole tables.  The gradient is the complete flat gradient: every table row gets
2e-5 W plus its occurrences (Q28).  deepctr's layer details are RECALLED, not read from its source (Q27).
Plain torch float64, forward and backward written out by hand (no autograd), device-agnostic.

The error bound is tower_oracle's: |got - ref| <= C_TOL * sqrt(n) * 2^-24 * M elementwise, M from a magnitude
pass (the same sums over |operands|, plus the propagated error of z) and n the longest fp32 accumulation chain.
"""
import math

import numpy as np
import torch

from oracle import feature_oracle as FO
from oracle import tf32
from oracle.tower_oracle import C_TOL, EPS32, P_FLOOR

FIELDS, DENSE, ROWS, DIM = 26, 13, 10000, 4
NS, F = FIELDS * DIM, FIELDS * DIM + DENSE
H = (256, 128, 64)
LAMBDA = 1e-5
TILE = 64
N_PARAMS, N_TABLES = 1371438, 1300000
O_LIN = FIELDS * ROWS * DIM
DNN_SHAPES = [(DENSE, 1), (F, H[0]), (H[0],), (H[0], H[1]), (H[1],), (H[1], H[2]), (H[2],), (H[2], 1), (1,)]
EPS = float(torch.tensor(1e-7, dtype=torch.float32))
HI = float(torch.tensor(1.0, dtype=torch.float32) - EPS)
MUTATIONS = ("l2_touched_only", "no_l2", "dense_first", "no_linear_kernel", "no_global_bias", "unclipped",
             "no_last_relu", "bins_off_by_one")


def ids_from_raw(raw, bins=ROWS):
    """raw: 26 lists of B byte strings -> int64 [26, B] (Hash(bins), tf.strings.to_hash_bucket_fast)."""
    return torch.from_numpy(np.stack([FO.hashing([bytes(s) for s in col], bins) for col in raw]))


def unflatten(flat):
    """(deep [26, 10000, 4], linear [26, 10000], [w_lin, W0, b0, W1, b1, W2, b2, wd, gb])."""
    deep = flat[:O_LIN].reshape(FIELDS, ROWS, DIM)
    lin = flat[O_LIN:N_TABLES].reshape(FIELDS, ROWS)
    out, o = [], N_TABLES
    for s in DNN_SHAPES:
        k = math.prod(s)
        out.append(flat[o:o + k].reshape(s))
        o += k
    assert o == N_PARAMS
    return deep, lin, out


def reference(ids, dense, labels, flat, mutate=(), contraction=None):
    """{loss, logits [B], grads [1371438], B, M: magnitudes of each}.  ids int [26, B] in [0, 10000), dense
    [13, B], labels [B], flat [1371438].  mutate: names of MUTATIONS to build in (bins_off_by_one acts on raw rows:
    see mutations()).  contraction: the hidden layers' forward, data and weight contractions in the modes of
    oracle/tf32.py (tf32.modes; exact by default)."""
    mode = tf32.modes(contraction)

    def mm(kind, a, b):
        return tf32.contract(a, b, mode[kind])

    dev = flat.device
    flat = flat.to(torch.float64)
    ids = ids.long().to(dev)
    I = dense.to(device=dev, dtype=torch.float64).t()  # noqa: E741  [B, 13]
    y = labels.to(device=dev, dtype=torch.float64)
    B = I.shape[0]
    deep, lin, (wl, W0, b0, W1, b1, W2, b2, wd, gb) = unflatten(flat)
    fa = torch.arange(FIELDS, device=dev).unsqueeze(1)
    E = deep[fa, ids].permute(1, 0, 2).reshape(B, NS)  # [B, 104]
    x = torch.cat([I, E], 1) if "dense_first" in mutate else torch.cat([E, I], 1)
    a1 = mm("forward", x, W0) + b0
    h1 = a1.clamp(min=0)
    a2 = mm("forward", h1, W1) + b1
    h2 = a2.clamp(min=0)
    a3 = mm("forward", h2, W2) + b2
    h3 = a3 if "no_last_relu" in mutate else a3.clamp(min=0)
    lv = lin[fa, ids]  # [26, B]
    z = (h3 @ wd)[:, 0] + lv.sum(0)
    if "no_linear_kernel" not in mutate:
        z = z + (I @ wl)[:, 0]
    if "no_global_bias" not in mutate:
        z = z + gb[0]
    p = torch.sigmoid(z)
    if "unclipped" in mutate:
        loss_b = -(y * torch.log(p) + (1 - y) * torch.log(1 - p))
        dz = (p - y) / B
    else:
        pc = p.clamp(EPS, HI)
        loss_b = -(y * torch.log(pc + EPS) + (1 - y) * torch.log(1 - pc + EPS))
        passes = (p >= EPS) & (p <= HI)
        dz = torch.where(passes, -(y / (pc + EPS) - (1 - y) / (1 - pc + EPS)) * p * (1 - p), torch.zeros_like(p)) / B
    l2 = 0.0 if "no_l2" in mutate else LAMBDA
    sq = (deep * deep).sum() + (lin * lin).sum() + (wl * wl).sum()
    loss = loss_b.mean() + l2 * sq

    m3 = (a3 > 0) | ("no_last_relu" in mutate)
    dh3 = dz.unsqueeze(1) * wd[:, 0] * m3
    dh2 = mm("data", dh3, W2.t()) * (a2 > 0)
    dh1 = mm("data", dh2, W1.t()) * (a1 > 0)
    dx = mm("data", dh1, W0.t())
    dE = dx[:, DENSE:] if "dense_first" in mutate else dx[:, :NS]
    gdeep = torch.zeros_like(deep)
    glin = torch.zeros_like(lin)
    for j in range(FIELDS):
        gdeep[j].index_add_(0, ids[j], dE[:, DIM * j:DIM * (j + 1)])
        glin[j].index_add_(0, ids[j], dz)
    if "l2_touched_only" in mutate:
        touched = torch.zeros((FIELDS, ROWS), dtype=torch.bool, device=dev)
        touched[fa.expand_as(ids), ids] = True
        gdeep = gdeep + 2 * l2 * deep * touched.unsqueeze(2)
        glin = glin + 2 * l2 * lin * touched
    else:
        gdeep = gdeep + 2 * l2 * deep
        glin = glin + 2 * l2 * lin
    grads = torch.cat([gdeep.reshape(-1), glin.reshape(-1), (I.t() @ dz + 2 * l2 * wl[:, 0]).reshape(-1),
                       mm("weight", x.t(), dh1).reshape(-1), dh1.sum(0), mm("weight", h1.t(), dh2).reshape(-1),
                       dh2.sum(0), mm("weight", h2.t(), dh3).reshape(-1), dh3.sum(0), h3.t() @ dz,
                       dz.sum().reshape(1)])

    # magnitudes
    ax, aI = x.abs(), I.abs()
    Mh1 = ax @ W0.abs() + b0.abs()
    Mh2 = Mh1 @ W1.abs() + b1.abs()
    Mh3 = Mh2 @ W2.abs() + b2.abs()
    Mz = (Mh3 @ wd.abs())[:, 0] + lv.abs().sum(0) + (aI @ wl.abs())[:, 0] + gb.abs()[0]
    Mdz = dz.abs() + (0.25 * Mz + P_FLOOR) / B
    Mdh3 = Mdz.unsqueeze(1) * wd[:, 0].abs()
    Mdh2 = Mdh3 @ W2.abs().t()
    Mdh1 = Mdh2 @ W1.abs().t()
    Mdx = Mdh1 @ W0.abs().t()
    MdE = Mdx[:, DENSE:] if "dense_first" in mutate else Mdx[:, :NS]
    Mdeep = 2 * LAMBDA * deep.abs()
    Mlin = 2 * LAMBDA * lin.abs()
    for j in range(FIELDS):
        Mdeep[j].index_add_(0, ids[j], MdE[:, DIM * j:DIM * (j + 1)])
        Mlin[j].index_add_(0, ids[j], Mdz)
    Mgrads = torch.cat([Mdeep.reshape(-1), Mlin.reshape(-1), (aI.t() @ Mdz + 2 * LAMBDA * wl[:, 0].abs()).reshape(-1),
                        (ax.t() @ Mdh1).reshape(-1), Mdh1.sum(0), (Mh1.t() @ Mdh2).reshape(-1), Mdh2.sum(0),
                        (Mh2.t() @ Mdh3).reshape(-1), Mdh3.sum(0), Mh3.t() @ Mdz, Mdz.sum().reshape(1)])
    Mloss = (loss_b.abs() + Mz).mean() + LAMBDA * sq
    return {"logits": z, "loss": loss, "grads": grads, "B": B,
            "M": {"logits": Mz, "loss": Mloss, "grads": Mgrads}}


def chain_lengths(B, n_sm=132):
    """Longest fp32 accumulation chain behind each output family: the forward's F + 256 + 128 + 64 + 39
    products, the backward's 64 + 128 + 256, then the batch sums (per CTA at most ceil(tiles / CTAs) tiles of 64,
    then over the CTAs' partials; a table row sums at most B occurrences)."""
    fwd = F + sum(H) + FIELDS + DENSE + 4
    tiles = -(-B // TILE)
    ctas = max(1, min(tiles, n_sm))
    per_cta = TILE * -(-tiles // ctas)
    return {"logits": fwd, "loss": fwd + per_cta + ctas + N_TABLES // (4 * n_sm),
            "grads": fwd + sum(H) + max(per_cta + ctas, B)}


def _ratio(got, want, m, n, c):
    g = torch.as_tensor(got).to(device=want.device, dtype=torch.float64).reshape(want.shape)
    bound = c * math.sqrt(n) * EPS32 * m
    err = (g - want).abs()
    r = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                    torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
    r = torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))
    i = int(torch.argmax(r.reshape(-1)))
    return float(r.reshape(-1)[i]), i, float(g.reshape(-1)[i]), float(want.reshape(-1)[i])


def ratios(got, ref, c=C_TOL, n_sm=132):
    """Per family (logits, loss, grads): (worst err / bound, flat index, got, want)."""
    n = chain_lengths(ref["B"], n_sm)
    return {fam: _ratio(got[fam], ref[fam], ref["M"][fam], n[fam], c) for fam in ("logits", "loss", "grads")
            if fam in got}


def caught_by(got, ref, c=C_TOL, n_sm=132):
    return {fam for fam, (r, *_rest) in ratios(got, ref, c, n_sm).items() if not r <= 1.0}


def check(got, ref, c=C_TOL, label="", n_sm=132):
    """Assert every family within the bound; returns {family: worst ratio}."""
    rs = ratios(got, ref, c, n_sm)
    bad = {f: v for f, v in rs.items() if not v[0] <= 1.0}
    if bad:
        raise AssertionError("\n".join("%s %s: err/bound %.3g at %s (got %r, want %r)" % (label, f, r, w, gv, wv)
                                       for f, (r, w, gv, wv) in bad.items()))
    return {f: v[0] for f, v in rs.items()}


def mutations(ids, dense, labels, flat, raw=None, names=MUTATIONS):
    """name -> reference outputs with that fault built in.  bins_off_by_one hashes `raw` (26 lists of B byte
    strings) into 9999 buckets and is left out without raw."""
    out = {}
    for name in names:
        if name == "bins_off_by_one":
            if raw is not None:
                out[name] = reference(ids_from_raw(raw, ROWS - 1), dense, labels, flat)
        else:
            out[name] = reference(ids, dense, labels, flat, mutate=(name,))
    return out
