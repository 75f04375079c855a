"""Float64 reference of the census wide & deep tower (include/b200_census.h) -- TEST INFRASTRUCTURE.

The model of model_zoo/census_wide_deep_model/wide_deep_functional_api.py:164-212: per group g the sum of four
embedding rows, wide w_g(b) (groups 1, 2, dim 1) and deep e_g(b) (groups 1..3, dim 8); the DNN input x(b), three
Dense layers 24 -> 16 -> 8 -> 4 without activation, logit = w_1 + w_2 + sum(h3), loss = mean sigmoid
cross-entropy.  Plain torch float64, forward and backward written out by hand (no autograd), device-agnostic.

reference_reshape=False: x(b) = [e_1(b) | e_2(b) | e_3(b)].  reference_reshape=True (quirk Q11): the reference's
tf.reshape(deep_embeddings, (-1, 24)) of the list [e_1, e_2, e_3], i.e. stack -> [3, B, 8] -> [B, 24].

The error bound is tower_oracle's: |got - ref| <= C_TOL * sqrt(n) * 2^-24 * M elementwise, M from a magnitude
pass (the same sums over |operands|) and n the longest fp32 accumulation chain behind the output (`chain_lengths`).
Multi-step checks push each step's gradients into oracle.ps_oracle.OracleServer: the MLP gradients as dense
gradients and the five tables' rows as IndexedSlices on dense parameters (the Indexed kernels).
"""
import math

import numpy as np
import torch

from oracle.tower_oracle import C_TOL, EPS32, P_FLOOR

TILE = 256  # B200_CENSUS_TILE
GROUP_ROWS = (28, 75, 115)
# name, shape in flat order (b200_census.h); Keras auto-names in creation order (wide, then deep, then Dense)
PARAMS = [("dense/kernel:0", (24, 16)), ("dense/bias:0", (16,)), ("dense_1/kernel:0", (16, 8)),
          ("dense_1/bias:0", (8,)), ("dense_2/kernel:0", (8, 4)), ("dense_2/bias:0", (4,)),
          ("embedding/embeddings:0", (28, 1)), ("embedding_1/embeddings:0", (75, 1)),
          ("embedding_2/embeddings:0", (28, 8)), ("embedding_3/embeddings:0", (75, 8)),
          ("embedding_4/embeddings:0", (115, 8))]
MLP_NAMES = [n for n, _ in PARAMS[:6]]
TABLE_NAMES = [n for n, _ in PARAMS[6:]]
TABLE_GROUP = (0, 1, 0, 1, 2)  # id group of each table
TABLE_DIM = (1, 1, 8, 8, 8)
OFFSETS = {}
_o = 0
for _n, _s in PARAMS:
    OFFSETS[_n] = _o
    _o += int(np.prod(_s))
N_PARAMS = _o
N_MLP = OFFSETS["embedding/embeddings:0"]
UNIQ_OFF = (0, 28, 103, 131, 206)
GSUM_OFF = tuple(OFFSETS[n] - N_MLP for n in TABLE_NAMES)
assert (N_PARAMS, N_MLP, GSUM_OFF) == (2419, 572, (0, 28, 103, 327, 927))


def unflatten(flat):
    """{name: view of the flat buffer in its shape}."""
    return {n: flat[OFFSETS[n]:OFFSETS[n] + int(np.prod(s))].view(s) for n, s in PARAMS}


def random_params(gen, device, emb=0.05, dtype=torch.float32):
    """The reference's initial values: Keras "uniform" embeddings U(-0.05, 0.05), glorot-uniform kernels and zero
    biases (biases drawn U(-0.1, 0.1) here instead, so that they matter in the checks)."""
    flat = torch.empty(N_PARAMS, dtype=dtype, device=device)
    v = unflatten(flat)
    for n, s in PARAMS:
        if n.endswith("embeddings:0"):
            lim = emb
        elif n.endswith("kernel:0"):
            lim = math.sqrt(6.0 / (s[0] + s[1]))
        else:
            lim = 0.1
        v[n].copy_((torch.rand(s, generator=gen, device=device, dtype=dtype) * 2 - 1) * lim)
    return flat


def dnn_input(e, reference_reshape):
    """e: [3, B, 8] (e_1, e_2, e_3) -> x [B, 24]."""
    B = e.shape[1]
    if reference_reshape:
        return e.reshape(B, 24)  # the stacked [3, B, 8] read row-major as [B, 24]
    return e.permute(1, 0, 2).reshape(B, 24)


def dnn_input_grad(dx, reference_reshape):
    """Inverse of dnn_input for the gradient: dx [B, 24] -> de [3, B, 8]."""
    B = dx.shape[0]
    if reference_reshape:
        return dx.reshape(3, B, 8)
    return dx.reshape(B, 3, 8).permute(1, 0, 2)


def _rows_sum(table, ids):
    """table [R, k], ids [4, B] -> [B, k]: the sum of the four rows of every sample."""
    return table[ids].sum(0)


def _scatter(vals, ids, rows):
    """vals [B, k] per sample, ids [4, B] -> [rows, k]: each sample's value added to each of its four rows."""
    out = torch.zeros((rows, vals.shape[1]), dtype=vals.dtype, device=vals.device)
    for j in range(ids.shape[0]):
        out.index_add_(0, ids[j], vals)
    return out


def census_reference(ids, labels, params, reference_reshape=False, weight=None):
    """Float64 forward + backward of one batch.  ids [12, B] (in range), labels [B], params [2419].
    weight [B] (optional): a multiplicity per sample in every reduction (1 everywhere is the real model).

    Returns a dict of float64 tensors on the inputs' device: logits [B], loss [], grads [572], x [B, 24],
    gsum [5 tables: [rows, dim]], touched [5 tables: bool [rows]], uniq [5: int64 ascending], n_unique [5],
    "M" (magnitudes of logits, loss, grads, gsum), "B"."""
    f64 = torch.float64
    dev = labels.device
    ids = torch.as_tensor(ids).to(device=dev, dtype=torch.int64)
    B = ids.shape[1]
    for g, rows in enumerate(GROUP_ROWS):
        gi = ids[4 * g:4 * g + 4]
        if gi.numel() and (int(gi.min()) < 0 or int(gi.max()) >= rows):
            raise ValueError("group %d has ids outside [0, %d)" % (g, rows))
    p = {n: v.to(f64) for n, v in unflatten(params.to(dev)).items()}
    y = labels.to(f64)
    w = torch.ones(B, dtype=f64, device=dev) if weight is None else weight.to(f64)
    gid = [ids[4 * g:4 * g + 4] for g in range(3)]
    W1, b1, W2, b2, W3, b3 = (p[n] for n in MLP_NAMES)
    wide_t = [p[TABLE_NAMES[0]], p[TABLE_NAMES[1]]]
    deep_t = [p[n] for n in TABLE_NAMES[2:]]

    # forward
    wide = [_rows_sum(wide_t[g], gid[g])[:, 0] for g in range(2)]
    e = torch.stack([_rows_sum(deep_t[g], gid[g]) for g in range(3)])  # [3, B, 8]
    x = dnn_input(e, reference_reshape)
    h1 = x @ W1 + b1
    h2 = h1 @ W2 + b2
    h3 = h2 @ W3 + b3
    z = wide[0] + wide[1] + h3.sum(1)
    lb = z.clamp_min(0) - z * y + torch.log1p(torch.exp(-z.abs()))
    loss = (w * lb).sum() / B

    # backward
    pz = torch.sigmoid(z)
    dz = (pz - y) / B * w
    dh3 = dz.unsqueeze(1).expand(B, 4)
    dh2 = dh3 @ W3.t()
    dh1 = dh2 @ W2.t()
    dx = dh1 @ W1.t()
    grads = torch.cat([(x.t() @ dh1).reshape(-1), dh1.sum(0), (h1.t() @ dh2).reshape(-1), dh2.sum(0),
                       (h2.t() @ dh3).reshape(-1), dh3.sum(0)])
    de = dnn_input_grad(dx, reference_reshape)
    gsum = [_scatter(dz.unsqueeze(1), gid[0], 28), _scatter(dz.unsqueeze(1), gid[1], 75)]
    gsum += [_scatter(de[g], gid[g], GROUP_ROWS[g]) for g in range(3)]

    # magnitude pass: the same sums over |operands|
    aw = w.abs()
    Mwide = [_rows_sum(wide_t[g].abs(), gid[g])[:, 0] for g in range(2)]
    Me = torch.stack([_rows_sum(deep_t[g].abs(), gid[g]) for g in range(3)])
    Mx = dnn_input(Me, reference_reshape)
    Mh1 = Mx @ W1.abs() + b1.abs()
    Mh2 = Mh1 @ W2.abs() + b2.abs()
    Mh3 = Mh2 @ W3.abs() + b3.abs()
    Mz = Mwide[0] + Mwide[1] + Mh3.sum(1)
    Mloss = (aw * (Mz * (1 + y.abs()) + torch.log1p(torch.exp(-z.abs())))).sum() / B
    Mdz = (pz * (1 - pz) * Mz + pz + y.abs() + P_FLOOR) / B * aw
    Mdh3 = Mdz.unsqueeze(1).expand(B, 4)
    Mdh2 = Mdh3 @ W3.abs().t()
    Mdh1 = Mdh2 @ W2.abs().t()
    Mdx = Mdh1 @ W1.abs().t()
    Mgrads = torch.cat([(Mx.t() @ Mdh1).reshape(-1), Mdh1.sum(0), (Mh1.t() @ Mdh2).reshape(-1), Mdh2.sum(0),
                        (Mh2.t() @ Mdh3).reshape(-1), Mdh3.sum(0)])
    Mde = dnn_input_grad(Mdx, reference_reshape)
    Mgsum = [_scatter(Mdz.unsqueeze(1), gid[0], 28), _scatter(Mdz.unsqueeze(1), gid[1], 75)]
    Mgsum += [_scatter(Mde[g], gid[g], GROUP_ROWS[g]) for g in range(3)]

    ones = torch.ones((B, 1), dtype=f64, device=dev)
    occ = [_scatter(ones, gid[TABLE_GROUP[t]], GROUP_ROWS[TABLE_GROUP[t]])[:, 0] for t in range(5)]
    touched = [o > 0 for o in occ]
    uniq = [torch.nonzero(tc).reshape(-1) for tc in touched]
    return {"logits": z, "loss": loss, "grads": grads, "x": x, "gsum": gsum, "occ": occ, "touched": touched,
            "uniq": uniq, "n_unique": [int(u.numel()) for u in uniq], "B": B,
            "M": {"logits": Mz, "loss": Mloss, "grads": Mgrads, "gsum": Mgsum}}


def chain_lengths(B, n_sm=132):
    """Longest fp32 accumulation chain behind each output family.  Forward: four rows per group, the 24 -> 16 ->
    8 -> 4 products and the logit's sum.  The batch sums run per CTA over its tiles (at most ceil(tiles / CTAs)
    tiles of 256 when there is one CTA per SM), then over the CTAs' partials; a row's sum has up to four
    occurrences per sample."""
    fwd = 4 + 24 + 16 + 8 + 8
    tiles = -(-B // TILE)
    ctas = max(1, min(tiles, n_sm))
    per_cta = TILE * -(-tiles // ctas)
    return {"logits": fwd, "loss": fwd + per_cta + ctas, "grads": fwd + 24 + per_cta + ctas,
            "gsum": fwd + 24 + 4 * per_cta + ctas}


def _ratio(got, want, m, n, c):
    g = torch.as_tensor(got).to(device=want.device, dtype=torch.float64).reshape(want.shape)
    bound = c * math.sqrt(n) * EPS32 * m
    err = (g - want).abs()
    r = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                    torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
    r = torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))
    if r.numel() == 0:
        return 0.0, (), float("nan"), float("nan")
    i = int(torch.argmax(r.reshape(-1)))
    where = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), r.shape)) if r.dim() else ()
    return float(r.reshape(-1)[i]), where, float(g.reshape(-1)[i]), float(want.reshape(-1)[i])


def ratios(got, ref, c=C_TOL, n_sm=132):
    """Per family (logits, loss, grads, gsum_0 .. gsum_4): (worst err / bound, where, got, want).  got["gsum"] is
    a list of five dense [rows, dim] tensors (rows not touched are compared too: they must be 0)."""
    n = chain_lengths(ref["B"], n_sm)
    out = {}
    for fam in ("logits", "loss", "grads"):
        if fam in got:
            out[fam] = _ratio(got[fam], ref[fam], ref["M"][fam], n[fam], c)
    if "gsum" in got:
        for t in range(5):
            out["gsum_%d" % t] = _ratio(got["gsum"][t], ref["gsum"][t], ref["M"]["gsum"][t], n["gsum"], c)
    return out


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


def mutations(ref, inputs):
    """The reference's outputs with one classic fault each: name -> dict of outputs.
    inputs: (ids, labels, params, reference_reshape)."""
    B = ref["B"]
    dev = ref["logits"].device
    keys = ("logits", "loss", "grads", "gsum")
    base = {k: ref[k] for k in keys}

    def weighted(wt):
        r = census_reference(*inputs, weight=wt)
        return {k: r[k] for k in keys}

    one = torch.ones(B, dtype=torch.float64, device=dev)
    out = {}
    wt = one.clone()
    wt[B // 2] = 0
    out["drop_one_sample"] = weighted(wt)
    wt = one.clone()
    wt[B - 1] = 2
    out["last_sample_twice"] = weighted(wt)
    if B >= 2 * TILE:
        t = (B // TILE) // 2
        wt = one.clone()
        wt[t * TILE:(t + 1) * TILE] = 0
        out["tile_missing_from_grads"] = dict(base, grads=weighted(wt)["grads"])
    gs = [g.clone() for g in ref["gsum"]]
    gs[4][int(ref["uniq"][4][0])] = 0
    out["row_missing"] = dict(base, gsum=gs)
    if B > 1:
        out["loss_not_divided_by_B"] = dict(base, loss=ref["loss"] * B)
    other = census_reference(inputs[0], inputs[1], inputs[2], not inputs[3])
    out["other_reshape_mode"] = {k: other[k] for k in keys}
    return out

