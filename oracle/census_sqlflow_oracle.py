"""Float64 reference of the census_model_sqlflow wide & deep models -- TEST INFRASTRUCTURE.

Two parts, restated from the reference (model_zoo/census_model_sqlflow/wide_and_deep/, elasticdl_preprocessing/)
independently of the CUDA code:

  sqlflow_ids(numeric, strings, variant): the raw rows -> ids [12, B] (-1 = absent) of the two id rules, on
      oracle/feature_oracle.py's Hashing and Discretization.  keras: ToSparse drops "" and 0.0 (to_sparse.py:55-
      63), IndexLookup(num_oov_tokens=1) maps an unknown string to len(vocabulary) (index_table_from_tensor with
      one OOV bucket: V + Fingerprint64 % 1), then ConcatenateWithOffset adds the offset to what is present.  fc:
      the categorical columns drop "", a vocabulary column maps an unknown string to -1, and
      concatenated_categorical_column adds the offset to every id it holds (feature_column.py:157-177); a negative
      id is pruned by safe_embedding_lookup_sparse; bucketized columns are dense.
  csql_reference(ids, labels, params, reference_reshape): forward and backward of one batch written out by hand
      (no autograd): per group the mean of the present ids' rows (zero for a group with none), Dense 24 -> 16 -> 8
      -> 4, logit = w_1 + w_2 + sum(h3), the mean sigmoid cross-entropy; reference_reshape = quirk Q11.

The error bound is tower_oracle's, as census_oracle uses it: |got - ref| <= C_TOL * sqrt(n) * 2^-24 * M, with M
from a magnitude pass and n the longest fp32 chain (`chain_lengths`).
"""
import math

import numpy as np
import torch

from oracle import census_oracle as CO
from oracle import feature_oracle as FO
from oracle.tower_oracle import C_TOL, P_FLOOR

TILE = 256  # B200_CSQL_TILE
GROUP_ROWS = (27, 73, 113)
SHAPES = [(24, 16), (16,), (16, 8), (8,), (8, 4), (4,), (27, 1), (73, 1), (27, 8), (73, 8), (113, 8)]
OFFS = [int(v) for v in np.cumsum([0] + [int(np.prod(s)) for s in SHAPES])]
N_PARAMS, N_MLP = OFFS[-1], OFFS[6]
TABLE_GROUP = (0, 1, 0, 1, 2)
assert (N_PARAMS, N_MLP, tuple(o - N_MLP for o in OFFS[6:11])) == (2376, 572, (0, 27, 100, 316, 900))


# ---------------------------------------------------------------------------------------------- the id rules
def _bucket_count(op, param):
    return param if op == "hash" else len(param) + (op == "bucketize")


def sqlflow_ids(numeric, strings, variant, features, groups, numeric_keys, string_keys, mutate=None):
    """numeric float32 [4, B] (numpy), strings: 8 lists of str; features {name: (op, param)}, groups [[4 names]]
    (feature_configs.py's data).  Returns int64 [12, B].  mutate: "offset_on_absent" (a dropped cell gets -1 +
    offset) or "swap_rules" (the other variant's rule)."""
    if mutate == "swap_rules":
        variant = "fc" if variant == "keras" else "keras"
    keras = variant == "keras"
    numeric = np.asarray(numeric, dtype=np.float32)
    B = numeric.shape[1]
    out = np.empty((12, B), dtype=np.int64)
    r = 0
    for names in groups:
        offsets = np.cumsum([0] + [_bucket_count(*features[n]) for n in names])[:-1]
        for name, off in zip(names, offsets):
            op, param = features[name]
            if op == "bucketize":
                x = numeric[numeric_keys.index(name)]
                ids = FO.discretize(x, param)
                dropped = (x == 0.0) if keras else np.zeros(B, dtype=bool)
            else:
                s = strings[string_keys.index(name)]
                dropped = np.array([v == "" for v in s], dtype=bool)
                if op == "hash":
                    ids = FO.hashing(s, param)
                else:
                    ids = np.array([param.index(v) if v in param else (len(param) if keras else -1) for v in s],
                                   dtype=np.int64)
            ids = ids + off
            out[r] = np.where(dropped, off - 1 if mutate == "offset_on_absent" else -1, ids)
            r += 1
    if not keras:
        out[out < 0] = -1  # pruned
    return out


# ------------------------------------------------------------------------------------------------ the tower
def unflatten(flat):
    return [flat[OFFS[i]:OFFS[i + 1]].view(s) for i, s in enumerate(SHAPES)]


def random_params(gen, device, emb=0.5, dtype=torch.float32):
    """Uniform embeddings U(-emb, emb), glorot-uniform kernels and biases U(-0.1, 0.1) (so that they matter)."""
    flat = torch.empty(N_PARAMS, dtype=dtype, device=device)
    for i, (v, s) in enumerate(zip(unflatten(flat), SHAPES)):
        lim = emb if i >= 6 else (math.sqrt(6.0 / (s[0] + s[1])) if i % 2 == 0 else 0.1)
        v.copy_((torch.rand(s, generator=gen, device=device, dtype=dtype) * 2 - 1) * lim)
    return flat


def _pool(table, gi, mutate):
    """table [R, k], gi [4, B] (-1 = absent) -> (pooled [B, k], per-sample scale of a row's gradient [B])."""
    present = gi >= 0
    n = present.sum(0).to(table.dtype)
    rows = table[gi.clamp_min(0)] * present.unsqueeze(2).to(table.dtype)
    s = rows.sum(0)
    if mutate == "sum":
        return s, present.any(0).to(table.dtype)
    div = torch.full_like(n, 4.0) if mutate == "absent_in_divisor" else n.clamp_min(1.0)
    out = s / div.unsqueeze(1)
    scale = torch.where(n > 0, 1.0 / div, torch.zeros_like(n))
    if mutate == "empty_not_zero":
        out = torch.where((n == 0).unsqueeze(1), table[0].expand_as(out), out)
    return out, scale


def _scatter(vals, gi, rows):
    """vals [B, k] per sample, gi [4, B] -> [rows, k]: each sample's value added to each of its present rows."""
    out = torch.zeros((rows, vals.shape[1]), dtype=vals.dtype, device=vals.device)
    for j in range(gi.shape[0]):
        m = gi[j] >= 0
        out.index_add_(0, gi[j][m], vals[m])
    return out


def csql_reference(ids, labels, params, reference_reshape=False, weight=None, mutate=None):
    """Float64 forward + backward of one batch.  ids [12, B] in [-1, rows), labels [B], params [2376]; weight [B]
    (optional) multiplies each sample in every reduction.  mutate: "sum", "absent_in_divisor" or "empty_not_zero"
    (faults in the pooling).  Returns the dict census_oracle.census_reference returns."""
    f64 = torch.float64
    dev = labels.device
    ids = torch.as_tensor(ids).to(device=dev, dtype=torch.int64)
    B = ids.shape[1]
    for g, rows in enumerate(GROUP_ROWS):
        gi = ids[4 * g:4 * g + 4]
        if gi.numel() and (int(gi.min()) < -1 or int(gi.max()) >= rows):
            raise ValueError("group %d has ids outside [-1, %d)" % (g, rows))
    p = [v.to(f64) for v in unflatten(params.to(dev))]
    y = labels.to(f64)
    w = torch.ones(B, dtype=f64, device=dev) if weight is None else weight.to(f64)
    gid = [ids[4 * g:4 * g + 4] for g in range(3)]
    W1, b1, W2, b2, W3, b3 = p[:6]

    wide_sc = [_pool(p[6 + g], gid[g], mutate) for g in range(2)]
    deep_sc = [_pool(p[8 + g], gid[g], mutate) for g in range(3)]
    wide = [v[:, 0] for v, _ in wide_sc]
    e = torch.stack([v for v, _ in deep_sc])
    x = CO.dnn_input(e, reference_reshape)
    h1 = x @ W1 + b1
    h2 = h1 @ W2 + b2
    h3 = h2 @ W3 + b3
    z = wide[0] + wide[1] + h3.sum(1)
    lb = z.clamp_min(0) - z * y + torch.log1p(torch.exp(-z.abs()))
    loss = (w * lb).sum() / B

    pz = torch.sigmoid(z)
    dz = (pz - y) / B * w
    dh3 = dz.unsqueeze(1).expand(B, 4)
    dh2 = dh3 @ W3.t()
    dh1 = dh2 @ W2.t()
    dx = dh1 @ W1.t()
    grads = torch.cat([(x.t() @ dh1).reshape(-1), dh1.sum(0), (h1.t() @ dh2).reshape(-1), dh2.sum(0),
                       (h2.t() @ dh3).reshape(-1), dh3.sum(0)])
    de = CO.dnn_input_grad(dx, reference_reshape)
    gsum = [_scatter((dz * wide_sc[g][1]).unsqueeze(1), gid[g], GROUP_ROWS[g]) for g in range(2)]
    gsum += [_scatter(de[g] * deep_sc[g][1].unsqueeze(1), gid[g], GROUP_ROWS[g]) for g in range(3)]

    # magnitude pass: the same sums over |operands|
    aw = w.abs()
    Mw = [_pool(p[6 + g].abs(), gid[g], None) for g in range(2)]
    Md = [_pool(p[8 + g].abs(), gid[g], None) for g in range(3)]
    Mx = CO.dnn_input(torch.stack([v for v, _ in Md]), reference_reshape)
    Mh1 = Mx @ W1.abs() + b1.abs()
    Mh2 = Mh1 @ W2.abs() + b2.abs()
    Mh3 = Mh2 @ W3.abs() + b3.abs()
    Mz = Mw[0][0][:, 0] + Mw[1][0][:, 0] + Mh3.sum(1)
    Mloss = (aw * (Mz * (1 + y.abs()) + torch.log1p(torch.exp(-z.abs())))).sum() / B
    Mdz = (pz * (1 - pz) * Mz + pz + y.abs() + P_FLOOR) / B * aw
    Mdh3 = Mdz.unsqueeze(1).expand(B, 4)
    Mdh2 = Mdh3 @ W3.abs().t()
    Mdh1 = Mdh2 @ W2.abs().t()
    Mdx = Mdh1 @ W1.abs().t()
    Mgrads = torch.cat([(Mx.t() @ Mdh1).reshape(-1), Mdh1.sum(0), (Mh1.t() @ Mdh2).reshape(-1), Mdh2.sum(0),
                        (Mh2.t() @ Mdh3).reshape(-1), Mdh3.sum(0)])
    Mde = CO.dnn_input_grad(Mdx, reference_reshape)
    Mgsum = [_scatter((Mdz * Mw[g][1]).unsqueeze(1), gid[g], GROUP_ROWS[g]) for g in range(2)]
    Mgsum += [_scatter(Mde[g] * Md[g][1].unsqueeze(1), gid[g], GROUP_ROWS[g]) for g in range(3)]

    ones = torch.ones((B, 1), dtype=f64, device=dev)
    occ = [_scatter(ones, gid[TABLE_GROUP[t]], GROUP_ROWS[TABLE_GROUP[t]])[:, 0] for t in range(5)]
    touched = [o > 0 for o in occ]
    uniq = [torch.nonzero(tc).reshape(-1) for tc in touched]
    return {"logits": z, "loss": loss, "grads": grads, "x": x, "gsum": gsum, "occ": occ, "touched": touched,
            "uniq": uniq, "n_unique": [int(u.numel()) for u in uniq], "B": B,
            "M": {"logits": Mz, "loss": Mloss, "grads": Mgrads, "gsum": Mgsum}}


def chain_lengths(B, n_sm=132):
    """census_oracle's chains plus one rounding for the mean's division in the forward and in each row scale."""
    n = CO.chain_lengths(B, n_sm)
    return {k: v + 2 for k, v in n.items()}


def ratios(got, ref, c=C_TOL, n_sm=132):
    n = chain_lengths(ref["B"], n_sm)
    out = {}
    for fam in ("logits", "loss", "grads"):
        if fam in got:
            out[fam] = CO._ratio(got[fam], ref[fam], ref["M"][fam], n[fam], c)
    if "gsum" in got:
        for t in range(5):
            out["gsum_%d" % t] = CO._ratio(got["gsum"][t], ref["gsum"][t], ref["M"]["gsum"][t], n["gsum"], c)
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


TOWER_MUTATIONS = ("sum", "absent_in_divisor", "empty_not_zero", "other_reshape_mode", "tile_missing_from_grads")
ID_MUTATIONS = ("offset_on_absent", "swap_rules")


def mutations(ref, inputs):
    """The tower faults: name -> outputs.  inputs: (ids, labels, params, reference_reshape).  The id-rule faults
    (ID_MUTATIONS) are sqlflow_ids(..., mutate=name)."""
    ids, labels, params, q11 = inputs
    keys = ("logits", "loss", "grads", "gsum")
    out = {}
    for m in ("sum", "absent_in_divisor", "empty_not_zero"):
        r = csql_reference(ids, labels, params, q11, mutate=m)
        out[m] = {k: r[k] for k in keys}
    r = csql_reference(ids, labels, params, not q11)
    out["other_reshape_mode"] = {k: r[k] for k in keys}
    B = ref["B"]
    if B >= 2 * TILE:
        t = (B // TILE) // 2
        wt = torch.ones(B, dtype=torch.float64, device=ref["logits"].device)
        wt[t * TILE:(t + 1) * TILE] = 0
        r = csql_reference(ids, labels, params, q11, weight=wt)
        out["tile_missing_from_grads"] = dict({k: ref[k] for k in keys}, grads=r["grads"])
    return out
