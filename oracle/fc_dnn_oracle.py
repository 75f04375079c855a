"""Float64 reference of the feature-column DNN tower (include/b200_fc_dnn.h) -- TEST INFRASTRUCTURE.

The models of model_zoo/census_dnn_model/census_functional_api.py:19-30 and model_zoo/heart_functional_api/
heart_functional_api.py:45-57: x = DenseFeatures(columns) [B, F], h1 = relu(x W1 + b1), h2 = relu(h1 W2 + b2),
z = h2 W3 + b3, p = sigmoid(z), Keras binary cross-entropy on p with the clip (DESIGN.md section 4, Q19), the
loss and the gradients a batch sum or mean (Q16).  Plain torch float64, forward and backward written out by hand
(no autograd), device-agnostic.  A layout is the plain data of fc_dnn.Layout.spec(): {"F", "blocks": [(kind, src,
width, offset)], "tables": [(rows, dim)], "loss_mean"}.

The error bound is tower_oracle's: |got - ref| <= C_TOL * sqrt(n) * 2^-24 * M elementwise, M from a magnitude
pass (the same sums over |operands|, plus the propagated error of z) and n the longest fp32 accumulation chain.
"""
import math

import torch

from oracle.tower_oracle import C_TOL, EPS32, P_FLOOR

NUMERIC, BUCKET, EMBEDDING = 0, 1, 2
H = 16
TILE = 64  # B200_FC_DNN_TILE
EPS = float(torch.tensor(1e-7, dtype=torch.float32))        # Keras backend.epsilon() as a float32 tensor
HI = float(torch.tensor(1.0, dtype=torch.float32) - EPS)     # 1 - epsilon in float32


def unflatten(F, flat):
    sizes = [(F, H), (H,), (H, H), (H,), (H, 1), (1,)]
    out, o = [], 0
    for s in sizes:
        k = math.prod(s)
        out.append(flat[o:o + k].reshape(s))
        o += k
    return out


def dense_features(spec, numeric, ids, empty, inv, rows, sort_columns=True, zero_empty=True):
    """x [B, F] float64.  rows: [table k's [U_k, dim] unique rows]; inv [T, B]; empty bool [T, B].
    sort_columns=False puts the blocks in the order they are listed in reverse (a mutation: columns unsorted)."""
    B = numeric.shape[1]
    dev = numeric.device
    cols = []
    for kind, src, width, off in spec["blocks"]:
        if kind == NUMERIC:
            c = numeric[src].to(torch.float64).unsqueeze(1)
        elif kind == BUCKET:
            c = (ids[src].long().unsqueeze(1) == torch.arange(width, device=dev)).to(torch.float64)
        else:
            r = rows[src].to(torch.float64)
            c = r[inv[src].long()]
            if zero_empty:
                c = c * (~empty[src]).to(torch.float64).unsqueeze(1)
        cols.append((off, c))
    cols.sort(key=lambda oc: oc[0], reverse=not sort_columns)
    x = torch.cat([c for _, c in cols], 1)
    assert x.shape == (B, spec["F"])
    return x


def fc_dnn_reference(spec, numeric, ids, empty, inv, n_unique, rows, labels, flat, weight=None, mutate=()):
    """{logits, loss, grads [16 F + 305], gsum [table k's [n_unique_k, dim]], B, M: magnitudes}.

    weight [B] (optional) scales each sample's loss (0 drops a sample, 2 counts it twice).  mutate: names of
    faults to build in -- "no_relu_mask", "unsorted", "empty_not_zeroed", "swap_reduction", "clip_grad_kept"."""
    F = spec["F"]
    B = numeric.shape[1]
    mean = spec["loss_mean"] != ("swap_reduction" in mutate)
    W1, b1, W2, b2, W3, b3 = [t.to(torch.float64) for t in unflatten(F, flat)]
    x = dense_features(spec, numeric, ids, empty, inv, rows, "unsorted" not in mutate, "empty_not_zeroed" not in mutate)
    a1 = x @ W1 + b1
    h1 = a1.clamp(min=0)
    a2 = h1 @ W2 + b2
    h2 = a2.clamp(min=0)
    z = (h2 @ W3 + b3)[:, 0]
    y = labels.to(torch.float64)
    p = torch.sigmoid(z)
    pc = p.clamp(EPS, HI)
    lo, l1 = torch.log(pc + EPS), torch.log(1 - pc + EPS)
    loss_b = -(y * lo + (1 - y) * l1)
    wt = torch.ones_like(z) if weight is None else weight.to(torch.float64)
    scale = 1.0 / B if mean else 1.0
    passes = (p >= EPS) & (p <= HI)
    if "clip_grad_kept" in mutate:
        passes = torch.ones_like(passes)
    dz = torch.where(passes, -(y / (pc + EPS) - (1 - y) / (1 - pc + EPS)) * p * (1 - p), torch.zeros_like(p))
    dz = dz * wt * scale
    m1 = (a1 > 0) | ("no_relu_mask" in mutate)
    m2 = (a2 > 0) | ("no_relu_mask" in mutate)
    dh2 = dz.unsqueeze(1) * W3[:, 0] * m2
    dh1 = (dh2 @ W2.t()) * m1
    grads = torch.cat([(x.t() @ dh1).reshape(-1), dh1.sum(0), (h1.t() @ dh2).reshape(-1), dh2.sum(0),
                       h2.t() @ dz, dz.sum().reshape(1)])
    loss = (loss_b * wt).sum() * scale

    # magnitudes
    ax = x.abs()
    Mh1 = ax @ W1.abs() + b1.abs()
    Mh2 = Mh1 @ W2.abs() + b2.abs()
    Mz = (Mh2 @ W3.abs())[:, 0] + b3.abs()
    Mdz = (dz.abs() + (0.25 * Mz + P_FLOOR) * wt.abs() * scale)
    Mdh2 = Mdz.unsqueeze(1) * W3[:, 0].abs()
    Mdh1 = Mdh2 @ W2.abs().t()
    Mgrads = torch.cat([(ax.t() @ Mdh1).reshape(-1), Mdh1.sum(0), (Mh1.t() @ Mdh2).reshape(-1), Mdh2.sum(0),
                        Mh2.t() @ Mdz, Mdz.sum().reshape(1)])
    Mloss = ((loss_b.abs() + Mz) * wt.abs()).sum() * scale

    gsum, Mgsum = [], []
    for k, (r, dim) in enumerate(spec["tables"]):
        off = [o for kind, src, _, o in spec["blocks"] if kind == EMBEDDING and src == k][0]
        U = int(n_unique[k])
        keep = (~empty[k]) if "empty_not_zeroed" not in mutate else torch.ones_like(empty[k])
        u = inv[k].long()
        S = torch.zeros((U, H), dtype=torch.float64, device=x.device)
        MS = torch.zeros_like(S)
        S.index_add_(0, u[keep], dh1[keep])
        MS.index_add_(0, u[keep], Mdh1[keep])
        Wk = W1[off:off + dim]
        gsum.append(S @ Wk.t())
        Mgsum.append(MS @ Wk.abs().t())
    return {"logits": z, "loss": loss, "grads": grads, "gsum": gsum, "B": B,
            "M": {"logits": Mz, "loss": Mloss, "grads": Mgrads, "gsum": Mgsum}, "F": F}


def chain_lengths(F, B, n_sm=132):
    """Longest fp32 accumulation chain behind each output family: the forward's F + 16 + 16 products, then the
    batch sums per CTA (at most ceil(tiles / CTAs) tiles of 64) and over the CTAs' partials, and for a row's
    gradient the 16 products of W1's block."""
    fwd = F + 2 * H + 4
    tiles = -(-B // TILE)
    ctas = max(1, min(tiles, n_sm))
    per_cta = TILE * -(-tiles // ctas)
    return {"logits": fwd, "loss": fwd + per_cta + ctas, "grads": fwd + 2 * H + per_cta + ctas,
            "gsum": fwd + 3 * H + per_cta + ctas}


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
    """Per family (logits, loss, grads, gsum_k): (worst err / bound, where, got, want).  got["gsum"][k] holds
    table k's first n_unique rows, in the dedup's order."""
    n = chain_lengths(ref["F"], ref["B"], n_sm)
    out = {}
    for fam in ("logits", "loss", "grads"):
        if fam in got:
            out[fam] = _ratio(got[fam], ref[fam], ref["M"][fam], n[fam], c)
    for k, (g, w, m) in enumerate(zip(got.get("gsum", []), ref["gsum"], ref["M"]["gsum"])):
        if tuple(g.shape) != tuple(w.shape):
            out["gsum_%d" % k] = (math.inf, (), float("nan"), float("nan"))
        else:
            out["gsum_%d" % k] = _ratio(g, w, m, n["gsum"], c)
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


MUTATIONS = ("no_relu_mask", "unsorted", "empty_not_zeroed", "swap_reduction", "clip_grad_kept", "tile_missing")


def mutations(spec, inputs, names=MUTATIONS):
    """name -> the outputs with that fault built in.  inputs: the arguments of fc_dnn_reference after spec.
    tile_missing: the gradients without the samples of one tile (the loss and logits as they were)."""
    keys = ("logits", "loss", "grads", "gsum")
    out = {}
    for name in names:
        if name == "tile_missing":
            B = inputs[0].shape[1]
            if B < 2 * TILE:
                continue
            t = (B // TILE) // 2
            wt = torch.ones(B, dtype=torch.float64, device=inputs[0].device)
            wt[t * TILE:(t + 1) * TILE] = 0
            base = fc_dnn_reference(spec, *inputs)
            r = fc_dnn_reference(spec, *inputs, weight=wt)
            out[name] = dict({k: base[k] for k in keys}, grads=r["grads"], gsum=r["gsum"])
        else:
            r = fc_dnn_reference(spec, *inputs, mutate=(name,))
            out[name] = {k: r[k] for k in keys}
    return out
