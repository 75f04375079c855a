"""Float64 reference of the Wide & Deep tower (include/b200_deepfm.h, b200_deepfm_wide_deep_*) -- TEST INFRASTRUCTURE.

Wide & Deep is DeepFM without the FM term (workloads.deepfm.WideDeepTower):
    logit = sum(wide) + w_dense . dense + w3 . relu(W2 relu(W1 [dense | deep] + b1) + b2),  loss = mean BCE,
with DeepFM's flat parameter layout.  `wide_deep_reference` is tower_oracle.tower_reference with the FM term left
out of the logit, of the row gradients and of the magnitude pass; the bound, the comparator and the helpers are
tower_oracle's (re-exported here), which applies unchanged: Wide & Deep's accumulation chains are a subset of
DeepFM's, so `chain_lengths` is still an upper bound.
"""
import torch

from oracle.tower_oracle import (  # noqa: F401  (re-exported: the tests use this module as the tower's oracle)
    C_TOL, D, FAMILIES, H1, H2, ND, P_FLOOR, WD_PAD, _scatter_rows, caught_by, chain_lengths, check,
    first_occurrence_inverse, flatten, layout, near_relu_kink, random_params, ratios, unflatten)


def wide_deep_reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params, weight=None):
    """Float64 forward + backward of one batch, with the inputs, the optional per-sample weight and the outputs of
    tower_oracle.tower_reference: logits, loss, grads, gsum_wide, gsum_deep, h1, h2, "M" (magnitudes), n_unique,
    occ."""
    f64 = torch.float64
    G, B = inv.shape
    dev = inv.device
    inv_l = inv.long()
    wide = torch.gather(bet_wide.reshape(G, B), 1, inv_l).to(f64)  # [G, B]
    deep = torch.gather(bet_deep.reshape(G, B, D), 1, inv_l.unsqueeze(2).expand(G, B, D)).to(f64)  # [G, B, 8]
    dense = dense.to(f64)
    y = labels.to(f64)
    wd, W1, b1, W2, b2, w3 = (t.to(f64) for t in unflatten(params, G))
    w = torch.ones(B, dtype=f64, device=dev) if weight is None else weight.to(f64)

    # forward: x = [dense | deep of group 0 | ... | deep of group G-1]
    x = torch.cat([dense, deep.permute(1, 0, 2).reshape(B, G * D)], 1)
    h1 = x @ W1.t() + b1
    m1 = (h1 > 0).to(f64)
    a1 = h1 * m1
    h2 = a1 @ W2.t() + b2
    m2 = (h2 > 0).to(f64)
    a2 = h2 * m2
    z = wide.sum(0) + dense @ wd + a2 @ w3
    lb = z.clamp_min(0) - z * y + torch.log1p(torch.exp(-z.abs()))  # BCE with logits
    loss = (w * lb).sum() / B

    # backward
    p = torch.sigmoid(z)
    dz = (p - y) / B * w
    dh2 = dz.unsqueeze(1) * w3 * m2
    dh1 = (dh2 @ W2) * m1
    ddeep = (dh1 @ W1)[:, ND:].reshape(B, G, D).permute(1, 0, 2)
    grads = flatten((dense.t() @ dz, dh1.t() @ x, dh1.sum(0), dh2.t() @ a1, dh2.sum(0), a2.t() @ dz), G)

    # magnitude pass: the same sums over |operands|, masks of the float64 forward
    aw = w.abs()
    X = x.abs()
    W1a, W2a, w3a = W1.abs(), W2.abs(), w3.abs()
    Mh1 = X @ W1a.t() + b1.abs()
    Ma1 = Mh1 * m1
    Mh2 = Ma1 @ W2a.t() + b2.abs()
    Ma2 = Mh2 * m2
    Mz = wide.abs().sum(0) + dense.abs() @ wd.abs() + Ma2 @ w3a
    # an error e in z moves the sample's loss by |p - y| e <= (1 + |y|) e and p by p (1 - p) e
    Mlb = Mz * (1 + y.abs()) + torch.log1p(torch.exp(-z.abs()))
    Mdz = (p * (1 - p) * Mz + p + y.abs() + P_FLOOR) / B * aw
    Mdh2 = Mdz.unsqueeze(1) * w3a * m2
    Mdh1 = (Mdh2 @ W2a) * m1
    Mddeep = (Mdh1 @ W1a)[:, ND:].reshape(B, G, D).permute(1, 0, 2)
    M = {
        "logits": Mz, "loss": (aw * Mlb).sum() / B, "h1": Mh1, "h2": Mh2,
        "grads": flatten((dense.abs().t() @ Mdz, Mdh1.t() @ X, Mdh1.sum(0), Mdh2.t() @ Ma1, Mdh2.sum(0),
                          Ma2.t() @ Mdz), G),
        "gsum_deep": _scatter_rows(Mddeep, inv, B),
        "gsum_wide": _scatter_rows(Mdz.unsqueeze(0).expand(G, B).unsqueeze(2), inv, B).squeeze(2),
    }
    occ = _scatter_rows(torch.ones((G, B, 1), dtype=f64, device=dev), inv, B).squeeze(2)
    return {"logits": z, "loss": loss, "grads": grads,
            "gsum_wide": _scatter_rows(dz.unsqueeze(0).expand(G, B).unsqueeze(2), inv, B).squeeze(2),
            "gsum_deep": _scatter_rows(ddeep, inv, B),
            "h1": h1, "h2": h2, "M": M, "n_unique": n_unique.to(device=dev, dtype=torch.int64), "occ": occ}


def mutations(ref, inputs, tile=32):
    """tower_oracle.mutations for Wide & Deep: the reference's outputs with one classic tiled-reduction fault each,
    name -> dict of outputs.  inputs: the tuple wide_deep_reference took."""
    G, B = ref["gsum_wide"].shape
    dev = ref["logits"].device
    keys = ("logits", "loss", "grads", "gsum_wide", "gsum_deep")
    base = {k: ref[k] for k in keys}
    out = {}

    def weighted(wt):
        r = wide_deep_reference(*inputs, weight=wt)
        return {k: r[k] for k in keys}

    one = torch.ones(B, dtype=torch.float64, device=dev)
    drop = B // 2 + 7 if B > 64 else B // 2
    wt = one.clone()
    wt[drop] = 0
    out["drop_one_sample"] = weighted(wt)
    wt = one.clone()
    wt[B - 1] = 32  # dead lanes of a partial tile replaying the last sample, unmasked
    out["last_sample_x32"] = weighted(wt)
    t = (B // tile) // 2
    wt = one.clone()
    wt[t * tile:(t + 1) * tile] = 0
    out["tile_missing_from_grads"] = dict(base, grads=weighted(wt)["grads"])
    gw, gd = ref["gsum_wide"].clone(), ref["gsum_deep"].clone()
    gw[G - 1, 0] = 0
    gd[G - 1, 0] = 0
    out["id_row_missing"] = dict(base, gsum_wide=gw, gsum_deep=gd)
    out["loss_not_divided_by_B"] = dict(base, loss=ref["loss"] * B)
    return out
