"""Float64 reference of the DCN tower (include/b200_deepfm.h, b200_deepfm_dcn_*) -- TEST INFRASTRUCTURE.

The companion of tower_oracle.py for the dac_ctr Deep & Cross Network: the same inputs (inv, n_unique, pulled
rows, dense, labels, flat parameters in the DCN layout), the same outputs and the same bound,
|got - ref| <= c * sqrt(n) * 2^-24 * M.  Plain torch float64, forward and backward written out by hand.

It computes the cross network's LITERAL layer recursion x_{l+1} = x0 (x_l . w_l) + b_l + x_l and its backward
layer by layer, not the closed form ((1 + a)(1 + c) + beta) e + gamma the CUDA tower uses, so a test against it
checks that algebra too.  `closed_form` evaluates the closed form separately.

CrossNet is deepctr's (third party, not in the reference tree, version unpinned by model_zoo/requirements.txt):
restated from the DCN paper's eq. 3 with deepctr's "vector" parameterization and l2 regularization of the two
kernels, loss += 1e-5 (|w_0|^2 + |w_1|^2).

Magnitudes of products: an fp32 product of k inexact factors x_i (|x_i| <= M_i, error <= c sqrt(n) eps M_i) is off
by at most c sqrt(n) eps k prod M_i, so such a product's magnitude is k prod M_i.
"""
import math

import torch

from oracle.tower_oracle import (C_TOL, D, EPS32, FAMILIES, FLT_MIN, H1, H2, ND, P_FLOOR, WD_PAD, _scatter_rows,
                                 first_occurrence_inverse, near_relu_kink)

L2 = 1e-5
CROSS_LAYERS = 2
__all__ = ["layout", "unflatten", "flatten", "random_params", "dcn_reference", "closed_form", "chain_lengths",
           "ratios", "caught_by", "check", "mutations", "first_occurrence_inverse", "near_relu_kink"]


def layout(G):
    """Offsets of the flat DCN buffer: [w_dense 13 (+3 pad) | w1 16 x in | b1 16 | w2 4 x 16 | b2 4 | w_out 4 + in |
    w_0 w_1 2 x in | b_0 b_1 2 x in], in = 13 + 8G."""
    n_in = ND + D * G
    o = {"in": n_in, "wd": 0, "w1": WD_PAD}
    o["b1"] = o["w1"] + H1 * n_in
    o["w2"] = o["b1"] + H1
    o["b2"] = o["w2"] + H2 * H1
    o["wout"] = o["b2"] + H2
    o["cw"] = o["wout"] + H2 + n_in
    o["cb"] = o["cw"] + CROSS_LAYERS * n_in
    o["total"] = o["cb"] + CROSS_LAYERS * n_in
    return o


def unflatten(flat, G):
    """(wd [13], W1 [16, in], b1 [16], W2 [4, 16], b2 [4], w_out [4 + in], cw [2, in], cb [2, in]) views."""
    o = layout(G)
    n = o["in"]
    return (flat[o["wd"]:o["wd"] + ND], flat[o["w1"]:o["b1"]].view(H1, n), flat[o["b1"]:o["b1"] + H1],
            flat[o["w2"]:o["b2"]].view(H2, H1), flat[o["b2"]:o["b2"] + H2], flat[o["wout"]:o["cw"]],
            flat[o["cw"]:o["cb"]].view(CROSS_LAYERS, n), flat[o["cb"]:o["total"]].view(CROSS_LAYERS, n))


def flatten(parts, G, pad=0.0):
    """Inverse of unflatten; the 3 padding floats after w_dense are set to `pad`."""
    o = layout(G)
    flat = torch.full((o["total"],), pad, dtype=parts[0].dtype, device=parts[0].device)
    starts = ("wd", "w1", "b1", "w2", "b2", "wout", "cw", "cb")
    for k, part in zip(starts, parts):
        flat[o[k]:o[k] + part.numel()] = part.reshape(-1)
    return flat


def random_params(G, gen, device, w1_gain=2.0, b1=None, b2=None, wd_std=0.3, pad=0.0, cross_gain=1.0, cb_std=0.1):
    """A float32 flat DCN buffer with every part O(1)-relevant: the DNN as tower_oracle.random_params draws it,
    w_out ~ U(-1, 1) on the DNN units and N(0, 1 / in) on the cross units, cross kernels N(0, cross_gain^2 / in)
    (a, c = O(cross_gain)) and cross biases N(0, cb_std^2) (nonzero, so that beta, gamma and the rank-1 parts of
    the gradients are exercised)."""
    n_in = ND + D * G

    def u(shape, a):
        return (torch.rand(shape, generator=gen, device=device) * 2 - 1) * a

    wd = torch.randn(ND, generator=gen, device=device) * wd_std
    w1 = torch.randn((H1, n_in), generator=gen, device=device) * (w1_gain / math.sqrt(n_in))
    bb1 = u(H1, 0.3) if b1 is None else torch.full((H1,), float(b1), device=device)
    w2 = u((H2, H1), 0.5)
    bb2 = u(H2, 0.5) if b2 is None else torch.as_tensor(b2, dtype=torch.float32, device=device).expand(H2).clone()
    wout = torch.cat([u(H2, 1.0), torch.randn(n_in, generator=gen, device=device) / math.sqrt(n_in)])
    cw = torch.randn((CROSS_LAYERS, n_in), generator=gen, device=device) * (cross_gain / math.sqrt(n_in))
    cb = torch.randn((CROSS_LAYERS, n_in), generator=gen, device=device) * cb_std
    return flatten((wd, w1, bb1, w2, bb2, wout, cw, cb), G, pad=pad)


def closed_form(x0, cw, cb, wc):
    """The cross logit w_out_cross . x_2 as the CUDA tower computes it: ((1 + a)(1 + c) + beta) e + gamma with
    a = x0.w0, c = x0.w1, e = x0.wc, beta = b0.w1, gamma = wc.(b0 + b1).  x0 [B, in] float64."""
    a, c, e = x0 @ cw[0], x0 @ cw[1], x0 @ wc
    beta, gamma = cb[0] @ cw[1], wc @ (cb[0] + cb[1])
    return ((1 + a) * (1 + c) + beta) * e + gamma


def chain_lengths(G, B, n_sm=132):
    """tower_oracle.chain_lengths with the cross network's chains: the logit adds beta / gamma, reductions over
    the 13 + 8G inputs of their own (the prologue's), and the loss the l2 term's reduction over 2 (13 + 8G)."""
    n_in = ND + D * G
    fwd = 2 * n_in + 32
    bwd = fwd + 32
    per_cta = 32 * -(-(-(-B // 32)) // n_sm)
    nb = min(B, per_cta + 8 * n_sm)
    return {"logits": fwd, "loss": fwd + nb + 2 * n_in, "grads": bwd + nb, "gsum_wide": bwd, "gsum_deep": bwd}


def dcn_reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params, weight=None):
    """Float64 forward + backward of one batch (tower_oracle.tower_reference's contract, DCN model and layout).
    weight [B] (optional): a multiplicity per sample in every reduction (the comparator's mutations).
    Returns logits, loss, grads, gsum_wide, gsum_deep, h1 / h2 (DNN pre-activations), "x1" / "x2" (the cross
    layers' outputs), "M", "n_unique", "occ"."""
    f64 = torch.float64
    G, B = inv.shape
    dev = inv.device
    inv_l = inv.long()
    wide = torch.gather(bet_wide.reshape(G, B), 1, inv_l).to(f64)
    deep = torch.gather(bet_deep.reshape(G, B, D), 1, inv_l.unsqueeze(2).expand(G, B, D)).to(f64)
    dense = dense.to(f64)
    y = labels.to(f64)
    wd, W1, b1, W2, b2, wout, cw, cb = (t.to(f64) for t in unflatten(params, G))
    w3, wc = wout[:H2], wout[H2:]
    w = torch.ones(B, dtype=f64, device=dev) if weight is None else weight.to(f64)

    # forward: x0 = [dense | deep of group 0 | ... | deep of group G-1]
    x0 = torch.cat([dense, deep.permute(1, 0, 2).reshape(B, G * D)], 1)
    h1 = x0 @ W1.t() + b1
    m1 = (h1 > 0).to(f64)
    a1 = h1 * m1
    h2 = a1 @ W2.t() + b2
    m2 = (h2 > 0).to(f64)
    a2 = h2 * m2
    xs, ss = [x0], []  # x_l and s_l = x_l . w_l, layer by layer
    for l in range(CROSS_LAYERS):
        ss.append(xs[-1] @ cw[l])
        xs.append(x0 * ss[-1].unsqueeze(1) + cb[l] + xs[-1])
    xL = xs[-1]
    lin = wide.sum(0) + dense @ wd
    z = lin + a2 @ w3 + xL @ wc
    lb = z.clamp_min(0) - z * y + torch.log1p(torch.exp(-z.abs()))
    l2 = L2 * (cw * cw).sum()
    loss = (w * lb).sum() / B + l2

    # backward
    p = torch.sigmoid(z)
    dz = (p - y) / B * w
    dw3 = a2.t() @ dz
    dwc = xL.t() @ dz
    dh2 = dz.unsqueeze(1) * w3 * m2
    dW2 = dh2.t() @ a1
    db2 = dh2.sum(0)
    dh1 = (dh2 @ W2) * m1
    dW1 = dh1.t() @ x0
    db1 = dh1.sum(0)
    dwd = dense.t() @ dz
    # cross layers, last to first: x_{l+1} = x0 s_l + b_l + x_l, s_l = x_l . w_l
    dx = dz.unsqueeze(1) * wc  # d loss / d x_L
    dx0_cross = torch.zeros_like(x0)
    dcw, dcb = torch.zeros_like(cw), torch.zeros_like(cb)
    for l in reversed(range(CROSS_LAYERS)):
        ds = (dx * x0).sum(1)  # d / d s_l
        dx0_cross = dx0_cross + dx * ss[l].unsqueeze(1)
        dcb[l] = dx.sum(0)
        dcw[l] = xs[l].t() @ ds
        dx = dx + ds.unsqueeze(1) * cw[l]  # d / d x_l through s_l and the residual
    dcw = dcw + 2 * L2 * cw
    dx0 = dh1 @ W1 + dx0_cross + dx  # dx: what reached x_0 through the residual chain
    ddeep = dx0[:, ND:].reshape(B, G, D).permute(1, 0, 2)
    dwide = dz.unsqueeze(0).expand(G, B)
    gsum_deep = _scatter_rows(ddeep, inv, B)
    gsum_wide = _scatter_rows(dwide.unsqueeze(2), inv, B).squeeze(2)
    grads = flatten((dwd, dW1, db1, dW2, db2, torch.cat([dw3, dwc]), dcw, dcb), G)

    # magnitude pass: the same sums over |operands| (masks of the float64 forward), products of k inexact
    # factors weighted k (module docstring); the cross terms follow the factors the tower multiplies:
    # a, c, e (first-layer contractions), beta, gamma (prologue), K = (1 + a)(1 + c) + beta
    aw = w.abs()
    X = x0.abs()
    W1a, W2a, w3a, wca, cwa, cba = W1.abs(), W2.abs(), w3.abs(), wc.abs(), cw.abs(), cb.abs()
    Mh1 = X @ W1a.t() + b1.abs()
    Ma1 = Mh1 * m1
    Mh2 = Ma1 @ W2a.t() + b2.abs()
    Ma2 = Mh2 * m2
    Ma, Mc, Me = X @ cwa[0], X @ cwa[1], X @ wca
    Mbeta, Mgamma = cba[0] @ cwa[1], wca @ (cba[0] + cba[1])
    MK = 2 * (1 + Ma) * (1 + Mc) + Mbeta
    Mz = wide.abs().sum(0) + dense.abs() @ wd.abs() + Ma2 @ w3a + 2 * MK * Me + Mgamma
    Ml2 = L2 * (cw * cw).sum()
    Mlb = Mz * (1 + y.abs()) + torch.log1p(torch.exp(-z.abs()))
    Mloss = (aw * Mlb).sum() / B + Ml2
    Mdz = (p * (1 - p) * Mz + p + y.abs() + P_FLOOR) / B * aw
    Mdw3 = Ma2.t() @ Mdz
    Mdh2 = Mdz.unsqueeze(1) * w3a * m2
    MdW2 = Mdh2.t() @ Ma1
    Mdb2 = Mdh2.sum(0)
    Mdh1 = (Mdh2 @ W2a) * m1
    MdW1 = Mdh1.t() @ X
    Mdb1 = Mdh1.sum(0)
    Mdwd = dense.abs().t() @ Mdz
    Mge = 2 * Mdz * Me  # g e
    Mda = 3 * Mdz * (1 + Mc) * Me  # g (1 + c) e
    Mdc = 3 * Mdz * (1 + Ma) * Me  # g (1 + a) e
    Mde = 2 * Mdz * MK  # g K
    Mdcw = torch.stack([X.t() @ Mda, X.t() @ Mdc + cba[0] * Mge.sum()]) + 2 * L2 * cwa
    Mdwc = X.t() @ Mde + (cba[0] + cba[1]) * Mdz.sum()
    Mdcb = torch.stack([cwa[1] * Mge.sum() + wca * Mdz.sum(), wca * Mdz.sum()])
    Mdx0 = Mdh1 @ W1a + Mda.unsqueeze(1) * cwa[0] + Mdc.unsqueeze(1) * cwa[1] + Mde.unsqueeze(1) * wca
    Mddeep = Mdx0[:, ND:].reshape(B, G, D).permute(1, 0, 2)
    M = {
        "logits": Mz, "loss": Mloss, "h1": Mh1, "h2": Mh2,
        "grads": flatten((Mdwd, MdW1, Mdb1, MdW2, Mdb2, torch.cat([Mdw3, Mdwc]), Mdcw, Mdcb), G),
        "gsum_deep": _scatter_rows(Mddeep, inv, B),
        "gsum_wide": _scatter_rows(Mdz.unsqueeze(0).expand(G, B).unsqueeze(2), inv, B).squeeze(2),
    }
    occ = _scatter_rows(torch.ones((G, B, 1), dtype=f64, device=dev), inv, B).squeeze(2)
    return {"logits": z, "loss": loss, "grads": grads, "gsum_wide": gsum_wide, "gsum_deep": gsum_deep,
            "h1": h1, "h2": h2, "x1": xs[1], "x2": xs[2], "M": M,
            "n_unique": n_unique.to(device=dev, dtype=torch.int64), "occ": occ}


def ratios(got, ref, families=FAMILIES, c=C_TOL, n_sm=132):
    """tower_oracle.ratios with the DCN chain lengths: per family (worst err / bound, where, got, want)."""
    G, B = ref["gsum_wide"].shape
    n = chain_lengths(G, B, n_sm)
    out = {}
    for fam in families:
        if fam not in got:
            continue
        want = ref[fam]
        g = torch.as_tensor(got[fam]).to(device=want.device, dtype=torch.float64).reshape(want.shape)
        m = ref["M"][fam]
        nn = torch.full_like(m, float(n[fam]))
        if fam.startswith("gsum"):
            occ = ref["occ"] if fam == "gsum_wide" else ref["occ"].unsqueeze(2)
            nn = nn + occ
        bound = c * torch.sqrt(nn) * EPS32 * m
        if fam.startswith("gsum"):  # one atomic add per occurrence at most
            bound = bound + FLT_MIN * (occ + 1)
        elif fam in ("grads", "loss"):  # a few atomic adds per CTA
            bound = bound + FLT_MIN * 8 * n_sm * 2
        err = (g - want).abs()
        r = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                        torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
        r = torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))
        if fam.startswith("gsum"):
            live = torch.arange(B, device=want.device).unsqueeze(0) < ref["n_unique"].unsqueeze(1)
            if fam == "gsum_deep":
                live = live.unsqueeze(2)
            r = torch.where(live, r, torch.zeros_like(r))
        if r.numel() == 0:
            out[fam] = (0.0, (), float("nan"), float("nan"))
            continue
        i = int(torch.argmax(r.reshape(-1)))
        where = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), r.shape)) if r.dim() else ()
        out[fam] = (float(r.reshape(-1)[i]), where, float(g.reshape(-1)[i]), float(want.reshape(-1)[i]))
    return out


def caught_by(got, ref, families=FAMILIES, c=C_TOL, n_sm=132):
    """The families in which got lies outside the bound somewhere."""
    return {fam for fam, (r, *_rest) in ratios(got, ref, families, c, n_sm).items() if not r <= 1.0}


def check(got, ref, families=FAMILIES, c=C_TOL, label="", n_sm=132):
    """Assert every family of got within the bound; returns {family: worst ratio}."""
    rs = ratios(got, ref, families, c, n_sm)
    bad = {f: v for f, v in rs.items() if not v[0] <= 1.0}
    if bad:
        lines = ["%s %s: err/bound %.3g at %s (got %r, want %r)" % (label, f, r, w, gv, wv)
                 for f, (r, w, gv, wv) in bad.items()]
        raise AssertionError("\n".join(lines))
    return {f: v[0] for f, v in rs.items()}


def mutations(ref, inputs, tile=32):
    """tower_oracle.mutations for the DCN reference: name -> outputs with one classic tiled-reduction fault."""
    G, B = ref["gsum_wide"].shape
    dev = ref["logits"].device
    keys = FAMILIES
    base = {k: ref[k] for k in keys}
    out = {}

    def weighted(wt):
        r = dcn_reference(*inputs, weight=wt)
        return {k: r[k] for k in keys}

    one = torch.ones(B, dtype=torch.float64, device=dev)
    drop = B // 2 + 7 if B > 64 else B // 2
    wt = one.clone()
    wt[drop] = 0
    out["drop_one_sample"] = weighted(wt)
    wt = one.clone()
    wt[B - 1] = 32
    out["last_sample_x32"] = weighted(wt)
    t = (B // tile) // 2
    wt = one.clone()
    wt[t * tile:(t + 1) * tile] = 0
    out["tile_missing_from_grads"] = dict(base, grads=weighted(wt)["grads"])
    gw, gd = ref["gsum_wide"].clone(), ref["gsum_deep"].clone()
    gw[G - 1, 0] = 0
    gd[G - 1, 0] = 0
    out["id_row_missing"] = dict(base, gsum_wide=gw, gsum_deep=gd)
    l2 = L2 * (unflatten(inputs[6], G)[6].to(torch.float64) ** 2).sum()
    out["loss_not_divided_by_B"] = dict(base, loss=(ref["loss"] - l2) * B + l2)
    return out
