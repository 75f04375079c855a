"""Float64 reference of the DeepFM tower (include/b200_deepfm.h) -- TEST INFRASTRUCTURE.

Plain torch float64, forward and backward written out by hand (no autograd), device-agnostic: the same
code runs on the CPU in the non-GPU tests and on the device next to the CUDA towers.  The inputs are the
kernel's own: inv [G, B], n_unique [G], the pulled rows bet_wide [G, B] / bet_deep [G, B, 8] (only the
first n_unique[g] rows of a group are read), dense [B, 13], labels [B] and the flat parameter buffer.

Besides the values, `tower_reference` runs a MAGNITUDE PASS: the same sums over the absolute value of
every operand, with the ReLU masks taken from the float64 forward.  M bounds the size of everything an
fp32 kernel adds up on the way to an output, so an fp32 result is expected within

    |got - ref| <= c * sqrt(n) * 2^-24 * M        (elementwise)

where n is the length of the longest fp32 accumulation chain behind that output (`chain_lengths`).
`ratios` / `check` apply that bound per output family.
"""
import math

import torch

from oracle import tf32 as _tf32

ND, D, H1, H2 = 13, 8, 16, 4
WD_PAD = 16
EPS32 = 2.0 ** -24
C_TOL = 8.0  # one constant for every tower
# p = sigmoid(z) underflows in fp32 below z ~ -88 (the kernels then return p = 0 instead of ~1e-39); this
# absolute floor of |p| keeps the bound of dz above that representable limit
P_FLOOR = 2.0 ** -100
# fp32 atomic adds to global memory flush subnormal operands and results to zero: every atomic add behind an
# output may lose up to the smallest normal number (saturated samples of a large-logit batch put dz ~ 1e-39
# into the per-id sums)
FLT_MIN = 2.0 ** -126
FAMILIES = ("logits", "loss", "grads", "gsum_wide", "gsum_deep")


def layout(G):
    """Offsets of the flat parameter buffer: [w_dense 13 (+3 pad) | w1 16 x (13 + 8G) | b1 16 | w2 4 x 16 | b2 4 | w3 4]."""
    n_in = ND + D * G
    o = {"in": n_in, "wd": 0, "w1": WD_PAD}
    o["b1"] = o["w1"] + H1 * n_in
    o["w2"] = o["b1"] + H1
    o["b2"] = o["w2"] + H2 * H1
    o["w3"] = o["b2"] + H2
    o["total"] = o["w3"] + H2
    return o


def unflatten(flat, G):
    """(wd [13], W1 [16, 13 + 8G], b1 [16], W2 [4, 16], b2 [4], w3 [4]) views of a flat buffer."""
    o = layout(G)
    return (flat[o["wd"]:o["wd"] + ND], flat[o["w1"]:o["b1"]].view(H1, o["in"]), flat[o["b1"]:o["b1"] + H1],
            flat[o["w2"]:o["b2"]].view(H2, H1), flat[o["b2"]:o["b2"] + H2], flat[o["w3"]:o["w3"] + H2])


def flatten(parts, G, pad=0.0):
    """Inverse of unflatten; the 3 padding floats after w_dense are set to `pad`."""
    wd, w1, b1, w2, b2, w3 = parts
    o = layout(G)
    flat = torch.full((o["total"],), pad, dtype=wd.dtype, device=wd.device)
    flat[o["wd"]:o["wd"] + ND] = wd.reshape(-1)
    flat[o["w1"]:o["b1"]] = w1.reshape(-1)
    flat[o["b1"]:o["b1"] + H1] = b1.reshape(-1)
    flat[o["w2"]:o["b2"]] = w2.reshape(-1)
    flat[o["b2"]:o["b2"] + H2] = b2.reshape(-1)
    flat[o["w3"]:o["w3"] + H2] = w3.reshape(-1)
    return flat


def random_params(G, gen, device, w1_gain=2.0, b1=None, b2=None, wd_std=0.3, pad=0.0):
    """A float32 flat parameter buffer with every part O(1)-relevant: W1 ~ N(0, (w1_gain^2 / IN)),
    b1 ~ U(-0.3, 0.3) (some hidden units dead for part of the batch), W2 / b2 ~ U(-0.5, 0.5), w3 ~ U(-1, 1),
    w_dense ~ N(0, wd_std^2).  b1 / b2 given as numbers: constant biases."""
    n_in = ND + D * G

    def u(shape, a):
        return (torch.rand(shape, generator=gen, device=device) * 2 - 1) * a

    wd = torch.randn(ND, generator=gen, device=device) * wd_std
    w1 = torch.randn((H1, n_in), generator=gen, device=device) * (w1_gain / math.sqrt(n_in))
    bb1 = u(H1, 0.3) if b1 is None else torch.full((H1,), float(b1), device=device)
    w2 = u((H2, H1), 0.5)
    bb2 = u(H2, 0.5) if b2 is None else torch.as_tensor(b2, dtype=torch.float32, device=device).expand(H2).clone()
    w3 = u(H2, 1.0)
    return flatten((wd, w1, bb1, w2, bb2, w3), G, pad=pad)


def first_occurrence_inverse(ids):
    """ids [G, B] (or [B]) -> (inv int32 [G, B], n_unique int32 [G], uniq int64 [G, B]): tf.unique per group,
    unique ids in order of first occurrence (uniq[g, n_unique[g]:] = -1), inv[g, b] = rank of ids[g, b]."""
    ids = torch.as_tensor(ids)
    one = ids.dim() == 1
    ids2 = ids.reshape(-1, ids.shape[-1]).to(torch.int64)
    G, B = ids2.shape
    dev = ids2.device
    inv = torch.empty((G, B), dtype=torch.int32, device=dev)
    uniq = torch.full((G, B), -1, dtype=torch.int64, device=dev)
    n_unique = torch.empty(G, dtype=torch.int32, device=dev)
    pos = torch.arange(B, device=dev)
    for g in range(G):
        u, iv = torch.unique(ids2[g], sorted=True, return_inverse=True)
        first = torch.full((u.numel(),), B, dtype=torch.int64, device=dev).scatter_reduce_(0, iv, pos, "amin")
        order = torch.argsort(first)
        rank = torch.empty_like(order)
        rank[order] = torch.arange(u.numel(), device=dev)
        inv[g] = rank[iv].to(torch.int32)
        uniq[g, :u.numel()] = u[order]
        n_unique[g] = u.numel()
    if one:
        return inv[0], n_unique[0], uniq[0]
    return inv, n_unique, uniq


def chain_lengths(G, B, n_sm=132):
    """Longest fp32 accumulation chain behind each output family (the per-row part of gsum is added by
    `ratios`: the occurrences of the id).  Forward: the first-layer dot product (13 + 8G inputs + bias),
    then the 16 -> 4 -> 1 tail and the final sum; backward to the embedding rows: 4 + 16 more terms.
    The loss and the parameter gradients sum over the batch, but no tower adds all B samples in one chain:
    each CTA keeps a running sum over its own tiles (at most ceil(B / 32 / n_sm) tiles of 32 when there is
    one CTA per SM -- twice a CTA's even share at two per SM, room for the dynamic tile counter), and the
    partial sums of at most 8 * n_sm CTAs meet in fp32 atomics.  The chain is the sum of the two."""
    fwd = ND + D * G + 32
    bwd = fwd + 32
    per_cta = 32 * -(-(-(-B // 32)) // n_sm)
    nb = min(B, per_cta + 8 * n_sm)
    return {"logits": fwd, "loss": fwd + nb, "grads": bwd + nb, "gsum_wide": bwd, "gsum_deep": bwd}


def _scatter_rows(occ, inv, n_rows):
    """occ [G, B, k] per-occurrence values -> [G, n_rows, k] summed per rank inv[g, b]."""
    G, B, k = occ.shape
    out = torch.zeros((G * n_rows, k), dtype=occ.dtype, device=occ.device)
    idx = (inv.long() + torch.arange(G, device=occ.device).unsqueeze(1) * n_rows).reshape(-1)
    out.index_add_(0, idx, occ.reshape(G * B, k))
    return out.view(G, n_rows, k)


def tower_reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params, weight=None, contraction=None,
                    dnn_masks=None):
    """Float64 forward + backward of one batch.  weight [B] (optional): a multiplicity per sample in every
    reduction (loss, parameter gradients, per-id sums) -- 1 everywhere is the real tower; the comparator
    tests use 0 / 32 to model a dropped / replayed sample.

    contraction (oracle/tf32.py modes): the first layer's three contractions evaluated with the TF32 products of
    a mode, with the operands the mma tower (csrc/deepfm_tower_mma.cu) splits: "forward" H = [x | 1] [W1 | b1]^T,
    "data" dX = dH1 W1[:, deep columns], "weight" [dW1 | db1] = dH1^T [x | 1].  dnn_masks (m1 [B, 16], m2 [B, 4]
    bool): the ReLU masks to use instead of h > 0 (an emulated run takes the exact run's, so that its error does
    not flip a unit).  The magnitudes are those of the exact run's operands either way.

    Returns a dict of float64 tensors on the inputs' device:
      logits [B], loss [], grads [P] (flat layout, padding 0), gsum_wide [G, B], gsum_deep [G, B, 8]
      (rows >= n_unique[g] are 0), h1 [B, 16] / h2 [B, 4] (pre-activations of the hidden layers),
      "M": the magnitude of every one of those, "n_unique", "occ" [G, B] (occurrences per rank)."""
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
    cm = _tf32.modes(contraction)
    one = torch.ones((B, 1), dtype=f64, device=dev)

    # forward (workloads.deepfm.DeepFMTower): x = [dense | deep of group 0 | ... | deep of group G-1]
    x = torch.cat([dense, deep.permute(1, 0, 2).reshape(B, G * D)], 1)
    if cm["forward"] == "fp32":
        h1 = x @ W1.t() + b1
    else:  # the bias is the tile's constant column
        h1 = _tf32.contract(torch.cat([x, one], 1), torch.cat([W1, b1.unsqueeze(1)], 1).t(), cm["forward"])
    m1 = (h1 > 0 if dnn_masks is None else dnn_masks[0]).to(f64)
    a1 = h1 * m1
    h2 = a1 @ W2.t() + b2
    m2 = (h2 > 0 if dnn_masks is None else dnn_masks[1]).to(f64)
    a2 = h2 * m2
    dnn = a2 @ w3
    s = deep.sum(0)  # [B, 8]
    q = (deep * deep).sum((0, 2))
    fm = 0.5 * ((s * s).sum(1) - q)
    lin = wide.sum(0) + dense @ wd
    z = lin + dnn + fm
    lb = z.clamp_min(0) - z * y + torch.log1p(torch.exp(-z.abs()))  # BCE with logits
    loss = (w * lb).sum() / B

    # backward
    p = torch.sigmoid(z)
    dz = (p - y) / B * w
    dw3 = a2.t() @ dz
    dh2 = dz.unsqueeze(1) * w3 * m2
    dW2 = dh2.t() @ a1
    db2 = dh2.sum(0)
    dh1 = (dh2 @ W2) * m1
    if cm["weight"] == "fp32":
        dW1 = dh1.t() @ x
        db1 = dh1.sum(0)
    else:
        dW1b = _tf32.contract(dh1.t(), torch.cat([x, one], 1), cm["weight"])
        dW1, db1 = dW1b[:, :-1], dW1b[:, -1]
    dwd = dense.t() @ dz
    dx = dh1 @ W1 if cm["data"] == "fp32" else _tf32.contract(dh1, W1, cm["data"])
    ddeep = dx[:, ND:].reshape(B, G, D).permute(1, 0, 2) + dz.view(1, B, 1) * (s.unsqueeze(0) - deep)
    dwide = dz.unsqueeze(0).expand(G, B)
    gsum_deep = _scatter_rows(ddeep, inv, B)
    gsum_wide = _scatter_rows(dwide.unsqueeze(2), inv, B).squeeze(2)
    grads = flatten((dwd, dW1, db1, dW2, db2, dw3), G)

    # magnitude pass: the same sums over |operands|, masks of the float64 forward
    aw = w.abs()
    X = x.abs()
    W1a, W2a, w3a = W1.abs(), W2.abs(), w3.abs()
    Mh1 = X @ W1a.t() + b1.abs()
    Ma1 = Mh1 * m1
    Mh2 = Ma1 @ W2a.t() + b2.abs()
    Ma2 = Mh2 * m2
    Ms = deep.abs().sum(0)
    Mz = wide.abs().sum(0) + dense.abs() @ wd.abs() + Ma2 @ w3a + 0.5 * ((Ms * Ms).sum(1) + q)
    # an error e in z moves the sample's loss by |p - y| e <= (1 + |y|) e and p by p (1 - p) e
    Mlb = Mz * (1 + y.abs()) + torch.log1p(torch.exp(-z.abs()))
    Mloss = (aw * Mlb).sum() / B
    Mdz = (p * (1 - p) * Mz + p + y.abs() + P_FLOOR) / B * aw
    Mdw3 = Ma2.t() @ Mdz
    Mdh2 = Mdz.unsqueeze(1) * w3a * m2
    MdW2 = Mdh2.t() @ Ma1
    Mdb2 = Mdh2.sum(0)
    Mdh1 = (Mdh2 @ W2a) * m1
    MdW1 = Mdh1.t() @ X
    Mdb1 = Mdh1.sum(0)
    Mdwd = dense.abs().t() @ Mdz
    Mdx = Mdh1 @ W1a
    Mddeep = Mdx[:, ND:].reshape(B, G, D).permute(1, 0, 2) + Mdz.view(1, B, 1) * (Ms.unsqueeze(0) + deep.abs())
    M = {
        "logits": Mz, "loss": Mloss, "h1": Mh1, "h2": Mh2,
        "grads": flatten((Mdwd, MdW1, Mdb1, MdW2, Mdb2, Mdw3), G),
        "gsum_deep": _scatter_rows(Mddeep, inv, B),
        "gsum_wide": _scatter_rows(Mdz.unsqueeze(0).expand(G, B).unsqueeze(2), inv, B).squeeze(2),
    }
    occ = _scatter_rows(torch.ones((G, B, 1), dtype=f64, device=dev), inv, B).squeeze(2)
    return {"logits": z, "loss": loss, "grads": grads, "gsum_wide": gsum_wide, "gsum_deep": gsum_deep,
            "h1": h1, "h2": h2, "M": M, "n_unique": n_unique.to(device=dev, dtype=torch.int64), "occ": occ}


PRECISION_CHECKS = ("forward", "data", "weight")


def precision_selection(ref, check):
    """(family, selection) for tf32.ratio: the elements the mma tower's first-layer contraction `check` feeds --
    the logits, the live rows of gsum_deep, dW1 and db1."""
    if check == "forward":
        return "logits", None
    if check == "data":
        return "gsum_deep", _tf32.live_rows(ref, "gsum_deep")
    o = layout(ref["gsum_wide"].shape[0])
    return "grads", slice(o["w1"], o["b1"] + H1)


def near_relu_kink(ref, tau=1e-4):
    """[B] bool: samples whose float64 layer-1 or layer-2 pre-activation lies within tau * M of 0 -- their
    ReLU mask may come out differently in fp32, which moves the backward by far more than rounding."""
    M = ref["M"]
    return (ref["h1"].abs() <= tau * M["h1"]).any(1) | (ref["h2"].abs() <= tau * M["h2"]).any(1)


def ratios(got, ref, families=FAMILIES, c=C_TOL, n_sm=132):
    """Per family: (worst err / bound, where, got, want).  got: dict family -> tensor (any float dtype, any
    device); a NaN or inf in got counts as an infinite ratio.  gsum rows >= n_unique[g] are not compared."""
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
        elif fam in ("grads", "loss"):  # one atomic add per CTA
            bound = bound + FLT_MIN * 8 * n_sm
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
    """Assert every family of got within the bound; the message names the worst element of each failure.
    Returns {family: worst ratio}."""
    rs = ratios(got, ref, families, c, n_sm)
    bad = {f: v for f, v in rs.items() if not v[0] <= 1.0}
    if bad:
        lines = ["%s %s: err/bound %.3g at %s (got %r, want %r)" % (label, f, r, w, gv, wv)
                 for f, (r, w, gv, wv) in bad.items()]
        raise AssertionError("\n".join(lines))
    return {f: v[0] for f, v in rs.items()}


def mutations(ref, inputs, tile=32):
    """The reference's outputs with one classic tiled-reduction fault each: name -> dict of outputs.
    inputs: the tuple tower_reference took (inv, n_unique, bet_wide, bet_deep, dense, labels, params)."""
    G, B = ref["gsum_wide"].shape
    dev = ref["logits"].device
    keys = ("logits", "loss", "grads", "gsum_wide", "gsum_deep")
    base = {k: ref[k] for k in keys}
    out = {}

    def weighted(wt):
        r = tower_reference(*inputs, weight=wt)
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
