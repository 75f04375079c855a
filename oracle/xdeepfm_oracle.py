"""Float64 reference of the xDeepFM tower (include/b200_deepfm.h, b200_deepfm_xdeepfm_*) -- TEST INFRASTRUCTURE.

xDeepFM is Wide & Deep plus a Compressed Interaction Network (workloads.deepfm.XDeepFMTower):
    logit = sum(wide) + w_dense . dense + w3 . relu(W2 relu(W1 [dense | deep] + b1) + b2) + w_ex . p + b_ex,
    loss  = mean BCE + 1e-5 (|W_0|^2 + |W_1|^2).
The CIN runs deepctr's literal recursion, not the kernels' factorization: per layer k the outer product
Z_k[b, d, i, j] = X0[b, i, d] X_k[b, j, d], the reshape to K = i H_k + j, the filter contraction with bias and ReLU,
split-half after layer 0 and the sum over d of the direct channels.  Forward and backward are written out by hand
and run over batch chunks (in float64 at B = 32768, Z_0 and Z_1 of the whole batch would be 3 and 5 GB).

The bound is tower_oracle's, |got - ref| <= c sqrt(n) 2^-24 M, with the magnitude pass extended through the CIN and
the chain lengths of its K-long sums (`chain_lengths`).  Layer 1's input magnitude is |X_1| itself, not layer 0's
magnitude carried through: with K = G^2 and 64 G terms of random sign, carrying sums of absolute values through two
layers makes M thousands of times the logit and hides every fault under the bound; layer 0's own rounding enters
through the chain length instead.  The exception is dW_1, a sum over the batch: samples that share their rows share
layer 0's rounding of X_1, which then adds up coherently, so its magnitude carries layer 0's. `ratios` takes a chain length per element, since the
CIN's filter gradients are reduced over many more samples per CTA than the DNN's.  ReLU kinks of the CIN cannot be
moved away by redrawing a sample's dense row (its units depend on the shared deep rows only), so the reference
takes an optional mask override, used only where |pre| <= tau M_pre: a test feeds it the kernel's mask bits there.
"""
import math

import torch

from oracle.tower_oracle import (  # noqa: F401  (re-exported: the tests use this module as the tower's oracle)
    C_TOL, D, EPS32, FAMILIES, FLT_MIN, H1, H2, ND, P_FLOOR, WD_PAD, _scatter_rows, first_occurrence_inverse,
    near_relu_kink)
from oracle import tf32 as _tf32
from oracle import tower_oracle as _T

CIN_H, HALF, NP = 128, 64, 192
L2 = 1e-5


def layout(G):
    """Offsets of the flat buffer: Wide & Deep's (tower_oracle.layout) then W_0 128 x G^2 | b_0 | W_1 128 x 64G | b_1 |
    w_ex 192 | b_ex."""
    o = dict(_T.layout(G))
    o["cin_w0"] = o["total"]
    o["cin_b0"] = o["cin_w0"] + CIN_H * G * G
    o["cin_w1"] = o["cin_b0"] + CIN_H
    o["cin_b1"] = o["cin_w1"] + CIN_H * HALF * G
    o["wex"] = o["cin_b1"] + CIN_H
    o["bex"] = o["wex"] + NP
    o["total"] = o["bex"] + 1
    return o


def unflatten(flat, G):
    """(Wide & Deep's six parts, W_0 [128, G^2], b_0, W_1 [128, 64G], b_1, w_ex [192], b_ex [1])."""
    o = layout(G)
    wd = _T.unflatten(flat[:o["cin_w0"]], G)
    return wd + (flat[o["cin_w0"]:o["cin_b0"]].view(CIN_H, G * G), flat[o["cin_b0"]:o["cin_w1"]],
                 flat[o["cin_w1"]:o["cin_b1"]].view(CIN_H, HALF * G), flat[o["cin_b1"]:o["wex"]],
                 flat[o["wex"]:o["bex"]], flat[o["bex"]:o["total"]])


def flatten(parts, G, pad=0.0):
    o = layout(G)
    wd = _T.flatten(parts[:6], G, pad)
    flat = torch.full((o["total"],), pad, dtype=wd.dtype, device=wd.device)
    flat[:o["cin_w0"]] = wd
    for k, p in zip(("cin_w0", "cin_b0", "cin_w1", "cin_b1", "wex", "bex"), parts[6:]):
        flat[o[k]:o[k] + p.numel()] = p.reshape(-1)
    return flat


def random_params(G, gen, device, pad=0.0, cin_gain=1.0, **kw):
    """tower_oracle.random_params for the Wide & Deep part; the CIN glorot-uniform as the model initializes it
    (times cin_gain), its biases U(-0.1, 0.1) and w_ex glorot-uniform over (192, 1) times 4, so that the CIN logit
    moves the logit as much as the rest of it does."""
    wdp = _T.random_params(G, gen, device, pad=pad, **kw)
    o = layout(G)

    def u(shape, a):
        return (torch.rand(shape, generator=gen, device=device) * 2 - 1) * a

    parts = _T.unflatten(wdp, G) + (
        u((CIN_H, G * G), cin_gain * math.sqrt(6.0 / (G * G + CIN_H))), u(CIN_H, 0.1),
        u((CIN_H, HALF * G), cin_gain * math.sqrt(6.0 / (HALF * G + CIN_H))), u(CIN_H, 0.1),
        u(NP, 4 * math.sqrt(6.0 / (NP + 1))), u(1, 0.1))
    flat = flatten(parts, G, pad)
    assert flat.numel() == o["total"]
    return flat


def _outer(x0, xk, k_order):
    """Z [n, D, H0 * Hk]: deepctr's matmul of X0 against X_k, then the reshape (K = i Hk + j; "ji": K = j H0 + i)."""
    n = x0.shape[0]
    z = torch.einsum("bid,bjd->bdij" if k_order == "ij" else "bid,bjd->bdji", x0, xk)
    return z.reshape(n, x0.shape[2], -1)


def _split_back(dz, n, H0, Hk, k_order):
    """dZ [n, D, K] -> [n, D, H0, Hk] (the inverse of _outer's reshape)."""
    if k_order == "ij":
        return dz.reshape(n, D, H0, Hk)
    return dz.reshape(n, D, Hk, H0).transpose(2, 3)


def _cin_forward(x0, W, mask_override, k_order, swap_halves, magnitudes, cm=None):
    """One chunk: x0 [n, G, D] -> dict with p [n, 192], pre0 / pre1 [n, 128, D], masks, x1 and (magnitudes) their
    magnitudes.  cm: tf32.modes; the forward contraction's operands are k_cin_fwd's, A = W_k and B = Z_k formed
    as the fp32 product X0 X_k."""
    fwd = _tf32.modes(cm)["forward"]
    W0, b0, W1, b1 = W
    n, G, _ = x0.shape
    out = {}
    xk, mxk = x0, x0.abs()
    direct, mdirect = [], []
    for k, (w, b) in enumerate(((W0, b0), (W1, b1))):
        z = _outer(x0, xk, k_order)
        if fwd == "fp32":
            pre = (z @ w.t() + b).transpose(1, 2)  # [n, 128, D]
        else:
            pre = _tf32.contract(w, z, fwd, eq="hk,bdk->bhd") + b.view(1, -1, 1)
        mpre = None
        if magnitudes or mask_override is not None:
            mpre = (_outer(x0.abs(), mxk, k_order) @ w.abs().t() + b.abs()).transpose(1, 2)
        m = pre > 0
        if mask_override is not None:
            mo, tau = mask_override[k], mask_override[2]
            near = pre.abs() <= tau * mpre
            m = torch.where(near, mo, m)
        m = m.to(pre.dtype)
        c = pre * m
        out["pre%d" % k], out["m%d" % k], out["mpre%d" % k] = pre, m, mpre
        mc = mpre * m if magnitudes else None
        if k == 0:
            lo, hi = (slice(HALF, None), slice(None, HALF)) if swap_halves else (slice(None, HALF), slice(HALF, None))
            xk, c = c[:, lo], c[:, hi]
            out["x1"] = xk
            mxk = xk.abs()
            if magnitudes:
                out["mx1_carried"] = mc[:, lo]
                mc = mc[:, hi]
                out["mx1"] = mxk
        direct.append(c)
        mdirect.append(mc)
    out["p"] = torch.cat(direct, 1).sum(2)
    if magnitudes:
        out["mp"] = torch.cat(mdirect, 1).sum(2)
    return out


def _cin_backward(x0, f, dz, W, wex, k_order, swap_halves, cm=None):
    """One chunk: d loss / d (x0, W_0, b_0, W_1, b_1) from the forward record f and dz [n] (already weighted).
    cm: tf32.modes, with the operands of csrc/xdeepfm_cin.cu.  Data pass (k_cin_data): A = W_k^T with the direct
    channels' rows scaled by their w_ex, B = mask ? dz : 0 (direct channels) or dC_0 (X_1's channels).  Weight
    pass (k_cin_weights): A = dC_0 and B = Z_0 for X_1's channels; else A = the 0/1 mask (exact) and B = dz Z_k,
    the output scaled by w_ex."""
    data, wgt = (_tf32.modes(cm)[k] for k in ("data", "weight"))
    f32 = _tf32.fp32
    W0, b0, W1, b1 = W
    n, G, _ = x0.shape
    x1 = f["x1"]
    lo, hi = (slice(HALF, None), slice(None, HALF)) if swap_halves else (slice(None, HALF), slice(HALF, None))
    dc1 = dz.view(n, 1, 1) * wex[HALF:].view(1, CIN_H, 1) * f["m1"]
    z1 = _outer(x0, f.get("x1_batch", x1), k_order)
    if wgt == "fp32":
        dW1 = torch.einsum("bhd,bdk->hk", dc1, z1)
    else:
        dW1 = _tf32.contract(f["m1"], f32(dz.view(n, 1, 1) * f32(z1)), wgt, eq="bhd,bdk->hk") * wex[HALF:].view(-1, 1)
    db1 = dc1.sum((0, 2))
    if data == "fp32":
        dZ1 = torch.einsum("bhd,hk->bdk", dc1, W1)
    else:
        dZ1 = _tf32.contract((W1 * wex[HALF:].view(-1, 1)).t(), dz.view(n, 1, 1) * f["m1"], data, eq="kh,bhd->bdk")
    dZ1 = _split_back(dZ1, n, G, HALF, k_order)  # [n, D, G, 64]
    dx0 = torch.einsum("bdij,bjd->bid", dZ1, x1)
    dx1 = torch.einsum("bdij,bid->bjd", dZ1, x0)
    dc0 = torch.zeros((n, CIN_H, D), dtype=x0.dtype, device=x0.device)
    dc0[:, lo] = dx1
    dc0[:, hi] = dz.view(n, 1, 1) * wex[:HALF].view(1, HALF, 1)
    dc0 = dc0 * f["m0"]
    z0 = _outer(x0, x0, k_order)
    if wgt == "fp32":
        dW0 = torch.einsum("bhd,bdk->hk", dc0, z0)
    else:
        dW0 = torch.empty_like(W0)
        dW0[lo] = _tf32.contract(dc0[:, lo], z0, wgt, eq="bhd,bdk->hk")
        dW0[hi] = _tf32.contract(f["m0"][:, hi], f32(dz.view(n, 1, 1) * f32(z0)), wgt,
                                 eq="bhd,bdk->hk") * wex[:HALF].view(-1, 1)
    db0 = dc0.sum((0, 2))
    if data == "fp32":
        dZ0 = torch.einsum("bhd,hk->bdk", dc0, W0)
    else:
        scale = torch.ones(CIN_H, dtype=W0.dtype, device=W0.device)
        scale[hi] = wex[:HALF]
        b_op = dz.view(n, 1, 1) * f["m0"]
        b_op[:, lo] = dc0[:, lo]
        dZ0 = _tf32.contract((W0 * scale.view(-1, 1)).t(), b_op, data, eq="kh,bhd->bdk")
    dZ0 = _split_back(dZ0, n, G, G, k_order)
    dx0 = dx0 + torch.einsum("bdij,bjd->bid", dZ0, x0) + torch.einsum("bdij,bid->bjd", dZ0, x0)
    return dx0, dW0, db0, dW1, db1


def xdeepfm_reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params, weight=None, mask_override=None,
                      norm=None, l2=True, magnitudes=True, k_order="ij", swap_halves=False, chunk=1024,
                      contraction=None):
    """Float64 forward + backward of one batch, with the inputs, the optional per-sample weight and the outputs of
    tower_oracle.tower_reference (logits, loss, grads, gsum_wide, gsum_deep, h1, h2, "M", n_unique, occ) plus the
    CIN's pre-activations pre0 / pre1 [B, 128, 8] and their magnitudes (M["pre0"], M["pre1"]), p [B, 192] and the
    CIN logit "cin" [B].
    mask_override (m0, m1, tau): bool [B, 128, 8] masks used where |pre| <= tau M_pre.  norm: the batch size the
    loss divides by (default B; a subset of a batch with the full batch's norm gives that subset's share of every
    output, which is how `mutations` models a sample counted differently); l2=False leaves the L2 term out.
    k_order="ji" and swap_halves are mutations (the K index transposed, the split halves swapped).
    contraction (oracle/tf32.py modes for "forward", "data", "weight"): the CIN's three tensor-core contractions
    evaluated with the TF32 products of a mode, on the operands the kernels split (_cin_forward, _cin_backward).
    An emulated run should take the exact run's masks (mask_override with tau = 1), so that its error does not
    flip a unit.  The magnitude pass is the exact one's."""
    f64 = torch.float64
    G, B = inv.shape
    Bn = B if norm is None else norm
    NR = bet_wide.shape[-1]
    dev = inv.device
    inv_l = inv.long()
    wide = torch.gather(bet_wide.reshape(G, NR), 1, inv_l).to(f64)
    deep = torch.gather(bet_deep.reshape(G, NR, D), 1, inv_l.unsqueeze(2).expand(G, B, D)).to(f64)
    dense = dense.to(f64)
    y = labels.to(f64)
    parts = [t.to(f64) for t in unflatten(params, G)]
    wd, W1, b1, W2, b2, w3 = parts[:6]
    Wc = parts[6:10]
    wex, bex = parts[10], parts[11]
    w = torch.ones(B, dtype=f64, device=dev) if weight is None else weight.to(f64)
    x0_all = deep.permute(1, 0, 2)  # [B, G, D]

    # Wide & Deep forward (oracle/wide_deep_oracle.py)
    x = torch.cat([dense, x0_all.reshape(B, G * D)], 1)
    h1 = x @ W1.t() + b1
    m1 = (h1 > 0).to(f64)
    a1 = h1 * m1
    h2 = a1 @ W2.t() + b2
    m2 = (h2 > 0).to(f64)
    a2 = h2 * m2
    z_wd = wide.sum(0) + dense @ wd + a2 @ w3

    # CIN forward, chunk by chunk
    recs = []
    for s0 in range(0, B, chunk):
        mo = None
        if mask_override is not None:
            mo = (mask_override[0][s0:s0 + chunk], mask_override[1][s0:s0 + chunk], mask_override[2])
        recs.append(_cin_forward(x0_all[s0:s0 + chunk], Wc, mo, k_order, swap_halves, magnitudes, contraction))
    p = torch.cat([r["p"] for r in recs])
    cin = p @ wex + bex[0]
    z = z_wd + cin
    lb = z.clamp_min(0) - z * y + torch.log1p(torch.exp(-z.abs()))
    reg = L2 * ((Wc[0] * Wc[0]).sum() + (Wc[2] * Wc[2]).sum())
    loss = (w * lb).sum() / Bn + (reg if l2 else 0.0)

    # backward
    pr = torch.sigmoid(z)
    dz = (pr - y) / Bn * w
    dh2 = dz.unsqueeze(1) * w3 * m2
    dh1 = (dh2 @ W2) * m1
    ddeep = (dh1 @ W1)[:, ND:].reshape(B, G, D)
    grads_cin = [torch.zeros_like(t) for t in Wc]
    for k, s0 in enumerate(range(0, B, chunk)):
        g = _cin_backward(x0_all[s0:s0 + chunk], recs[k], dz[s0:s0 + chunk], Wc, wex, k_order, swap_halves,
                          contraction)
        ddeep[s0:s0 + chunk] += g[0]
        for acc, v in zip(grads_cin, g[1:]):
            acc += v
    if l2:
        grads_cin[0] += 2 * L2 * Wc[0]
        grads_cin[2] += 2 * L2 * Wc[2]
    grads = flatten((dense.t() @ dz, dh1.t() @ x, dh1.sum(0), dh2.t() @ a1, dh2.sum(0), a2.t() @ dz,
                     *grads_cin, p.t() @ dz, dz.sum().reshape(1)), G)
    occ = _scatter_rows(torch.ones((G, B, 1), dtype=f64, device=dev), inv, NR).squeeze(2)
    out = {"logits": z, "loss": loss, "grads": grads,
           "gsum_wide": _scatter_rows(dz.unsqueeze(0).expand(G, B).unsqueeze(2), inv, NR).squeeze(2),
           "gsum_deep": _scatter_rows(ddeep.permute(1, 0, 2), inv, NR),
           "h1": h1, "h2": h2, "pre0": torch.cat([r["pre0"] for r in recs]),
           "pre1": torch.cat([r["pre1"] for r in recs]), "p": p, "cin": cin,
           "n_unique": n_unique.to(device=dev, dtype=torch.int64), "occ": occ}
    if not magnitudes:
        return out

    # magnitude pass: the same sums over |operands|, masks of the float64 forward
    aw = w.abs()
    X = x.abs()
    W1a, W2a, w3a = W1.abs(), W2.abs(), w3.abs()
    Wca = [t.abs() for t in Wc]
    Mh1 = X @ W1a.t() + b1.abs()
    Ma1 = Mh1 * m1
    Mh2 = Ma1 @ W2a.t() + b2.abs()
    Ma2 = Mh2 * m2
    Mp = torch.cat([r["mp"] for r in recs])
    Mz = wide.abs().sum(0) + dense.abs() @ wd.abs() + Ma2 @ w3a + Mp @ wex.abs() + bex.abs()[0]
    Mlb = Mz * (1 + y.abs()) + torch.log1p(torch.exp(-z.abs()))
    Mreg = L2 * ((Wc[0] * Wc[0]).sum() + (Wc[2] * Wc[2]).sum())
    Mdz = (pr * (1 - pr) * Mz + pr + y.abs() + P_FLOOR) / Bn * aw
    Mdh2 = Mdz.unsqueeze(1) * w3a * m2
    Mdh1 = (Mdh2 @ W2a) * m1
    Mddeep = (Mdh1 @ W1a)[:, ND:].reshape(B, G, D)
    Mg_cin = [torch.zeros_like(t) for t in Wc]
    for k, s0 in enumerate(range(0, B, chunk)):
        r = recs[k]
        mrec = {"x1": r["mx1"], "x1_batch": r["mx1_carried"], "m0": r["m0"], "m1": r["m1"]}
        g = _cin_backward(x0_all[s0:s0 + chunk].abs(), mrec, Mdz[s0:s0 + chunk], Wca, wex.abs(), k_order,
                          swap_halves)
        Mddeep[s0:s0 + chunk] += g[0]
        for acc, v in zip(Mg_cin, g[1:]):
            acc += v
    Mg_cin[0] += 2 * L2 * Wca[0]
    Mg_cin[2] += 2 * L2 * Wca[2]
    out["M"] = {
        "logits": Mz, "loss": (aw * Mlb).sum() / Bn + Mreg, "h1": Mh1, "h2": Mh2,
        "pre0": torch.cat([r["mpre0"] for r in recs]), "pre1": torch.cat([r["mpre1"] for r in recs]),
        "grads": flatten((dense.abs().t() @ Mdz, Mdh1.t() @ X, Mdh1.sum(0), Mdh2.t() @ Ma1, Mdh2.sum(0),
                          Ma2.t() @ Mdz, *Mg_cin, Mp.t() @ Mdz, Mdz.sum().reshape(1)), G),
        "gsum_deep": _scatter_rows(Mddeep.permute(1, 0, 2), inv, NR),
        "gsum_wide": _scatter_rows(Mdz.unsqueeze(0).expand(G, B).unsqueeze(2), inv, NR).squeeze(2),
    }
    return out


# The elements each CIN contraction feeds, as (family, selection) for tf32.ratio.  The weight pass is two checks:
# W_0's X_1 channels take A = dC_0 through all three products, every other filter row takes A = the exact 0/1 mask
# and two products (there a lost lo of A changes nothing, so "2x_no_a_lo" is the kernel itself).
PRECISION_CHECKS = ("forward", "data", "weight_dc0", "weight_mask")
CONTRACTION_OF = {"forward": "forward", "data": "data", "weight_dc0": "weight", "weight_mask": "weight"}


def precision_selection(ref, check):
    """(family, selection) of PRECISION_CHECKS' `check` for tf32.ratio."""
    G = ref["gsum_wide"].shape[0]
    o = layout(G)
    if check == "forward":
        return "logits", None
    if check == "data":
        return "gsum_deep", _tf32.live_rows(ref, "gsum_deep")
    sel = torch.zeros(o["total"], dtype=torch.bool, device=ref["grads"].device)
    dc0 = slice(o["cin_w0"], o["cin_w0"] + HALF * G * G)
    if check == "weight_dc0":
        sel[dc0] = True
    else:
        sel[dc0.stop:o["cin_b0"]] = True
        sel[o["cin_w1"]:o["cin_b1"]] = True
    return "grads", sel


def near_cin_kink(ref, tau=1e-4):
    """(near0, near1): bool [B, 128, 8], the CIN pre-activations within tau * M of 0."""
    return tuple(ref["pre%d" % k].abs() <= tau * ref["M"]["pre%d" % k] for k in (0, 1))


def decode_masks(words):
    """The kernels' ReLU mask bits, int32 [B, 64] (32 words per layer), as (m0, m1) bool [B, 128, 8]: word
    4 (h / 16) + 2 ((h / 8) % 2) + d % 2, bit 4 (h % 8) + d / 2."""
    w = words.to(torch.int64) & 0xffffffff
    h = torch.arange(CIN_H, device=w.device).view(CIN_H, 1)
    d = torch.arange(D, device=w.device).view(1, D)
    word = (h // 16) * 4 + ((h // 8) % 2) * 2 + d % 2
    bit = (h % 8) * 4 + d // 2
    return tuple(((w[:, 32 * k + word] >> bit) & 1).bool() for k in (0, 1))


def chain_lengths(G, B, n_sm=132):
    """tower_oracle.chain_lengths with the CIN's sums: the logit adds the CIN's two K-long contractions (G Hp0 and
    64 G, Hp0 = G rounded up to 8; the second's input carries the first's error) and its 192-long output sum; a row
    gradient adds the data pass's
    128-long channel sums and its contractions over i and j; the CIN's parameter gradients are reduced over the
    8 x 32 columns of each of a CTA's tiles (the weight pass splits the batch over ~4 n_sm / 31 CTAs per output
    tile) and across those CTAs.  "grads" is a tensor over the flat layout."""
    base = _T.chain_lengths(G, B, n_sm)
    hp0 = -(-G // 8) * 8
    cin_f = G * hp0 + 64 * G + 8 + NP
    cin_b = cin_f + 2 * CIN_H + 64 + 2 * hp0 + 32
    ntile = -(-B // 32)
    nb = -(-G * hp0 // 128) + -(-64 * G // 128)
    q = max(1, 4 * n_sm // nb)
    per = -(-ntile // q)
    o = layout(G)
    grads = torch.full((o["total"],), float(base["grads"] + cin_f))
    grads[o["cin_w0"]:] = cin_b + per * 32 * D + -(-ntile // per)
    return {"logits": base["logits"] + cin_f, "loss": base["loss"] + cin_f, "grads": grads,
            "gsum_wide": base["gsum_wide"] + cin_b, "gsum_deep": base["gsum_deep"] + cin_b}


def ratios(got, ref, families=FAMILIES, c=C_TOL, n_sm=132):
    """tower_oracle.ratios with this module's chain lengths (a tensor for "grads")."""
    G, B = ref["gsum_wide"].shape[0], ref["logits"].shape[0]
    n = chain_lengths(G, B, n_sm)
    out = {}
    for fam in families:
        if fam not in got:
            continue
        want = ref[fam]
        g = torch.as_tensor(got[fam]).to(device=want.device, dtype=torch.float64).reshape(want.shape)
        m = ref["M"][fam]
        nn = torch.as_tensor(n[fam], dtype=torch.float64).to(m.device).expand_as(m).clone()
        if fam.startswith("gsum"):
            occ = ref["occ"] if fam == "gsum_wide" else ref["occ"].unsqueeze(2)
            nn = nn + occ
        bound = c * torch.sqrt(nn) * EPS32 * m
        if fam.startswith("gsum"):
            bound = bound + FLT_MIN * (occ + 1)
        elif fam in ("grads", "loss"):
            bound = bound + FLT_MIN * 8 * n_sm
        err = (g - want).abs()
        r = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                        torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
        r = torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))
        if fam.startswith("gsum"):
            live = torch.arange(want.shape[1], device=want.device).unsqueeze(0) < ref["n_unique"].unsqueeze(1)
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
    return {fam for fam, (r, *_rest) in ratios(got, ref, families, c, n_sm).items() if not r <= 1.0}


def check(got, ref, families=FAMILIES, c=C_TOL, label="", n_sm=132):
    rs = ratios(got, ref, families, c, n_sm)
    bad = {f: v for f, v in rs.items() if not v[0] <= 1.0}
    if bad:
        lines = ["%s %s: err/bound %.3g at %s (got %r, want %r)" % (label, f, r, w, gv, wv)
                 for f, (r, w, gv, wv) in bad.items()]
        raise AssertionError("\n".join(lines))
    return {f: v[0] for f, v in rs.items()}


KEYS = ("logits", "loss", "grads", "gsum_wide", "gsum_deep")
# A sample counted differently, or a row left out, moves the row sums of its ids by its dz alone in gsum_wide, but
# by far less than the CIN's long sums allow for in gsum_deep: there it is caught through gsum_wide.
EXPECTED_CATCH = {"drop_one_sample": {"gsum_wide"}, "last_sample_x32": {"gsum_wide"},
                  "tile_missing_from_grads": {"grads"}, "id_row_missing": {"gsum_wide"},
                  "loss_not_divided_by_B": {"loss"}, "k_index_transposed": {"logits"},
                  "split_halves_swapped": {"logits"}, "l2_term_missing": {"grads"},
                  "b_ex_gradient_missing": {"grads"}}
# Faults the bound does not catch at the benchmarked 38 groups: there the CIN's magnitudes (sums of |W| |Z| over
# K = G^2 and 64 G terms) dominate the bound of every parameter gradient and of the loss, and a single tile's share
# of the gradients (0.46 of the bound) or the L2 term (0.57) lies under it.  Both are caught at G = 2, and the
# L2 term is checked exactly on the prologue's output.
UNCAUGHT_AT_MAXG = {"tile_missing_from_grads", "l2_term_missing"}


def mutations(ref, inputs, tile=32, mask_override=None):
    """tower_oracle.mutations' faults plus xDeepFM's: the K index transposed (j m + i), the split halves swapped, the
    L2 term missing, the b_ex gradient missing.  A sample counted w times instead of once adds (w - 1) times its
    share, computed on that subset alone (the reference is linear in the per-sample weights)."""
    inv, n_unique, bet_wide, bet_deep, dense, labels, params = inputs
    G, B = inv.shape
    dev = ref["logits"].device
    base = {k: ref[k] for k in KEYS}
    o = layout(G)
    out = {}

    def reweighted(idx, dw):
        idx = torch.as_tensor(idx, device=dev)
        mo = None if mask_override is None else (mask_override[0][idx], mask_override[1][idx], mask_override[2])
        r = xdeepfm_reference(inv[:, idx], n_unique, bet_wide, bet_deep, dense[idx], labels[idx], params,
                              weight=torch.full((idx.numel(),), float(dw), dtype=torch.float64, device=dev),
                              mask_override=mo, norm=B, l2=False, magnitudes=False)
        return {k: base[k] + r[k] if k != "logits" else base[k] for k in KEYS}

    drop = B // 2 + 7 if B > 64 else B // 2
    out["drop_one_sample"] = reweighted([drop], -1.0)
    out["last_sample_x32"] = reweighted([B - 1], 31.0)
    t = (B // tile) // 2
    out["tile_missing_from_grads"] = dict(base, grads=reweighted(list(range(t * tile, min(B, (t + 1) * tile))),
                                                                 -1.0)["grads"])
    gw, gd = ref["gsum_wide"].clone(), ref["gsum_deep"].clone()
    gw[G - 1, 0] = 0
    gd[G - 1, 0] = 0
    out["id_row_missing"] = dict(base, gsum_wide=gw, gsum_deep=gd)
    out["loss_not_divided_by_B"] = dict(base, loss=ref["loss"] * B)
    for name, kw in (("k_index_transposed", {"k_order": "ji"}), ("split_halves_swapped", {"swap_halves": True})):
        r = xdeepfm_reference(*inputs, mask_override=mask_override, magnitudes=False, **kw)
        out[name] = {k: r[k] for k in KEYS}
    Wc = unflatten(params, G)
    reg = L2 * ((Wc[6].double() ** 2).sum() + (Wc[8].double() ** 2).sum())
    g = ref["grads"].clone()
    g[o["cin_w0"]:o["cin_b0"]] -= 2 * L2 * Wc[6].double().reshape(-1)
    g[o["cin_w1"]:o["cin_b1"]] -= 2 * L2 * Wc[8].double().reshape(-1)
    out["l2_term_missing"] = dict(base, loss=ref["loss"] - reg, grads=g)
    g = ref["grads"].clone()
    g[o["bex"]] = 0
    out["b_ex_gradient_missing"] = dict(base, grads=g)
    return out
