"""Float64 reference of the frappe DeepFM tower (include/b200_frappe.h) -- TEST INFRASTRUCTURE.

The literal layer graph of model_zoo/deepfm_edl_embedding/deepfm_edl_embedding.py:40-88, not the collapsed form
the kernel computes: the mask multiply (ApplyMask, :24-37), first = sum of the masked bias rows, the FM as written
(0.5 * (square of sum - sum of squares), summed over the 64 dims, :50-56), Flatten (f-major), Dense(64) and
Dense(1) with their biases, the mean sigmoid cross-entropy; the backward written out layer by layer.  Plain torch
float64, device-agnostic.  The inputs are the kernel's own: ids [B, 10], the dedup's inv [10 B] and n_unique, the
unique rows bet_deep [U, 64] / bet_wide [U, 1], labels [B] and the flat dense buffer [41089].

The error bound is tower_oracle's: |got - ref| <= C_TOL * sqrt(n) * 2^-24 * M elementwise, M from a magnitude
pass (the same graph over |operands|) and n the longest fp32 accumulation chain behind the output, taken from
the kernel's reduction order (`chain_lengths`); every fp32 atomic add behind an output may also lose FLT_MIN.
"""
import math

import numpy as np
import torch

from oracle.tower_oracle import C_TOL, EPS32, FLT_MIN, P_FLOOR

F, D = 10, 64
X = F * D
TILE = 64  # B200_FRAPPE_TILE
DENSE_PARAMS = [("dense/kernel:0", (X, D)), ("dense/bias:0", (D,)), ("dense_1/kernel:0", (D, 1)),
                ("dense_1/bias:0", (1,))]
OFFSETS = {}
_o = 0
for _n, _s in DENSE_PARAMS:
    OFFSETS[_n] = _o
    _o += int(np.prod(_s))
N_PARAMS = _o
assert N_PARAMS == 41089
FAMILIES = ("logits", "loss", "grads", "gsum_deep", "gsum_wide")
FAULTS = (None, "no_mask", "d_major", "fm_sign", "no_c", "wide_twice")


def unflatten(flat):
    return {n: flat[OFFSETS[n]:OFFSETS[n] + int(np.prod(s))].view(s) for n, s in DENSE_PARAMS}


def random_params(gen, device, dtype=torch.float32, bias=0.1):
    """Glorot-uniform kernels (as the model initialises them); biases U(-bias, bias) instead of zero, so that the
    checks see them."""
    flat = torch.empty(N_PARAMS, dtype=dtype, device=device)
    v = unflatten(flat)
    for n, s in DENSE_PARAMS:
        lim = math.sqrt(6.0 / (s[0] + s[1])) if n.endswith("kernel:0") else bias
        v[n].copy_((torch.rand(s, generator=gen, device=device, dtype=dtype) * 2 - 1) * lim)
    return flat


def dedup(ids):
    """tf.unique of ids [B, 10] read sample-major: (uniq [U] first-occurrence order, inv int64 [10 B], U)."""
    flat = ids.reshape(-1).to(torch.int64)
    u, inv = torch.unique(flat, return_inverse=True)
    first = torch.full((u.numel(),), flat.numel(), dtype=torch.int64, device=flat.device)
    first.scatter_reduce_(0, inv, torch.arange(flat.numel(), device=flat.device), "amin")
    order = torch.argsort(first)
    rank = torch.empty_like(order)
    rank[order] = torch.arange(order.numel(), device=flat.device)
    return u[order], rank[inv], int(u.numel())


def frappe_reference(ids, inv, n_unique, bet_deep, bet_wide, labels, params, weight=None, fault=None):
    """Float64 forward + backward of one batch.  weight [B] (optional): a multiplicity per sample in every
    reduction (1 everywhere is the real model).  fault: one of FAULTS (a deliberately wrong model, for the
    mutation checks).

    Returns float64 tensors on the inputs' device: logits [B], loss [], grads [41089], gsum_deep [U, 64],
    gsum_wide [U, 1], row_id [U] (the id of every unique row), occ [U] (its occurrences), "M" (magnitudes of
    logits, loss, grads, gsum_deep, gsum_wide), "B"."""
    assert fault in FAULTS, fault
    f64 = torch.float64
    dev = labels.device
    ids = ids.to(device=dev, dtype=torch.int64)
    B = ids.shape[0]
    U = int(n_unique)
    inv = inv.to(device=dev, dtype=torch.int64).reshape(B, F)
    Eu = bet_deep[:U].to(device=dev, dtype=f64)
    Wu = bet_wide[:U].to(device=dev, dtype=f64).reshape(U, 1)
    p = {n: v.to(device=dev, dtype=f64) for n, v in unflatten(params).items()}
    K, b, w2, b2 = p["dense/kernel:0"], p["dense/bias:0"], p["dense_1/kernel:0"][:, 0], p["dense_1/bias:0"][0]
    y = labels.to(f64)
    wt = torch.ones(B, dtype=f64, device=dev) if weight is None else weight.to(device=dev, dtype=f64)
    m = (ids != 0).to(f64).unsqueeze(2)  # [B, 10, 1]
    if fault == "no_mask":
        m = torch.ones_like(m)

    def flatten(e):  # Flatten of [B, 10, 64]: f-major (d-major is a fault)
        return e.permute(0, 2, 1).reshape(B, X) if fault == "d_major" else e.reshape(B, X)

    def unflatten_grad(dx):
        return dx.reshape(B, D, F).permute(0, 2, 1) if fault == "d_major" else dx.reshape(B, F, D)

    fm_sign = -1.0 if fault == "fm_sign" else 1.0
    wide_k = 2.0 if fault == "wide_twice" else 1.0
    use_c = 0.0 if fault == "no_c" else 1.0

    # forward: the layers
    e = m * Eu[inv]  # ApplyMask
    w = m * Wu[inv]
    first = wide_k * w.sum((1, 2))
    S = e.sum(1)
    second = fm_sign * (0.5 * (S * S - (e * e).sum(1))).sum(1)
    x = flatten(e)
    h = x @ K + use_c * b
    deep = h @ w2 + use_c * b2
    z = first + second + deep
    lb = z.clamp_min(0) - z * y + torch.log1p(torch.exp(-z.abs()))
    loss = (wt * lb).sum() / B

    # backward
    pz = torch.sigmoid(z)
    gz = (pz - y) / B * wt
    dw2 = h.t() @ gz
    db2 = gz.sum()
    dh = gz.unsqueeze(1) * w2.unsqueeze(0)  # [B, 64]
    dK = x.t() @ dh
    db = dh.sum(0) * use_c
    de = unflatten_grad(dh @ K.t()) + fm_sign * gz.view(B, 1, 1) * (S.unsqueeze(1) - e)
    dE = m * de
    dW = m * (wide_k * gz.view(B, 1, 1))
    grads = torch.cat([dK.reshape(-1), db, dw2, db2.reshape(1)])
    gsum_deep = torch.zeros((U, D), dtype=f64, device=dev).index_add_(0, inv.reshape(-1), dE.reshape(B * F, D))
    gsum_wide = torch.zeros((U, 1), dtype=f64, device=dev).index_add_(0, inv.reshape(-1), dW.reshape(B * F, 1))

    # magnitude pass: the same graph over |operands|
    aw = wt.abs()
    ae, aK, ab, aw2 = e.abs(), K.abs(), b.abs(), w2.abs()
    aS = ae.sum(1)
    ax = flatten(ae)
    ah = ax @ aK + ab
    Mz = w.abs().sum((1, 2)) * wide_k + (0.5 * (aS * aS + (ae * ae).sum(1))).sum(1) + ah @ aw2 + b2.abs()
    Mloss = (aw * (Mz * (1 + y.abs()) + torch.log1p(torch.exp(-z.abs())))).sum() / B
    Mg = (pz * (1 - pz) * Mz + pz + y.abs() + P_FLOOR) / B * aw
    Mdh = Mg.unsqueeze(1) * aw2.unsqueeze(0)
    Mgrads = torch.cat([(ax.t() @ Mdh).reshape(-1), Mdh.sum(0), ah.t() @ Mg, Mg.sum().reshape(1)])
    MdE = m * (unflatten_grad(Mdh @ aK.t()) + Mg.view(B, 1, 1) * (aS.unsqueeze(1) + ae))
    Mgd = torch.zeros((U, D), dtype=f64, device=dev).index_add_(0, inv.reshape(-1), MdE.reshape(B * F, D))
    Mgw = torch.zeros((U, 1), dtype=f64, device=dev).index_add_(0, inv.reshape(-1),
                                                               (m * Mg.view(B, 1, 1) * wide_k).reshape(B * F, 1))
    row_id = torch.zeros(U, dtype=torch.int64, device=dev)
    row_id[inv.reshape(-1)] = ids.reshape(-1)
    occ = torch.zeros(U, dtype=torch.int64, device=dev).index_add_(0, inv.reshape(-1),
                                                                  torch.ones(B * F, dtype=torch.int64, device=dev))
    return {"logits": z, "loss": loss, "grads": grads, "gsum_deep": gsum_deep, "gsum_wide": gsum_wide,
            "row_id": row_id, "occ": occ, "B": B,
            "M": {"logits": Mz, "loss": Mloss, "grads": Mgrads, "gsum_deep": Mgd, "gsum_wide": Mgw}}


def chain_lengths(B, max_occ):
    """Longest fp32 accumulation chain behind each output family, in the kernel's order.  Forward: v = K w2 (64
    terms), a lane's 20-term dot with it, the 32-lane sum, S over 10 rows, the 10 bias rows and c.  The batch
    sums s, G and the loss are added per warp, per CTA and then across CTAs: at most B terms; K^T s adds 640
    more.  A row's gradient is summed over at most 32 samples per red and at most one red per occurrence."""
    fwd = 64 + 20 + 32 + 10 + 10 + 2
    return {"logits": fwd, "loss": fwd + B, "grads": fwd + B + X, "gsum_deep": fwd + 3 + max_occ,
            "gsum_wide": fwd + max_occ}


def _ratio(got, want, m, n, c, floor):
    g = torch.as_tensor(got).to(device=want.device, dtype=torch.float64).reshape(want.shape)
    bound = c * math.sqrt(n) * EPS32 * m + floor
    err = (g - want).abs()
    r = torch.where(bound > 0, err / torch.where(bound > 0, bound, torch.ones_like(bound)),
                    torch.where(err == 0, torch.zeros_like(err), torch.full_like(err, math.inf)))
    r = torch.where(torch.isfinite(g), r, torch.full_like(r, math.inf))
    if r.numel() == 0:
        return 0.0, (), float("nan"), float("nan")
    i = int(torch.argmax(r.reshape(-1)))
    where = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), r.shape)) if r.dim() else ()
    return float(r.reshape(-1)[i]), where, float(g.reshape(-1)[i]), float(want.reshape(-1)[i])


def ratios(got, ref, c=C_TOL):
    """Per family present in `got`: (worst err / bound, where, got, want)."""
    B = ref["B"]
    max_occ = int(ref["occ"].max()) if ref["occ"].numel() else 0
    n = chain_lengths(B, max_occ)
    out = {}
    for fam in FAMILIES:
        if fam in got:
            # every atomic add may flush a subnormal: one FLT_MIN per term of the chain (the row sums: where M > 0)
            floor = n[fam] * FLT_MIN if fam in ("loss", "grads") else (ref["M"][fam] > 0) * (n[fam] * FLT_MIN)
            out[fam] = _ratio(got[fam], ref[fam], ref["M"][fam], n[fam], c, floor)
    return out


def caught_by(got, ref, c=C_TOL):
    return {fam for fam, (r, *_rest) in ratios(got, ref, c).items() if not r <= 1.0}


def check(got, ref, c=C_TOL, label=""):
    """Assert every family within the bound; returns {family: worst ratio}."""
    rs = ratios(got, ref, c)
    bad = {f: v for f, v in rs.items() if not v[0] <= 1.0}
    if bad:
        raise AssertionError("\n".join("%s %s: err/bound %.3g at %s (got %r, want %r)" % (label, f, r, w, gv, wv)
                                       for f, (r, w, gv, wv) in bad.items()))
    return {f: v[0] for f, v in rs.items()}


def mutations(ref, inputs):
    """The reference's outputs with one classic fault each: name -> dict of outputs.
    inputs: (ids, inv, n_unique, bet_deep, bet_wide, labels, params); the batch should contain pads."""
    keys = FAMILIES
    B = ref["B"]
    dev = ref["logits"].device

    def run(**kw):
        r = frappe_reference(*inputs, **kw)
        return {k: r[k] for k in keys}

    out = {"mask_dropped": run(fault="no_mask"), "flatten_d_major": run(fault="d_major"),
           "fm_sign": run(fault="fm_sign"), "c_missing": run(fault="no_c"), "wide_twice": run(fault="wide_twice")}
    pad = ref["row_id"] == 0
    if bool(pad.any()):  # id 0's rows get the gradient an unmasked occurrence would give them
        unmasked = frappe_reference(*inputs, fault="no_mask")
        gd, gw = ref["gsum_deep"].clone(), ref["gsum_wide"].clone()
        gd[pad], gw[pad] = unmasked["gsum_deep"][pad], unmasked["gsum_wide"][pad]
        out["pad_row_gradient"] = dict({k: ref[k] for k in keys}, gsum_deep=gd, gsum_wide=gw)
    wt = torch.ones(B, dtype=torch.float64, device=dev)
    wt[B // 2] = 0
    out["drop_one_sample"] = run(weight=wt)
    return out


def make_teacher(seed, ref_ids, n_ids=5383):
    """A fixed random model of the same form that labels synthetic batches: bias rows N(0, 1), deep rows
    U(-0.05, 0.05), glorot kernels, zero biases; a sample is positive when its logit exceeds the median logit of
    `ref_ids` (so the labels are balanced)."""
    g = torch.Generator().manual_seed(int(seed))
    W = torch.randn((n_ids, 1), generator=g, dtype=torch.float64)
    E = (torch.rand((n_ids, D), generator=g, dtype=torch.float64) * 2 - 1) * 0.05
    flat = random_params(g, "cpu", dtype=torch.float64, bias=0.0)
    t = {"W": W, "E": E, "flat": flat, "threshold": 0.0}
    t["threshold"] = float(teacher_logits(t, ref_ids).median())
    return t


def teacher_logits(t, ids):
    ids = ids.cpu()
    uniq, inv, U = dedup(ids)
    r = frappe_reference(ids, inv, U, t["E"][uniq], t["W"][uniq], torch.zeros(ids.shape[0], dtype=torch.float64),
                         t["flat"])
    return r["logits"]


def teacher_labels(t, ids):
    """float32 labels of ids [B, 10] on the ids' device."""
    return (teacher_logits(t, ids) > t["threshold"]).to(device=ids.device, dtype=torch.float32)
