"""Float64 reference of the deepctr DeepFM estimator tower (include/b200_deepctr_deepfm.h) and of its two TF1
optimizers -- TEST INFRASTRUCTURE.

deepctr's DeepFMEstimator of model_zoo/deepctr/deepfm_estimator.py, from raw rows: ids = FarmHash Fingerprint64 %
1000 of the 26 string columns, with "" dropped (categorical_column_with_hash_bucket: id -1 here), e_j = the mean of
the ids that remain (E_j[id_j], or 0), x = [e_1 .. e_26 | I] (F = 117), three relu layers 256 -> 128 -> 64 and a
bias-free logit kernel, the FM 1/2 sum_d ((sum_j e_jd)^2 - sum_j e_jd^2), the linear model sum_j L_j[id_j] + I w_num
+ bias_weights, z the sum of the three; loss = sum_b sigmoid_cross_entropy(y, z) + 1e-5/2 (sum_b sum_j |e_bj|^2 +
sum_j |L_j|^2 + |w_num|^2).  The gradient is the complete flat gradient: an embedding row gets its occurrences of
dx + 1e-5 e (0 when untouched), a linear row 1e-5 w + its occurrences of dz.  deepctr's and TF1's details are
RECALLED, not read from their source (DESIGN.md section 4, Q31-Q35).  Plain torch float64, forward and backward
written out by hand (no autograd), device-agnostic.

TF1's Adagrad (no epsilon) and FTRL (lr_power -0.5, no l1 / l2 / shrinkage) steps are written out as well.

The error bound is tower_oracle's: |got - ref| <= C_TOL * sqrt(n) * 2^-24 * M elementwise, M from a magnitude
pass (the same sums over |operands|, plus the propagated error of z) and n the longest fp32 accumulation chain.
"""
import math

import numpy as np
import torch

from oracle import feature_oracle as FO
from oracle import tf32
from oracle.deepctr_wdl_oracle import _ratio
from oracle.tower_oracle import C_TOL, P_FLOOR

FIELDS, DENSE, ROWS, DIM = 26, 13, 1000, 4
NS, F = FIELDS * DIM, FIELDS * DIM + DENSE
H = (256, 128, 64)
LAMBDA = 1e-5
TILE = 64
N_PARAMS, N_DNN_GROUP = 201438, 175424
O_DNN = FIELDS * ROWS * DIM
DNN_SHAPES = [(F, H[0]), (H[0],), (H[0], H[1]), (H[1],), (H[1], H[2]), (H[2],), (H[2], 1)]
LOGIT_BIAS = 0.1  # the trained value the logit_bias mutation gives the bias deepctr leaves out
ADAGRAD_ACCUM, ADAGRAD_LR, FTRL_ACCUM, FTRL_LR = 0.1, 0.01, 0.1, 0.005
MUTATIONS = ("empty_as_bucket", "absent_as_row0", "fm_no_self_term", "lambda_in_loss", "two_lambda_in_grad",
             "l2_on_bias_weights", "mean_loss", "logit_bias")
# 1e-5 / 2 |bias_weights|^2 and 1e-5 / 2 of the regulariser hide under the summed cross-entropy's rounding; a batch
# whose logits all sit at +100 with every label 1 (cross-entropy and dz below 1e-43) shows them
SATURATED_MUTATIONS = ("lambda_in_loss", "l2_on_bias_weights")
OPTIMIZER_MUTATIONS = ("adagrad_epsilon", "adagrad_zero_accumulator")


def ids_from_raw(raw, bins=ROWS, drop_empty=True):
    """raw: 26 lists of B byte strings -> int64 [26, B]: Fingerprint64 % bins, and -1 for "" unless drop_empty is
    False (then "" hashes as an ordinary bucket, the WDL's rule)."""
    out = []
    for col in raw:
        col = [bytes(s) for s in col]
        ids = FO.hashing(col, bins)
        if drop_empty:
            ids = np.where(np.array([len(s) == 0 for s in col], dtype=bool), -1, ids)
        out.append(ids)
    return torch.from_numpy(np.stack(out).astype(np.int64))


def unflatten(flat):
    """(emb [26, 1000, 4], [W0, b0, W1, b1, W2, b2, wd], lin [26, 1000], w_num [13], bias_weights [1])."""
    emb = flat[:O_DNN].reshape(FIELDS, ROWS, DIM)
    dnn, o = [], O_DNN
    for s in DNN_SHAPES:
        k = math.prod(s)
        dnn.append(flat[o:o + k].reshape(s))
        o += k
    assert o == N_DNN_GROUP
    lin = flat[o:o + FIELDS * ROWS].reshape(FIELDS, ROWS)
    o += FIELDS * ROWS
    return emb, dnn, lin, flat[o:o + DENSE], flat[o + DENSE:o + DENSE + 1]


def reference(ids, dense, labels, flat, mutate=(), contraction=None):
    """{loss, logits [B], grads [201438], B, M: magnitudes of each}.  ids int [26, B] in [-1, 1000) (-1 absent),
    dense [13, B], labels [B], flat [201438].  mutate: names of MUTATIONS to build in (empty_as_bucket acts on raw
    rows: see mutations()).  contraction: the hidden layers' forward, data and weight contractions in the modes of
    oracle/tf32.py (exact by default)."""
    mode = tf32.modes(contraction)

    def mm(kind, a, b):
        return tf32.contract(a, b, mode[kind])

    dev = flat.device
    flat = flat.to(torch.float64)
    ids = ids.long().to(dev)
    I = dense.to(device=dev, dtype=torch.float64).t()  # noqa: E741  [B, 13]
    y = labels.to(device=dev, dtype=torch.float64)
    B = I.shape[0]
    emb, (W0, b0, W1, b1, W2, b2, wd), lin, wn, bw = unflatten(flat)
    if "absent_as_row0" in mutate:
        ids = ids.clamp(min=0)
    present = (ids >= 0) & (ids < ROWS)  # [26, B]
    rows = torch.where(present, ids, torch.zeros_like(ids))
    fa = torch.arange(FIELDS, device=dev).unsqueeze(1)
    pf = present.t().unsqueeze(2).to(torch.float64)  # [B, 26, 1]
    e = emb[fa, rows].permute(1, 0, 2) * pf  # [B, 26, 4]: the mean of the ids that remain
    x = torch.cat([e.reshape(B, NS), I], 1)
    a1 = mm("forward", x, W0) + b0
    h1 = a1.clamp(min=0)
    a2 = mm("forward", h1, W1) + b1
    h2 = a2.clamp(min=0)
    a3 = mm("forward", h2, W2) + b2
    h3 = a3.clamp(min=0)
    lv = lin[fa, rows] * present  # [26, B]
    S = e.sum(1)  # [B, 4]
    sq = (e * e).sum(1)  # [B, 4]
    fm = 0.5 * (S * S).sum(1) if "fm_no_self_term" in mutate else 0.5 * (S * S - sq).sum(1)
    z = lv.sum(0) + I @ wn + bw[0] + fm + (h3 @ wd)[:, 0]
    if "logit_bias" in mutate:
        z = z + LOGIT_BIAS
    ce = z.clamp(min=0) - z * y + torch.log1p(torch.exp(-z.abs()))
    dz = torch.sigmoid(z) - y
    if "mean_loss" in mutate:
        ce, dz = ce / B, dz / B
    lam_loss = LAMBDA if "lambda_in_loss" in mutate else 0.5 * LAMBDA
    lam_grad = 2 * LAMBDA if "two_lambda_in_grad" in mutate else LAMBDA
    reg = (e * e).sum() + (lin * lin).sum() + (wn * wn).sum()
    if "l2_on_bias_weights" in mutate:
        reg = reg + bw[0] * bw[0]
    loss = ce.sum() + lam_loss * reg

    dh3 = dz.unsqueeze(1) * wd[:, 0] * (a3 > 0)
    dh2 = mm("data", dh3, W2.t()) * (a2 > 0)
    dh1 = mm("data", dh2, W1.t()) * (a1 > 0)
    dx = mm("data", dh1, W0.t())
    fm_self = torch.zeros_like(e) if "fm_no_self_term" in mutate else e
    de = dx[:, :NS].reshape(B, FIELDS, DIM) + dz.view(B, 1, 1) * (S.unsqueeze(1) - fm_self) + lam_grad * e
    gemb = torch.zeros_like(emb)
    glin = lam_grad * lin
    for j in range(FIELDS):
        p = present[j]
        gemb[j].index_add_(0, ids[j][p], de[p, j])
        glin[j].index_add_(0, ids[j][p], dz[p])
    gbw = dz.sum().reshape(1) + (lam_grad * bw if "l2_on_bias_weights" in mutate else 0)
    grads = torch.cat([gemb.reshape(-1), mm("weight", x.t(), dh1).reshape(-1), dh1.sum(0),
                       mm("weight", h1.t(), dh2).reshape(-1), dh2.sum(0), mm("weight", h2.t(), dh3).reshape(-1),
                       dh3.sum(0), (h3.t() @ dz).reshape(-1), glin.reshape(-1), I.t() @ dz + lam_grad * wn, gbw])

    # magnitudes
    ae, ax, aI = e.abs(), x.abs(), I.abs()
    Mh1 = ax @ W0.abs() + b0.abs()
    Mh2 = Mh1 @ W1.abs() + b1.abs()
    Mh3 = Mh2 @ W2.abs() + b2.abs()
    MS = ae.sum(1)
    Mfm = 0.5 * (MS * MS + (ae * ae).sum(1)).sum(1)
    Mz = (Mh3 @ wd.abs())[:, 0] + lv.abs().sum(0) + aI @ wn.abs() + bw.abs()[0] + Mfm
    # z's rounding moves dz by at most sigmoid'(z) times it, taken a little nearer z = 0 to cover the move itself
    zn = (z.abs() - 1e-3 * Mz).clamp(min=0)
    Mdz = dz.abs() + torch.sigmoid(zn) * torch.sigmoid(-zn) * Mz + P_FLOOR
    Mdh3 = Mdz.unsqueeze(1) * wd[:, 0].abs()
    Mdh2 = Mdh3 @ W2.abs().t()
    Mdh1 = Mdh2 @ W1.abs().t()
    Mdx = Mdh1 @ W0.abs().t()
    Mde = Mdx[:, :NS].reshape(B, FIELDS, DIM) + Mdz.view(B, 1, 1) * (MS.unsqueeze(1) + ae) + LAMBDA * ae
    Memb = torch.zeros_like(emb)
    Mlin = LAMBDA * lin.abs()
    for j in range(FIELDS):
        p = present[j]
        Memb[j].index_add_(0, ids[j][p], Mde[p, j])
        Mlin[j].index_add_(0, ids[j][p], Mdz[p])
    Mgrads = torch.cat([Memb.reshape(-1), (ax.t() @ Mdh1).reshape(-1), Mdh1.sum(0), (Mh1.t() @ Mdh2).reshape(-1),
                        Mdh2.sum(0), (Mh2.t() @ Mdh3).reshape(-1), Mdh3.sum(0), (Mh3.t() @ Mdz).reshape(-1),
                        Mlin.reshape(-1), aI.t() @ Mdz + LAMBDA * wn.abs(), Mdz.sum().reshape(1)])
    Mloss = (ce.abs() + Mdz * Mz).sum() + LAMBDA * reg  # z's rounding moves ce by at most |dce/dz| = |dz| times it
    return {"logits": z, "loss": loss, "grads": grads, "B": B, "M": {"logits": Mz, "loss": Mloss, "grads": Mgrads}}


def chain_lengths(B, n_sm=132):
    """Longest fp32 accumulation chain behind each output family: the forward's F + 256 + 128 + 64 products, the
    26 linear rows, 13 numeric terms and the FM's 26-term sums; the backward's 64 + 128 + 256; then the batch sums
    (per CTA at most ceil(tiles / CTAs) tiles of 64, then over the CTAs' partials; a table row sums at most B
    occurrences; the linear rows' squares over 4 x n_sm table CTAs)."""
    fwd = F + sum(H) + 2 * FIELDS + DENSE + 4
    tiles = -(-B // TILE)
    ctas = max(1, min(tiles, n_sm))
    per_cta = TILE * -(-tiles // ctas)
    return {"logits": fwd, "loss": fwd + per_cta + ctas + FIELDS * ROWS // (32 * n_sm) + 4 * n_sm,
            "grads": fwd + sum(H) + max(per_cta + ctas, B)}


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
    """name -> reference outputs with that fault built in.  empty_as_bucket hashes `raw` (26 lists of B byte
    strings) with "" an ordinary bucket and is left out without raw."""
    out = {}
    for name in names:
        if name == "empty_as_bucket":
            if raw is not None:
                out[name] = reference(ids_from_raw(raw, drop_empty=False), dense, labels, flat)
        else:
            out[name] = reference(ids, dense, labels, flat, mutate=(name,))
    return out


# ---- the optimizers, on float64 tensors of one parameter
def adagrad_init(p, mutate=()):
    """TF1 AdagradOptimizer's accumulator: initial_accumulator_value = 0.1 (0 under adagrad_zero_accumulator)."""
    return torch.full_like(p, 0.0 if "adagrad_zero_accumulator" in mutate else ADAGRAD_ACCUM)


def adagrad_step(p, acc, g, lr=ADAGRAD_LR, mutate=()):
    """TF1 ApplyAdagrad: acc += g^2; p -= lr g / sqrt(acc), no epsilon (1e-7 under adagrad_epsilon, Keras' form).
    Returns (p, acc).  A zero accumulator with a zero gradient gives 0/0: the mutation's NaN is what it is."""
    acc = acc + g * g
    den = acc.sqrt() + (1e-7 if "adagrad_epsilon" in mutate else 0.0)
    return p - lr * g / den, acc


def ftrl_init(p):
    """TF1 FtrlOptimizer's slots: accumulator = initial_accumulator_value = 0.1, linear = 0."""
    return torch.full_like(p, FTRL_ACCUM), torch.zeros_like(p)


def ftrl_step(p, acc, linear, g, lr=FTRL_LR):
    """TF1 ApplyFtrl with learning_rate_power = -0.5 and l1 = l2 = l2_shrinkage = 0: acc' = acc + g^2; linear +=
    g - (sqrt(acc') - sqrt(acc)) / lr p; p = -linear / (sqrt(acc') / lr) (0 where linear is 0).  Returns
    (p, acc', linear)."""
    acc_new = acc + g * g
    linear = linear + g - (acc_new.sqrt() - acc.sqrt()) / lr * p
    quad = acc_new.sqrt() / lr
    p = torch.where(linear.abs() > 0, -linear / quad, torch.zeros_like(p))
    return p, acc_new, linear
