"""Float64 restatement of torch.optim.SGD and torch.optim.Adam for one data-parallel step, with the fp32 rounding
bound of an implementation that starts from the same state: the oracle of DistributedOptimizer, fused or not.

A step takes the state the implementation actually held before it (parameters, slots, Adam step count, all as
float64 arrays of its fp32 values) and every rank's fp32 gradient, and returns the exact next state and a
per-element bound, in the form of the tower and sparse oracles: every fp32 operation of the step may round once,
by up to 2^-24 of its result, and errors of the inputs propagate through each operation to first order.

Gradient combine (DistributedOptimizer._scale_factor): g = scale * sum_r g_r with
  op=Sum: scale 1; op=Average: 1 / world, 1 with reproduce_q10 (quirk Q10), or 1 / global_batch_num_per_step
  with fixed_global_batch_size.  gradient_predivide_factor f divides before the sum and multiplies after it:
  exactly the same g, two more roundings.
"""
import numpy as np

U = 2.0 ** -24
TINY = 2.0 ** -126  # one flushed or subnormal result per operation

# One data-parallel step's hyper-parameters: SGD {"lr", "momentum", "nesterov"};
# Adam {"lr", "betas", "eps", "amsgrad"}.


def scale_factor(world, op="Average", fixed_global_batch_size=False, global_batch_num_per_step=1,
                 reproduce_q10=False):
    if op != "Average":
        return 1.0
    if fixed_global_batch_size:
        return 1.0 / global_batch_num_per_step
    return 1.0 if reproduce_q10 else 1.0 / world


def combine(grads, scale, predivide=1.0):
    """(g, bound of g): the exact scaled rank sum of fp32 gradients and the fp32 error of summing them in any
    order ((world - 1) roundings of at most sum_r |g_r|), scaling (the factor's own rounding and the product's),
    and the predivide / postmultiply pair."""
    gs = np.stack([np.asarray(x, dtype=np.float64) for x in grads])
    world = gs.shape[0]
    absum = np.abs(gs).sum(axis=0)
    g = gs.sum(axis=0) * scale
    k = (world - 1) + 2 + (3 if predivide != 1.0 else 0)
    return g, k * U * absum * abs(scale) + 2 * TINY


def _sqrt_err(x, ex):
    """Bound of |sqrt(x + e) - sqrt(x)| for |e| <= ex, x >= 0."""
    with np.errstate(divide="ignore", invalid="ignore"):
        lin = np.where(x > 0, ex / np.sqrt(np.where(x > 0, x, 1.0)), np.inf)
    return np.minimum(np.sqrt(ex), lin)


def sgd_step(p, g, eg, buf, hp):
    """torch.optim.SGD (dampening 0, no weight decay): buf = g on the first step (buf None), else
    momentum * buf + g; d = g + momentum * buf (nesterov) or buf; p -= lr * d.
    Returns (p, {"buf": buf}, bounds {"p", "buf"})."""
    lr, mu, nest = float(hp["lr"]), float(hp["momentum"]), bool(hp["nesterov"])
    out, bnd = {}, {}
    if mu == 0.0:
        d, ed = g, eg
    else:
        if buf is None:
            nb, eb = g.copy(), eg.copy()
        else:
            nb = mu * buf + g
            eb = eg + 2 * U * mu * np.abs(buf) + U * np.abs(nb) + TINY
        out["buf"], bnd["buf"] = nb, eb
        if nest:
            d = g + mu * nb
            ed = eg + mu * eb + 2 * U * mu * np.abs(nb) + U * np.abs(d) + TINY
        else:
            d, ed = nb, eb
    newp = p - lr * d
    bnd["p"] = lr * ed + 2 * U * lr * np.abs(d) + U * np.abs(newp) + TINY
    return newp, out, bnd


def adam_step(p, g, eg, m, v, vmax, step, hp, fault=None):
    """torch.optim.Adam (no weight decay, not maximize), from step count `step` (0 before the first update):
    m = b1 m + (1-b1) g; v = b2 v + (1-b2) g^2; vmax = max(vmax, v) with amsgrad;
    p -= lr / (1 - b1^t) * m / (sqrt(vhat) / sqrt(1 - b2^t) + eps),  t = step + 1.
    fault (mutations only): "edl_eps" adds eps to sqrt(vhat) (ElasticDL's kernel_api.cc), "step_off" uses t + 1,
    "no_max" keeps v instead of max(vmax, v)."""
    b1, b2 = (float(x) for x in hp["betas"])
    lr, eps, ams = float(hp["lr"]), float(hp["eps"]), bool(hp["amsgrad"])
    t = step + 1 + (1 if fault == "step_off" else 0)
    nm = b1 * m + (1 - b1) * g
    nv = b2 * v + (1 - b2) * g * g
    em = (1 - b1) * eg + 3 * U * (np.abs(m) + (1 - b1) * np.abs(g)) + U * np.abs(nm) + TINY
    ev = (1 - b2) * (2 * np.abs(g) * eg + eg * eg) + 3 * U * (b2 * v + (1 - b2) * g * g) + U * nv + TINY
    out = {"m": nm, "v": nv}
    bnd = {"m": em, "v": ev}
    vhat = nv
    if ams:
        nvm = nv if fault == "no_max" else np.maximum(vmax, nv)
        out["vmax"], bnd["vmax"] = nvm, ev
        vhat = nvm
    bc1, bc2 = 1.0 - b1 ** t, 1.0 - b2 ** t
    s = np.sqrt(vhat)
    es = _sqrt_err(vhat, ev) + U * s
    # on alpha's scale: D = sqrt(vhat) + eps * sqrt(bc2), alpha = lr * sqrt(bc2) / bc1
    D = s + (eps if fault == "edl_eps" else eps * np.sqrt(bc2))
    eD = es + 3 * U * D
    alpha = lr * np.sqrt(bc2) / bc1
    q = alpha * nm / D
    rel = np.minimum(eD / D, 0.5)
    eq = alpha * (em / D + np.abs(nm) * eD / (D * D) / (1 - rel)) + 3 * U * np.abs(q) + TINY
    newp = p - q
    bnd["p"] = eq + U * np.abs(newp) + TINY
    return newp, out, bnd


def step(kind, p, grads, state, hp, scale, predivide=1.0, fault=None):
    """One DistributedOptimizer step of `kind` ("SGD" or "Adam") on flat float64 arrays.
    state: {"step": int, "buf": array or None} (SGD) or {"step", "m", "v", "vmax"} (Adam), as the implementation
    held it before the step.  grads: every rank's gradient.  Returns (p, new state, bounds {"p", slot...}).
    fault (mutations): "sum" (the sum, not the scaled sum), "drop_rank" (the last rank's gradient lost), and the
    Adam faults of adam_step."""
    p = np.asarray(p, dtype=np.float64)
    if fault == "drop_rank":
        grads = grads[:-1]
    g, eg = combine(grads, 1.0 if fault == "sum" else scale, predivide)
    if kind == "SGD":
        newp, out, bnd = sgd_step(p, g, eg, state.get("buf"), hp)
        out["step"] = state["step"] + 1
    else:
        z = np.zeros_like(p)
        newp, out, bnd = adam_step(p, g, eg, state.get("m", z), state.get("v", z), state.get("vmax", z),
                                   state["step"], hp, fault)
        out["step"] = state["step"] + 1
    return newp, out, bnd


def ratio(got, ref, bound):
    """(worst |got - ref| / bound, its flat index); NaN or Inf anywhere in got is infinitely bad."""
    got = np.asarray(got, dtype=np.float64).reshape(-1)
    ref = np.asarray(ref, dtype=np.float64).reshape(-1)
    bound = np.asarray(bound, dtype=np.float64).reshape(-1)
    if got.size == 0:
        return 0.0, -1
    r = np.abs(got - ref) / bound
    r = np.where(np.isfinite(got), r, np.inf)
    i = int(np.argmax(r))
    return float(r[i]), i


def caught_by(got, ref, bounds):
    """The names (keys of ref: "p" and the slots) whose got lies outside the bound somewhere."""
    return {k for k in ref if not ratio(got[k], ref[k], bounds[k])[0] <= 1.0}


def check(got, ref, bounds, label=""):
    """Assert every array of got ({"p": ..., slot: ...}) within the bound of ref; returns {name: worst ratio}."""
    out, bad = {}, []
    for k in ref:
        r, i = ratio(got[k], ref[k], bounds[k])
        out[k] = r
        if not r <= 1.0:
            g = np.asarray(got[k], dtype=np.float64).reshape(-1)
            w = np.asarray(ref[k], dtype=np.float64).reshape(-1)
            bad.append("%s %s: err/bound %.3g at %d (got %r, want %r)" % (label, k, r, i, g[i], w[i]))
    if bad:
        raise AssertionError("\n".join(bad))
    return out


def mutations(kind, p, grads, state, hp, scale, predivide=1.0, hp_built=None, p_before_edit=None):
    """The step's outcome under one classic fault each of a fused drop-in optimizer: name -> (p, state).
      sum               the rank sum without the scale;
      drop_rank         the last rank's gradient lost;
      lr0_as_built      a step at lr 0 taken at the construction lr (hp_built["lr"]), only when hp["lr"] == 0;
      momentum_frozen   momentum / beta1 kept at its construction value, only when it differs from hp_built's;
      edit_discarded    the step applied to p_before_edit (the copy held before an in-place edit), when given;
      edl_eps, step_off, no_max   (Adam) ElasticDL's eps, the step count off by one, AMSGrad's max not kept."""
    out = {}

    def run(fault=None, **kw):
        args = dict(kind=kind, p=p, grads=grads, state=state, hp=hp, scale=scale, predivide=predivide)
        args.update(kw)
        newp, st, _ = step(fault=fault, **args)
        return newp, st

    out["sum"] = run("sum")
    if len(grads) > 1:
        out["drop_rank"] = run("drop_rank")
    if hp_built is not None:
        if float(hp["lr"]) == 0.0 and float(hp_built["lr"]) != 0.0:
            out["lr0_as_built"] = run(hp=dict(hp, lr=hp_built["lr"]))
        key = "momentum" if kind == "SGD" else "betas"
        if hp.get(key) != hp_built.get(key):
            frozen = hp_built[key] if kind == "SGD" else (hp_built["betas"][0], hp["betas"][1])
            out["momentum_frozen"] = run(hp=dict(hp, **{key: frozen}))
    if p_before_edit is not None:
        out["edit_discarded"] = run(p=p_before_edit)
    if kind == "Adam":
        out["edl_eps"] = run("edl_eps")
        out["step_off"] = run("step_off")
        if hp["amsgrad"]:
            out["no_max"] = run("no_max")
    return out
