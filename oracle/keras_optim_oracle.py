"""CPU oracle of the Keras optimizers the PS applies besides the Go four and FTRL -- TEST INFRASTRUCTURE (see
ps_oracle.py's header: only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import oracle/).

RMSprop (plain, momentum, centered, centered + momentum), Adadelta, Adamax and Nadam, as the reference's Python PS
applies them (elasticdl/python/ps/optimizer_wrapper.py:116-149, slot names :200-210): a push updates only its
rows, with their deduplicated gradient sum, and decays their slots only then (the wrapper's sparse update,
optimizer_wrapper_test.py:421-426).  Dense parameters get the same per-element formula.  `t` is the shard's step
after the push's bump (quirk Q2) and `lr` the push's effective lr, as for Adam.

PARITY WITH TENSORFLOW IS UNPINNED, as it is for FTRL: TensorFlow is not installed and its sources are not in the
reference tree.  The formulas are restated from TF 2.5's training_ops (SparseApply[Centered]RMSProp,
SparseApplyAdadelta) and Keras optimizer_v2 (RMSprop's momentum = 0 python branch, Adamax and Nadam
_resource_apply_sparse) as recalled; DESIGN.md section 4 lists them.  What pins them independently is
torch.optim in float64 (tests/test_oracle_keras_optimizers.py).

The orders of operations below are the contract the device kernels (opt_update<OPT> and k_push_begin in
elasticdl_b200/csrc/ps_kernels.cuh) match bit for bit.  Every per-element operation is one float32 numpy
operation: IEEE round-to-nearest, never fused, so it computes what a C restatement built with
-ffp-contract=off computes.  Per-push scalars are formed in double from the float32 hyper-parameters and rounded
to float32 once, as k_push_begin forms them.

Nadam's per-push scalars are folded into the three per-push words every row kernel takes (ps_types.cuh PushRt):
    p -= lr * mbar / (sqrt(v / (1 - b2^t)) + eps),  mbar = (1 - u_t) g / (1 - S_t) + u_{t+1} m / (1 - S_{t+1})
is applied as p -= (cg * g + cm * m) / (sqrt(v) + ce) with cg = lr (1 - u_t) sqrt(1 - b2^t) / (1 - S_t),
cm = lr u_{t+1} sqrt(1 - b2^t) / (1 - S_{t+1}) and ce = eps sqrt(1 - b2^t).
"""
import math

import numpy as np

from oracle import ps_oracle as O

F = np.float32

KERAS_OPT_ARGS = {  # Keras get_config() key names, the `k=v;` grammar of optimizer.go:304-326
    "RMSprop": ["learning_rate", "rho", "momentum", "epsilon", "centered"],
    "Adadelta": ["learning_rate", "rho", "epsilon"],
    "Adamax": ["learning_rate", "beta_1", "beta_2", "epsilon"],
    "Nadam": ["learning_rate", "beta_1", "beta_2", "epsilon"],
}

# kind -> (device OptKind number, slot names in the record's order)
KINDS = {
    "rmsprop": (6, ["rms"]),
    "rmsprop_momentum": (7, ["rms", "momentum"]),
    "rmsprop_centered": (8, ["rms", "mg"]),
    "rmsprop_centered_momentum": (9, ["rms", "momentum", "mg"]),
    "adadelta": (10, ["accum_grad", "accum_var"]),
    "adamax": (11, ["m", "v"]),
    "nadam": (12, ["m", "v"]),
}

NADAM_MAX_STEPS = 1 << 16  # ps_types.cuh kNadamMaxSteps


def parse_opt_args(opt_type, opt_args):
    """'k=v;k=v;' -> dict; the refusals and messages of ps_oracle.parse_opt_args (optimizer.go:304-326)."""
    args = {}
    for kv in opt_args.split(";"):
        if kv == "":
            continue
        arr = kv.split("=")
        args[arr[0]] = arr[1]
    if opt_type not in KERAS_OPT_ARGS:
        raise ValueError("Unknown optimizer type %s" % opt_type)
    for name in KERAS_OPT_ARGS[opt_type]:
        if name not in args:
            raise ValueError("Args passed to ps should contain %s" % name)
    if len(args) != len(KERAS_OPT_ARGS[opt_type]):
        raise ValueError("Args passed to ps contain redundant items: %s" % args)
    return args


def hyper_params(opt_type, opt_args):
    """(kind, hp): the kind the parser picks and the float32 hyper-parameters the kernels read."""
    a = parse_opt_args(opt_type, opt_args)
    hp = {"lr": F(float(a["learning_rate"])), "epsilon": F(float(a["epsilon"]))}
    if opt_type in ("RMSprop", "Adadelta"):
        hp["rho"] = F(float(a["rho"]))
        hp["c_rho"] = F(1.0 - float(hp["rho"]))
    if opt_type == "RMSprop":
        hp["mu"] = F(float(a["momentum"]))
        centered = O.parse_bool(a["centered"])
        kind = "rmsprop" + ("_centered" if centered else "") + ("_momentum" if hp["mu"] > 0 else "")
    elif opt_type == "Adadelta":
        kind = "adadelta"
    else:
        kind = opt_type.lower()
        hp["beta1"], hp["beta2"] = F(float(a["beta_1"])), F(float(a["beta_2"]))
        hp["c1"], hp["c2"] = F(1.0 - float(hp["beta1"])), F(1.0 - float(hp["beta2"]))
        if kind == "nadam":
            hp["sched"] = nadam_schedule(hp["beta1"])
    return kind, hp


def nadam_u(beta1, t):
    """Keras' momentum cache u_t = beta_1 * (1 - 0.5 * 0.96^(0.004 t)): double, rounded to float32 once."""
    return F(float(F(beta1)) * (1.0 - 0.5 * math.pow(0.96, 0.004 * float(t))))


def nadam_schedule(beta1):
    """S_t for t = 0..last: S_0 = 1, S_t = S_{t-1} * u_t in float32 (Keras' m_cache), up to the first t where it
    stops changing; from there on S_t = S_last.  Raises ValueError when it has not settled within
    NADAM_MAX_STEPS steps (the group refuses that beta_1)."""
    b1 = F(beta1)
    s = [F(1.0)]
    settles = 0.0 <= float(b1) <= 1.0
    for t in range(1, NADAM_MAX_STEPS + 1):
        with np.errstate(over="ignore"):  # beta_1 > 1 overflows to inf and is refused below
            cur = F(s[-1] * nadam_u(b1, t))
        s.append(cur)
        if cur == s[-2] and (cur == 0.0 or settles):
            return np.asarray(s, dtype=np.float32)
    raise ValueError("Nadam: the momentum schedule of beta_1 = %r does not settle within %d steps"
                     % (float(b1), NADAM_MAX_STEPS))


def push_scalars(kind, hp, lr, t):
    """The three per-push words (PushRt lr, alpha, l2adj) k_push_begin writes for a push at step t with
    effective lr `lr`."""
    lr = F(lr)
    if kind == "adamax":
        return lr, F(float(lr) / (1.0 - float(hp["beta1"]) ** float(t))), F(0)
    if kind == "nadam":
        s = hp["sched"]
        last = len(s) - 1
        ut, ut1 = float(nadam_u(hp["beta1"], t)), float(nadam_u(hp["beta1"], t + 1))
        st, st1 = float(s[min(t, last)]), float(s[min(t + 1, last)])
        sb = math.sqrt(1.0 - float(hp["beta2"]) ** float(t))
        return (F(float(lr) * (1.0 - ut) * sb / (1.0 - st)), F(float(lr) * ut1 * sb / (1.0 - st1)),
                F(float(hp["epsilon"]) * sb))
    return lr, F(0), F(0)


def update(kind, hp, g, p, slots, w_lr, w_alpha, w_l2):
    """One element-wise update in opt_update<OPT>'s operation order.  g, p and the slots are float32 arrays of
    one shape; p and the slots are updated in place."""
    g = np.asarray(g, dtype=np.float32)
    eps = hp["epsilon"]
    if kind.startswith("rmsprop"):
        rho, c_rho = hp["rho"], hp["c_rho"]
        mom = kind.endswith("_momentum")
        rms = rho * slots[0] + c_rho * (g * g)
        slots[0][...] = rms
        den = rms
        if "centered" in kind:
            mg_slot = slots[2] if mom else slots[1]
            mg = rho * mg_slot + c_rho * g
            mg_slot[...] = mg
            den = rms - mg * mg
        if mom:
            m = hp["mu"] * slots[1] + (w_lr * g) / np.sqrt(den + eps)
            slots[1][...] = m
            p[...] = p - m
        else:
            p[...] = p - (w_lr * g) / (np.sqrt(den) + eps)
    elif kind == "adadelta":
        rho, c_rho = hp["rho"], hp["c_rho"]
        ag = rho * slots[0] + c_rho * (g * g)
        slots[0][...] = ag
        u = (np.sqrt(slots[1] + eps) / np.sqrt(ag + eps)) * g
        p[...] = p - w_lr * u
        slots[1][...] = rho * slots[1] + c_rho * (u * u)
    elif kind == "adamax":
        m = hp["beta1"] * slots[0] + hp["c1"] * g
        v = np.fmax(hp["beta2"] * slots[1], np.abs(g))
        slots[0][...] = m
        slots[1][...] = v
        p[...] = p - (w_alpha * m) / (v + eps)
    elif kind == "nadam":
        m = hp["beta1"] * slots[0] + hp["c1"] * g
        v = hp["beta2"] * slots[1] + hp["c2"] * (g * g)
        slots[0][...] = m
        slots[1][...] = v
        p[...] = p - (w_lr * g + w_alpha * m) / (np.sqrt(v) + w_l2)
    else:
        raise ValueError(kind)


def apply_rows(kind, hp, rows, slot_rows, gsum, lr, t):
    """The update of one push on deduplicated rows: rows [n, dim] and slot_rows (one [n, dim] array per slot) are
    the state before the push, gsum [n, dim] the rows' gradient sums.  Returns (rows, slot_rows) after it."""
    p = np.array(rows, dtype=np.float32)
    s = [np.array(x, dtype=np.float32) for x in slot_rows]
    update(kind, hp, np.asarray(gsum, dtype=np.float32), p, s, *push_scalars(kind, hp, lr, t))
    return p, s


def _occurrence_rounds(ids):
    """Index groups of `ids` such that each group holds at most one occurrence of an id, in occurrence order
    (the Go kernels apply a repeated id's rows one after another)."""
    seen, rounds = {}, []
    for i, x in enumerate(np.asarray(ids).tolist()):
        r = seen.get(x, 0)
        seen[x] = r + 1
        if r == len(rounds):
            rounds.append([])
        rounds[r].append(i)
    return [np.asarray(r, dtype=np.int64) for r in rounds]


class KerasOracleOptimizer(O.OracleOptimizer):
    """ps_oracle.OracleOptimizer for the Keras kinds: same slots bookkeeping (every slot starts at 0), the
    updates above."""

    def __init__(self, opt_type, opt_args, reproduce_q1=False):
        self.kind, self.hp = hyper_params(opt_type, opt_args)
        self.lr = self.hp["lr"]
        self.step = 0
        self.reproduce_q1 = reproduce_q1
        self.slots = {}
        self.slot_names = list(KINDS[self.kind][1])
        self.dense_slots = {n: {} for n in self.slot_names}
        self.table_slots = {n: {} for n in self.slot_names}

    def dense_kernel(self, g, p, name, lr):
        g = np.ascontiguousarray(g, dtype=np.float32).reshape(p.shape)
        s = [self.dense_slots[k][name] for k in self.slot_names]
        update(self.kind, self.hp, g, p, s, *push_scalars(self.kind, self.hp, lr, self.step))

    def sparse_kernel(self, ids, g, table, name, lr):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        g = np.ascontiguousarray(g, dtype=np.float32)
        if g.shape[1] != table.dim:  # kernel.go:36-38
            raise ValueError("grad width is not equal to embedding dim")
        tabs = [self.table_slots[k][name] for k in self.slot_names]
        w = push_scalars(self.kind, self.hp, lr, self.step)
        for r in _occurrence_rounds(ids):
            rid = ids[r]
            p = table.get(rid)
            s = [t.get(rid) for t in tabs]
            update(self.kind, self.hp, g[r], p, s, *w)
            table.set(rid, p)
            for t, x in zip(tabs, s):
                t.set(rid, x)

    def indexed_kernel(self, ids, g, p, name, lr):
        ids = np.ascontiguousarray(ids, dtype=np.int64)
        g = np.ascontiguousarray(g, dtype=np.float32)
        if g.shape[1] != p.shape[1]:  # kernel.go:86-88
            raise ValueError("grad width is not equal to embedding dim")
        arrs = [self.dense_slots[k][name] for k in self.slot_names]
        w = push_scalars(self.kind, self.hp, lr, self.step)
        for r in _occurrence_rounds(ids):
            rid = ids[r]
            pr = p[rid]
            s = [a[rid] for a in arrs]
            update(self.kind, self.hp, g[r], pr, s, *w)
            p[rid] = pr
            for a, x in zip(arrs, s):
                a[rid] = x


class KerasOracleServer(O.OracleServer):
    """ps_oracle.OracleServer with a KerasOracleOptimizer; works with ps_oracle.OraclePSClient."""

    def __init__(self, ps_id, opt_type, opt_args, num_ps=1, lr_staleness_modulation=False, seed=0):
        super().__init__(ps_id, "SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", num_ps,
                         lr_staleness_modulation, False, seed)
        self.opt = KerasOracleOptimizer(opt_type, opt_args)
