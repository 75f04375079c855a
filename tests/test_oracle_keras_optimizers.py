"""CPU checks of the Keras optimizers the PS applies besides the Go four and FTRL (RMSprop and its momentum /
centered variants, Adadelta, Adamax, Nadam): the native parser's grammar, the kind (and slot count) it picks,
Nadam's schedule table, and the oracle (oracle/keras_optim_oracle.py) against a float64 literal of each formula
and against torch.optim in float64."""
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch

from oracle import keras_optim_oracle as K

F = np.float32

KERAS_OPTS = {
    "rmsprop": ("RMSprop", "learning_rate=0.01;rho=0.9;momentum=0.0;epsilon=1e-07;centered=false;"),
    "rmsprop_momentum": ("RMSprop", "learning_rate=0.01;rho=0.9;momentum=0.5;epsilon=1e-07;centered=false;"),
    "rmsprop_centered": ("RMSprop", "learning_rate=0.01;rho=0.9;momentum=0.0;epsilon=1e-07;centered=true;"),
    "rmsprop_centered_momentum": ("RMSprop", "learning_rate=0.01;rho=0.8;momentum=0.9;epsilon=1e-07;centered=True;"),
    "adadelta": ("Adadelta", "learning_rate=1.0;rho=0.95;epsilon=1e-07;"),
    "adamax": ("Adamax", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;"),
    "nadam": ("Nadam", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;"),
}


def _create(opt_type, opt_args):
    from elasticdl_b200 import _lib

    h = ctypes.c_void_p()
    rc = _lib.lib().b200ps_create(1, 0, opt_type.encode(), opt_args.encode(), 0, 0, ctypes.byref(h))
    msg = _lib.lib().b200ps_last_error().decode()
    if rc == 0:
        _lib.lib().b200ps_destroy(h)
    return rc, msg


# ------------------------------------------------------------------ grammar
@pytest.mark.parametrize("opt", list(KERAS_OPTS))
def test_parser_accepts_the_four_grammars(opt):
    from elasticdl_b200 import _lib

    rc, _ = _create(*KERAS_OPTS[opt])
    # past the parser: a group, or (without a device) the CUDA failure that follows parsing
    assert rc in (0, _lib.ECUDA), rc
    assert K.hyper_params(*KERAS_OPTS[opt])[0] == opt


@pytest.mark.parametrize("opt_type,args,msg", [
    ("RMSprop", "learning_rate=0.01;rho=0.9;momentum=0.0;epsilon=1e-07;", "should contain centered"),
    ("RMSprop", "learning_rate=0.01;rho=0.9;momentum=0.0;epsilon=1e-07;centered=false;amsgrad=false;",
     "contain redundant items"),
    ("RMSprop", "learning_rate=0.01;rho=0.9;momentum=0.0;epsilon=1e-07;centered=maybe;", "bad RMSprop argument"),
    ("Adadelta", "learning_rate=1.0;epsilon=1e-07;", "should contain rho"),
    ("Adadelta", "learning_rate=1.0;rho=0.95;epsilon=1e-07;beta=1;", "contain redundant items"),
    ("Adamax", "learning_rate=0.002;beta_1=0.9;epsilon=1e-07;", "should contain beta_2"),
    ("Adamax", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", "contain redundant items"),
    ("Nadam", "beta_1=0.9;beta_2=0.999;epsilon=1e-07;", "should contain learning_rate"),
    ("Nadam", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=x;", "bad Nadam argument"),
    ("Rmsprop", "learning_rate=0.01;", "Unknown optimizer type Rmsprop"),
])
def test_parser_refuses_missing_redundant_and_bad_values(opt_type, args, msg):
    from elasticdl_b200 import _lib

    rc, got = _create(opt_type, args)
    assert rc == _lib.EINVAL and msg in got, (rc, got)
    if "bad" not in msg:  # the oracle's parser refuses the same grammar with the same message
        with pytest.raises(ValueError, match=msg.split(" ")[-1]):
            K.hyper_params(opt_type, args)


@pytest.mark.parametrize("momentum,centered,kind,slots", [
    ("0.0", "false", "rmsprop", ["rms"]),
    ("0.1", "false", "rmsprop_momentum", ["rms", "momentum"]),
    ("0.0", "true", "rmsprop_centered", ["rms", "mg"]),
    ("0.1", "1", "rmsprop_centered_momentum", ["rms", "momentum", "mg"]),
    ("-0.5", "F", "rmsprop", ["rms"]),  # Keras: the momentum slot exists only for momentum > 0
])
def test_rmsprop_kind_follows_momentum_and_centered(momentum, centered, kind, slots):
    args = "learning_rate=0.01;rho=0.9;momentum=%s;epsilon=1e-07;centered=%s;" % (momentum, centered)
    k, _ = K.hyper_params("RMSprop", args)
    assert k == kind and K.KINDS[k][1] == slots
    opt = K.KerasOracleOptimizer("RMSprop", args)
    assert opt.slot_names == slots


# ------------------------------------------------------------------ Nadam schedule
def test_nadam_schedule_settles_in_keras_order():
    s = K.nadam_schedule(0.9)
    prod = F(1.0)
    for t in range(1, len(s)):  # Keras: m_schedule_new = m_cache * momentum_cache_t, float32
        prod = F(prod * F(float(F(0.9)) * (1.0 - 0.5 * 0.96 ** (0.004 * t))))
        assert s[t] == prod, t
    assert s[-1] == s[-2] and len(s) < 2000
    assert K.nadam_schedule(0.0)[-1] == 0.0
    for b1 in (0.0, 0.5, 0.99, 0.9999999, 1.0):  # the first factors are near beta_1 / 2: 0 within 160 steps
        s = K.nadam_schedule(b1)
        assert len(s) <= 160 and s[-1] == s[-2], b1


def test_nadam_refuses_a_schedule_that_does_not_settle():
    from elasticdl_b200 import _lib

    args = "learning_rate=0.002;beta_1=1.5;beta_2=0.999;epsilon=1e-07;"  # S_t grows to infinity
    rc, msg = _create("Nadam", args)
    assert rc == _lib.EINVAL and "does not settle within 65536 steps" in msg, (rc, msg)
    with pytest.raises(ValueError, match="does not settle"):
        K.hyper_params("Nadam", args)


# ------------------------------------------------------------------ float64 literal of each formula
def _literal(kind, hp, g, p, s, lr, t):
    """One step in float64, written as DESIGN.md section 4 states the formulas (not in the kernel's order)."""
    eps = float(hp["epsilon"])
    s = [x.copy() for x in s]
    if kind.startswith("rmsprop"):
        rho, mom = float(hp["rho"]), kind.endswith("_momentum")
        s[0] = rho * s[0] + (1 - rho) * g * g
        den = s[0]
        if "centered" in kind:
            j = 2 if mom else 1
            s[j] = rho * s[j] + (1 - rho) * g
            den = s[0] - s[j] ** 2
        if mom:
            s[1] = float(hp["mu"]) * s[1] + lr * g / np.sqrt(den + eps)
            p = p - s[1]
        else:
            p = p - lr * g / (np.sqrt(den) + eps)
    elif kind == "adadelta":
        rho = float(hp["rho"])
        s[0] = rho * s[0] + (1 - rho) * g * g
        u = np.sqrt(s[1] + eps) / np.sqrt(s[0] + eps) * g
        p = p - lr * u
        s[1] = rho * s[1] + (1 - rho) * u * u
    elif kind == "adamax":
        b1, b2 = float(hp["beta1"]), float(hp["beta2"])
        s[0] = b1 * s[0] + (1 - b1) * g
        s[1] = np.maximum(b2 * s[1], np.abs(g))
        p = p - lr / (1 - b1 ** t) * s[0] / (s[1] + eps)
    else:
        b1, b2 = float(hp["beta1"]), float(hp["beta2"])
        u = lambda k: b1 * (1 - 0.5 * 0.96 ** (0.004 * k))  # noqa: E731
        st = float(hp["sched"][min(t, len(hp["sched"]) - 1)])
        st1 = st * u(t + 1)
        s[0] = b1 * s[0] + (1 - b1) * g
        s[1] = b2 * s[1] + (1 - b2) * g * g
        mbar = (1 - u(t)) * g / (1 - st) + u(t + 1) * s[0] / (1 - st1)
        p = p - lr * mbar / (np.sqrt(s[1] / (1 - b2 ** t)) + eps)
    return p, s


@pytest.mark.parametrize("opt", list(KERAS_OPTS))
def test_oracle_matches_a_float64_literal_over_many_steps(opt):
    kind, hp = K.hyper_params(*KERAS_OPTS[opt])
    rng = np.random.RandomState(zlib.crc32(opt.encode()))
    n = 4096
    p = rng.randn(n).astype(F)
    s = [np.zeros(n, dtype=F) for _ in K.KINDS[kind][1]]
    for t in range(1, 301):
        g = (rng.randn(n) * 10.0 ** rng.uniform(-3, 1, n)).astype(F)
        g[rng.rand(n) < 0.05] = 0.0
        lr = F(hp["lr"] * (0.5 if t % 7 == 0 else 1.0))
        want_p, want_s = _literal(kind, hp, g.astype(np.float64), p.astype(np.float64),
                                  [x.astype(np.float64) for x in s], float(lr), t)
        p0, s0 = p.copy(), [x.astype(np.float64) for x in s]
        K.update(kind, hp, g, p, s, *K.push_scalars(kind, hp, lr, t))
        # a few float32 roundings of each result, of the terms a sum cancels (|new| + |old|), and of a momentum
        # slot's terms where p subtracts that slot
        step = np.abs(want_p - p0.astype(np.float64))
        if kind.endswith("_momentum"):
            step = step + np.abs(s0[1])
        assert np.all(np.abs(p - want_p) <= 2.0 ** -22 * np.abs(want_p) + 2.0 ** -20 * step + 1e-30), (opt, t)
        for x, w, old in zip(s, want_s, s0):
            assert np.all(np.abs(x - w) <= 2.0 ** -20 * (np.abs(w) + np.abs(old)) + 1e-30), (opt, t)
    assert all(np.any(x != 0) for x in s)


def test_rmsprop_epsilon_quirk_hand_computed():
    """Q13: momentum = 0 divides by sqrt(rms) + eps, momentum > 0 by sqrt(rms + eps).  rms << eps tells them
    apart: g = 1e-3, rho = 0.9 -> rms = 1e-7, eps = 1e-2."""
    g = np.array([1e-3], dtype=F)
    out = {}
    for mom in ("0.0", "0.5"):
        args = "learning_rate=0.1;rho=0.9;momentum=%s;epsilon=0.01;centered=false;" % mom
        kind, hp = K.hyper_params("RMSprop", args)
        p = np.zeros(1, dtype=F)
        s = [np.zeros(1, dtype=F) for _ in K.KINDS[kind][1]]
        K.update(kind, hp, g, p, s, *K.push_scalars(kind, hp, F(0.1), 1))
        out[mom] = float(-p[0])
    rms = 0.1 * 1e-6
    assert math.isclose(out["0.0"], 0.1 * 1e-3 / (math.sqrt(rms) + 0.01), rel_tol=1e-6)  # 9.6934e-3
    assert math.isclose(out["0.5"], 0.1 * 1e-3 / math.sqrt(rms + 0.01), rel_tol=1e-6)  # 9.99995e-4
    assert out["0.0"] > 9 * out["0.5"]


# ------------------------------------------------------------------ torch.optim in float64
def _torch_opt(opt, hp, param):
    lr = float(hp["lr"])
    if opt.startswith("rmsprop"):
        return torch.optim.RMSprop([param], lr=lr, alpha=float(hp["rho"]), eps=float(hp["epsilon"]),
                                   momentum=float(hp["mu"]), centered="centered" in opt)
    if opt == "adadelta":
        return torch.optim.Adadelta([param], lr=lr, rho=float(hp["rho"]), eps=float(hp["epsilon"]))
    if opt == "adamax":
        return torch.optim.Adamax([param], lr=lr, betas=(float(hp["beta1"]), float(hp["beta2"])),
                                  eps=float(hp["epsilon"]))
    return torch.optim.NAdam([param], lr=lr, betas=(float(hp["beta1"]), float(hp["beta2"])),
                             eps=float(hp["epsilon"]), momentum_decay=0.004)


# torch has the same math in float64: Adadelta and NAdam exactly, RMSprop without momentum with its eps,
# RMSprop with momentum at eps = 0 (torch's buf times lr is TF's mom), Adamax at eps = 0 (torch adds eps
# inside the max).
TORCH_PINS = {
    "rmsprop": "learning_rate=0.01;rho=0.9;momentum=0.0;epsilon=1e-03;centered=false;",
    "rmsprop_centered": "learning_rate=0.01;rho=0.9;momentum=0.0;epsilon=1e-03;centered=true;",
    "rmsprop_momentum": "learning_rate=0.01;rho=0.9;momentum=0.5;epsilon=0;centered=false;",
    "rmsprop_centered_momentum": "learning_rate=0.01;rho=0.8;momentum=0.9;epsilon=0;centered=true;",
    "adadelta": "learning_rate=1.0;rho=0.95;epsilon=1e-06;",
    "adamax": "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=0;",
    "nadam": "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;",
}


@pytest.mark.parametrize("opt", list(TORCH_PINS))
def test_oracle_matches_torch_optim_in_float64(opt):
    opt_type = {"adadelta": "Adadelta", "adamax": "Adamax", "nadam": "Nadam"}.get(opt, "RMSprop")
    kind, hp = K.hyper_params(opt_type, TORCH_PINS[opt])
    assert kind == opt
    rng = np.random.RandomState(len(opt))
    n = 2048
    p = rng.randn(n).astype(F)
    s = [np.zeros(n, dtype=F) for _ in K.KINDS[kind][1]]
    p_init = p.astype(np.float64)
    param = torch.nn.Parameter(torch.tensor(p, dtype=torch.float64))
    topt = _torch_opt(opt, hp, param)
    for t in range(1, 41):
        g = (rng.randn(n) * (0.1 + t % 3)).astype(F)
        param.grad = torch.tensor(g, dtype=torch.float64)
        topt.step()
        K.update(kind, hp, g, p, s, *K.push_scalars(kind, hp, hp["lr"], t))
    got = param.detach().numpy()
    moved = np.max(np.abs(got - p_init))
    assert np.allclose(p, got, rtol=2e-5, atol=2e-5 * moved), np.max(np.abs(p - got))
    st = topt.state[param]
    pairs = {"rmsprop": [("square_avg", 0)], "rmsprop_centered": [("square_avg", 0), ("grad_avg", 1)],
             "rmsprop_momentum": [("square_avg", 0)], "rmsprop_centered_momentum": [("square_avg", 0), ("grad_avg", 2)],
             "adadelta": [("square_avg", 0), ("acc_delta", 1)], "adamax": [("exp_avg", 0), ("exp_inf", 1)],
             "nadam": [("exp_avg", 0), ("exp_avg_sq", 1)]}[opt]
    for key, j in pairs:
        ref = st[key].numpy()  # an average of gradients of both signs cancels: absolute bound at its scale
        assert np.allclose(s[j], ref, rtol=1e-5, atol=1e-6 * np.max(np.abs(ref))), key
    if opt.endswith("_momentum"):  # TF's mom is lr times torch's buf
        ref = float(hp["lr"]) * st["momentum_buffer"].numpy()
        assert np.allclose(s[1], ref, rtol=1e-5, atol=1e-6 * np.max(np.abs(ref)))
    if opt == "nadam":  # torch's mu_product is S_t
        assert math.isclose(float(st["mu_product"]), float(hp["sched"][40]), rel_tol=1e-6)
