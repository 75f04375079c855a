"""oracle/torch_optim_oracle.py against torch.optim itself (CPU): the float64 restatement equals torch's float64
SGD / Adam over multi-step trajectories, an fp32 torch run (with the data-parallel gradient combine) stays inside
the bound at every step, and every mutation of a fused drop-in optimizer lies outside it."""
import numpy as np
import pytest
import torch

from oracle import torch_optim_oracle as T

CONFIGS = {
    "sgd": ("SGD", dict(lr=0.05, momentum=0.0, nesterov=False)),
    "momentum": ("SGD", dict(lr=0.05, momentum=0.9, nesterov=False)),
    "nesterov": ("SGD", dict(lr=0.05, momentum=0.9, nesterov=True)),
    "adam": ("Adam", dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, amsgrad=False)),
    "amsgrad": ("Adam", dict(lr=1e-3, betas=(0.85, 0.99), eps=1e-8, amsgrad=True)),
}


def torch_opt(kind, hp, params):
    if kind == "SGD":
        return torch.optim.SGD(params, lr=hp["lr"], momentum=hp["momentum"], nesterov=hp["nesterov"], foreach=False)
    return torch.optim.Adam(params, lr=hp["lr"], betas=hp["betas"], eps=hp["eps"], amsgrad=hp["amsgrad"],
                            foreach=False)


def wide_grads(rng, n, world):
    """Per-rank gradients whose magnitudes span 1e-9 .. 1e1, with exact zeros (in all ranks) and sign mixes."""
    sig = 10.0 ** rng.uniform(-9, 1, size=n)
    gs = [rng.standard_normal(n) * sig for _ in range(world)]
    zero = rng.random(n) < 0.1
    for g in gs:
        g[zero] = 0.0
    return gs


def torch_state(kind, opt, p):
    st = opt.state[p]
    if kind == "SGD":
        buf = st.get("momentum_buffer")
        return {"step": 0 if buf is None else 1, "buf": None if buf is None else buf.double().numpy().copy()}
    if not st:
        return {"step": 0}
    out = {"step": int(st["step"].item()), "m": st["exp_avg"].double().numpy().copy(),
           "v": st["exp_avg_sq"].double().numpy().copy()}
    if "max_exp_avg_sq" in st:
        out["vmax"] = st["max_exp_avg_sq"].double().numpy().copy()
    return out


def slots(kind, hp, st):
    if kind == "SGD":
        return {"buf": st["buf"]} if hp["momentum"] != 0.0 else {}
    out = {"m": st["m"], "v": st["v"]}
    if hp["amsgrad"]:
        out["vmax"] = st["vmax"]
    return out


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_oracle_equals_torch_float64(name):
    kind, hp = CONFIGS[name]
    rng = np.random.default_rng(1)
    n = 257
    p = torch.nn.Parameter(torch.tensor(rng.standard_normal(n), dtype=torch.float64))
    opt = torch_opt(kind, hp, [p])
    state = {"step": 0, "buf": None}
    want = p.detach().numpy().copy()
    lrs = [hp["lr"], hp["lr"] * 0.5, 0.0, hp["lr"]]  # a scheduler's lr, 0 included
    for k, lr in enumerate(lrs * 2):
        for gr in opt.param_groups:
            gr["lr"] = lr
        (g,) = wide_grads(rng, n, 1)
        p.grad = torch.tensor(g, dtype=torch.float64)
        opt.step()
        want, state, _ = T.step(kind, want, [g], state, dict(hp, lr=lr), 1.0)
        got = p.detach().numpy()
        # relative to each array's scale: elements that cancel to near 0 keep the absolute error of the others
        np.testing.assert_allclose(want, got, rtol=0, atol=4e-16 * np.abs(got).max(), err_msg="step %d" % k)
        ts = torch_state(kind, opt, p)
        for key, arr in slots(kind, hp, state).items():
            np.testing.assert_allclose(arr, ts[key], rtol=0, atol=4e-16 * np.abs(arr).max(),
                                       err_msg="%s step %d" % (key, k))
        if kind == "Adam":
            assert ts["step"] == state["step"]


MODES = [  # (world, op, fixed_global_batch_size, global_batch_num_per_step, predivide, reproduce_q10)
    (2, "Average", False, 1, 1.0, False),
    (3, "Sum", False, 1, 1.0, False),
    (3, "Average", False, 1, 2.0, False),
    (3, "Average", False, 1, 1.0, True),
    (3, "Average", True, 2, 1.0, False),
]


def combine_fp32(gs, scale, predivide):
    """DistributedOptimizer's unfused combine in fp32: optional predivide, the rank sum in rank order, one scale."""
    acc = None
    for g in gs:
        x = torch.tensor(g, dtype=torch.float32)
        if predivide != 1.0:
            x = x / predivide
        acc = x if acc is None else acc + x
    s = scale * predivide if predivide != 1.0 else scale
    return acc * s if s != 1.0 else acc


@pytest.mark.parametrize("mode", range(len(MODES)))
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_fp32_torch_stays_inside_bound(name, mode):
    kind, hp = CONFIGS[name]
    world, op, fixed, gbn, pre, q10 = MODES[mode]
    scale = T.scale_factor(world, op, fixed, gbn, q10)
    rng = np.random.default_rng(7 + mode)
    n = 4099
    p = torch.nn.Parameter(torch.tensor(rng.standard_normal(n) * 0.1, dtype=torch.float32))
    opt = torch_opt(kind, hp, [p])
    worst = {}
    for k, lr in enumerate([0.0, hp["lr"], hp["lr"], hp["lr"] * 0.3, hp["lr"]]):
        for gr in opt.param_groups:
            gr["lr"] = lr
        gs = [g.astype(np.float32) for g in wide_grads(rng, n, world)]
        st = torch_state(kind, opt, p)
        p0 = p.detach().double().numpy().copy()
        ref_p, ref_st, bnd = T.step(kind, p0, gs, st, dict(hp, lr=lr), scale, pre)
        p.grad = combine_fp32(gs, scale, pre)
        opt.step()
        got = {"p": p.detach().double().numpy()}
        got.update(slots(kind, hp, torch_state(kind, opt, p)))
        ref = {"p": ref_p}
        ref.update(slots(kind, hp, ref_st))
        for key, r in T.check(got, ref, bnd, label="%s mode %d step %d" % (name, mode, k)).items():
            worst[key] = max(worst.get(key, 0.0), r)
        if lr == 0.0:
            assert np.array_equal(got["p"], p0), "lr 0 moved the parameters"
    assert worst["p"] > 0.0


def _fp32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def _state(kind, hp, rng, n, step):
    """A mid-training state: slots of the size the wide gradients give, vmax above v on about half the elements."""
    if kind == "SGD":
        return {"step": step, "buf": _fp32(rng.standard_normal(n) * 10.0 ** rng.uniform(-9, 0, n))}
    v = _fp32((rng.standard_normal(n) * 10.0 ** rng.uniform(-9, 0, n)) ** 2)
    st = {"step": step, "m": _fp32(rng.standard_normal(n) * 10.0 ** rng.uniform(-9, 0, n)), "v": v}
    if hp["amsgrad"]:
        st["vmax"] = _fp32(np.where(rng.random(n) < 0.5, v * 3.0, v))
    return st


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_every_mutation_is_caught(name):
    kind, hp = CONFIGS[name]
    rng = np.random.default_rng(3)
    n, world = 2048, 3
    scale = T.scale_factor(world)
    p = _fp32(rng.standard_normal(n) * 0.1)
    gs = [_fp32(g) for g in wide_grads(rng, n, world)]
    for step, lr in [(0, 0.0), (2, hp["lr"])]:
        st = _state(kind, hp, rng, n, step) if step else {"step": 0}
        hp_now = dict(hp, lr=lr)
        built = dict(hp, lr=hp["lr"] * 2)
        if kind == "SGD":
            hp_now["momentum"] = 0.85 if hp["momentum"] else 0.0
        else:
            hp_now["betas"] = (hp["betas"][0] - 0.05, hp["betas"][1])
        edited = np.clip(p, -0.05, 0.05)  # the clamp_ the step must see; p is the copy from before it
        ref_p, ref_st, bnd = T.step(kind, edited, gs, st, hp_now, scale)
        ref = {"p": ref_p}
        ref.update(slots(kind, hp_now, ref_st) if step or kind == "Adam" or hp["momentum"] else {})
        T.check({k: _fp32(v) for k, v in ref.items()}, ref, bnd, label="fp32 rounding of the reference")
        muts = T.mutations(kind, edited, gs, st, hp_now, scale, hp_built=built, p_before_edit=p)
        if lr == 0.0:  # a zero step hides every other fault of the parameters
            expect = {"lr0_as_built"}
        else:
            expect = {"sum", "drop_rank", "edit_discarded"}
            if kind == "Adam" or hp["momentum"]:
                expect.add("momentum_frozen")
            if kind == "Adam":
                expect |= {"edl_eps", "step_off"} | ({"no_max"} if hp["amsgrad"] else set())
        assert expect <= set(muts), sorted(expect - set(muts))
        for mname in expect:
            mp, mst = muts[mname]
            got = {"p": _fp32(mp)}
            got.update({k: _fp32(v) for k, v in slots(kind, hp_now, mst).items()} if set(ref) - {"p"} else {})
            assert T.caught_by(got, ref, bnd), "%s step %d: mutation %s passes the bound" % (name, step, mname)


def test_combine_scale_modes():
    assert T.scale_factor(4) == 0.25
    assert T.scale_factor(4, reproduce_q10=True) == 1.0
    assert T.scale_factor(4, op="Sum") == 1.0
    assert T.scale_factor(4, fixed_global_batch_size=True, global_batch_num_per_step=8) == 0.125
    g, eg = T.combine([np.array([1.0, -2.0]), np.array([3.0, 2.0])], 0.5)
    np.testing.assert_array_equal(g, [2.0, 0.0])
    assert eg[1] > 0.0  # cancellation keeps the bound of the addends
