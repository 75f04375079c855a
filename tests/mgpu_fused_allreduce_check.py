"""DistributedOptimizer(fused=True) against the torch optimizer it wraps, step by step (torchrun, one rank per GPU;
B200_SHARED_GPU=1 puts every rank on cuda:0 as its own process):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \\
        --master-port 29555 tests/mgpu_fused_allreduce_check.py

Before every step each rank records the state the fused mode holds: the owner's copy of every parameter slice
(the flat parameters of that rank), every slice's optimizer slots (group.slot_dense on the owner), the Adam step
count of its shard (group.snapshot) and every rank's gradient.  After the step, the parameters and slots must lie
within the fp32 bound of oracle/torch_optim_oracle.py applied to that state.  An unfused DistributedOptimizer on
an identical model copy passes the same check from its own opt.state, which shows that the bound admits torch.

Scenarios: SGD, momentum, Nesterov, Adam and AMSGrad on gradients of 1e-9 .. 1e1 with exact zeros and a parameter
that gets no gradient on odd steps; parameters of 1, 3 and 4k+1 elements, one straddling two owners' slices, a
padded last slice and a frozen parameter; a slice longer than one grid-stride pass of the reduce kernel; op=Sum,
gradient_predivide_factor, reproduce_q10 and fixed_global_batch_size over two backward passes; LambdaLR warm-up
from lr 0 and StepLR; OneCycleLR and a hand-set momentum (ValueError); clamp_ between steps and a load_state_dict
resume; controller.broadcast() from ranks that start different; synchronize() + skip_synchronize() + step().
Then the refusals of fused=True and the silent fall-back of other truthy values.  Every scenario runs; the
failures are listed at the end."""
import copy
import os
import sys
import traceback

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticdl_b200.elasticai_api.pytorch.controller import create_elastic_controller  # noqa: E402
from elasticdl_b200.elasticai_api.pytorch.optimizer import DistributedOptimizer, Sum  # noqa: E402
from oracle import torch_optim_oracle as T  # noqa: E402

KEEP = []  # fused optimizers stay alive until exit: their shards are mapped by the peers

SMALL = [1, 3, 37, 35, 300, 9, 64]  # numel 1, 3, 4k+1; 300 straddles a slice boundary at world 2 and 3


class Net(torch.nn.Module):
    def __init__(self, sizes, seed):
        super().__init__()
        g = torch.Generator().manual_seed(seed)
        self.ws = torch.nn.ParameterList([torch.nn.Parameter(torch.randn(s, generator=g) * 0.1) for s in sizes])
        self.frozen = torch.nn.Parameter(torch.randn(5, generator=g), requires_grad=False)


def make_opt(kind, hp, params):
    if kind == "SGD":
        return torch.optim.SGD(params, lr=hp["lr"], momentum=hp["momentum"], nesterov=hp["nesterov"])
    return torch.optim.Adam(params, lr=hp["lr"], betas=hp["betas"], eps=hp["eps"], amsgrad=hp["amsgrad"])


def group_hp(kind, opt):
    g = opt.param_groups[0]
    if kind == "SGD":
        return {"lr": g["lr"], "momentum": g["momentum"], "nesterov": g["nesterov"]}
    return {"lr": g["lr"], "betas": tuple(g["betas"]), "eps": g["eps"], "amsgrad": g["amsgrad"]}


def wide(rng, n, scale):
    """Magnitudes 1e-9 .. 1e1 (times scale), about 10 % exact zeros at positions every rank shares."""
    return rng.standard_normal(n) * 10.0 ** rng.uniform(-9, 1, n) * scale


def gather_np(t):
    """Every rank's tensor t (same shape everywhere), as float64 numpy arrays in rank order."""
    out = [torch.empty_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t.contiguous())
    return [o.double().cpu().numpy() for o in out]


def slot_names(kind, hp):
    if kind == "SGD":
        return ["buf"] if hp["momentum"] else []
    return ["m", "v", "vmax"] if hp["amsgrad"] else ["m", "v"]


class Fused(object):
    """The fused optimizer's state in flat (bucket) space."""

    def __init__(self, opt, kind):
        self.opt, self.kind, self.ps = opt, kind, opt._ps
        self.name = "allreduce/slice_%d" % self.ps.rank

    def record(self, hp):
        self.opt._rebind_grads()  # what synchronize() does first: gradients that backward made land in the bucket
        ps = self.ps
        per, r = ps.per, ps.rank
        own = ps.flat_params[r * per:(r + 1) * per].clone()
        p = np.concatenate(gather_np(own))
        st = {}
        for k, key in enumerate(slot_names(self.kind, hp), start=1):
            st[key] = np.concatenate(gather_np(ps.group.slot_dense(self.name, k)))
        st["step"] = ps.group.snapshot()[r][1]
        if self.kind == "SGD" and "buf" not in st:
            st["buf"] = None
        g = gather_np(ps.flat_grads[:ps.total].clone())
        return p, g, st

    def after(self, hp):
        ps = self.ps
        got = {"p": ps.flat_params.double().cpu().numpy()}
        for k, key in enumerate(slot_names(self.kind, hp), start=1):
            got[key] = np.concatenate(gather_np(ps.group.slot_dense(self.name, k)))
        return got, ps.group.snapshot()[ps.rank][1]


def check_fused(fz, rec, hp, scale, predivide, label):
    p, g, st = rec
    ref_p, ref_st, bnd = T.step(fz.kind, p, g, st, hp, scale, predivide)
    got, step = fz.after(hp)
    ref = {"p": ref_p}
    ref.update({k: ref_st[k] for k in slot_names(fz.kind, hp)})
    T.check(got, ref, bnd, label="fused " + label)
    if fz.kind == "Adam":
        assert step == st["step"] + 1, "%s: shard step %d after %d" % (label, step, st["step"])


def record_unfused(opt, params, kind, hp):
    """Per parameter: (p, every rank's gradient, torch state) before the step."""
    out = []
    for q in params:
        grad = q.grad if q.grad is not None else torch.zeros_like(q)
        st = opt.state.get(q, {})
        if kind == "SGD":
            b = st.get("momentum_buffer")
            s = {"step": 0, "buf": None if b is None else b.double().cpu().numpy().reshape(-1).copy()}
        elif st:
            s = {"step": int(st["step"]), "m": st["exp_avg"].double().cpu().numpy().reshape(-1).copy(),
                 "v": st["exp_avg_sq"].double().cpu().numpy().reshape(-1).copy()}
            if "max_exp_avg_sq" in st:
                s["vmax"] = st["max_exp_avg_sq"].double().cpu().numpy().reshape(-1).copy()
        else:
            s = {"step": 0}
        out.append((q.detach().double().cpu().numpy().reshape(-1).copy(),
                    [x.reshape(-1) for x in gather_np(grad.detach())], s))
    return out


def check_unfused(opt, params, kind, recs, hp, scale, predivide, label):
    for i, (q, (p, g, st)) in enumerate(zip(params, recs)):
        ref_p, ref_st, bnd = T.step(kind, p, g, st, hp, scale, predivide)
        s = opt.state[q]
        got, ref = {"p": q.detach().double().cpu().numpy().reshape(-1)}, {"p": ref_p}
        torch_keys = {"buf": "momentum_buffer", "m": "exp_avg", "v": "exp_avg_sq", "vmax": "max_exp_avg_sq"}
        for key in slot_names(kind, hp):
            got[key] = s[torch_keys[key]].double().cpu().numpy().reshape(-1)
            ref[key] = ref_st[key]
        T.check(got, ref, bnd, label="unfused %s param %d" % (label, i))


def backward(model, cs, skip_unused):
    """loss = sum_i <w_i, c_i>: the gradient of w_i is exactly c_i (accumulated over calls); ws[0] gets none on
    odd steps when skip_unused."""
    loss = 0.0
    for i, (w, c) in enumerate(zip(model.ws, cs)):
        if i == 0 and skip_unused:
            continue
        loss = loss + (w * c).sum()
    loss.backward()


def scenario(name, kind, hp, dev, steps=3, sizes=SMALL, opt_kw=None, sched=None, passes=1, edit=None,
             resume=False, start_different=False, explicit_sync=False, raise_at=None, set_hp=None, controller=None):
    rank, world = dist.get_rank(), dist.get_world_size()
    opt_kw = dict(opt_kw or {})
    seed = 5 + (rank if start_different else 0)
    fmodel = Net(sizes, seed).to(dev)
    umodel = copy.deepcopy(fmodel)
    fopt = DistributedOptimizer(make_opt(kind, hp, fmodel.parameters()), named_parameters=fmodel.named_parameters(),
                                fused=True, **opt_kw)
    KEEP.append(fopt)
    assert fopt._ps is not None, "fused backend not selected"
    uopt = DistributedOptimizer(make_opt(kind, hp, umodel.parameters()), named_parameters=umodel.named_parameters(),
                                **opt_kw)
    if sizes is SMALL:  # the layout edges this model exists for
        per, n = fopt._ps.per, sum((s + 3) // 4 * 4 for s in sizes)
        assert n % (world * 64) != 0, "the last slice should be padded"
        offs = np.cumsum([0] + [(s + 3) // 4 * 4 for s in sizes])
        assert any(o // per != (o + s - 1) // per for o, s in zip(offs, sizes)), "no parameter straddles two slices"
    if start_different:
        for model, opt in ((fmodel, fopt), (umodel, uopt)):
            controller.set_broadcast_model(model)
            controller.set_broadcast_optimizer(opt)
            controller.broadcast()
            for w in model.ws:
                xs = gather_np(w.detach())
                assert all(np.array_equal(x, xs[0]) for x in xs), "broadcast left the ranks different"
    frozen0 = fmodel.frozen.detach().clone()  # after a broadcast, which sets it to rank 0's
    scheds = [sched(o) for o in (fopt, uopt)] if sched else []
    scale = T.scale_factor(world, opt_kw.get("op", "Average"), opt_kw.get("fixed_global_batch_size", False),
                           fopt._global_batch_num_per_step, opt_kw.get("reproduce_q10", False))
    predivide = opt_kw.get("gradient_predivide_factor", 1.0)
    fz = Fused(fopt, kind)
    ckpt = None
    for k in range(steps):
        mag = [1.0, 1e-2, 3.0, 1e-3][k % 4]  # falling magnitudes make AMSGrad's max matter
        rng = np.random.default_rng(1000 * k + 17 + rank)
        zrng = np.random.default_rng(1000 * k + 3)  # shared by the ranks: exact zeros of the sum
        for j in range(passes):
            cs = []
            for s in sizes:
                c = wide(rng, s, mag)
                c[zrng.random(s) < 0.1] = 0.0
                cs.append(torch.tensor(c, dtype=torch.float32, device=dev))
            for model, opt in ((fmodel, fopt), (umodel, uopt)):
                if passes == 1:
                    model.zero_grad(set_to_none=True)
                else:
                    opt.zero_grad()
                backward(model, cs, skip_unused=(k % 2 == 1 and passes == 1))
            if j < passes - 1:
                for opt in (fopt, uopt):
                    opt.step()  # an accumulation pass: no update yet
        if set_hp is not None and k == set_hp[0]:
            for opt in (fopt, uopt):
                opt.param_groups[0].update(set_hp[1])
        hp_now, hp_u = group_hp(kind, fopt), group_hp(kind, uopt)
        frec = fz.record(hp_now)
        urecs = record_unfused(uopt, list(umodel.ws), kind, hp_u)
        label = "%s step %d" % (name, k)
        if raise_at is not None and k == raise_at:
            try:
                fopt.step()
            except ValueError as e:
                assert "fused=True" in str(e), str(e)
            else:
                raise AssertionError("%s: fused step with a changed hyper-parameter did not raise" % label)
            uopt.step()
            check_unfused(uopt, list(umodel.ws), kind, urecs, hp_u, scale, predivide, label)
            return
        for opt in (fopt, uopt):
            if explicit_sync:
                opt.synchronize()
                with opt.skip_synchronize():
                    opt.step()
            else:
                opt.step()
        torch.cuda.synchronize()
        check_fused(fz, frec, hp_now, scale, predivide, label)
        check_unfused(uopt, list(umodel.ws), kind, urecs, hp_u, scale, predivide, label)
        for s in scheds:
            s.step()
        if edit is not None and k == edit:
            with torch.no_grad():
                for model in (fmodel, umodel):
                    for w in model.ws:
                        w.data.clamp_(-0.02, 0.02)
        if resume and k == 0:
            ckpt = [copy.deepcopy(m.state_dict()) for m in (fmodel, umodel)]
        if resume and k == 1:
            fmodel.load_state_dict(ckpt[0])
            umodel.load_state_dict(ckpt[1])
    assert torch.equal(fmodel.frozen, frozen0) and torch.equal(umodel.frozen, frozen0), "a frozen parameter moved"
    fopt._ps.group.check()


def refusals(dev):
    p = lambda: [torch.nn.Parameter(torch.randn(8, device=dev))]  # noqa: E731
    cases = {
        "AdamW": lambda: torch.optim.AdamW(p(), lr=1e-3),
        "weight_decay": lambda: torch.optim.SGD(p(), lr=0.1, weight_decay=0.1),
        "dampening": lambda: torch.optim.SGD(p(), lr=0.1, momentum=0.9, dampening=0.1),
        "maximize": lambda: torch.optim.SGD(p(), lr=0.1, maximize=True),
        "adam_maximize": lambda: torch.optim.Adam(p(), lr=1e-3, maximize=True),
        "two_groups": lambda: torch.optim.SGD([{"params": p()}, {"params": p()}], lr=0.1),
        "fp16": lambda: torch.optim.SGD([torch.nn.Parameter(torch.randn(8, device=dev).half())], lr=0.1),
        "cpu": lambda: torch.optim.SGD([torch.nn.Parameter(torch.randn(8))], lr=0.1),
        "adagrad": lambda: torch.optim.Adagrad(p(), lr=0.1),
    }
    for name, make in cases.items():
        try:
            opt = make()
            named = [("p%d" % i, q) for i, q in enumerate(q for g in opt.param_groups for q in g["params"])]
            DistributedOptimizer(opt, named_parameters=named, fused=True)
        except ValueError as e:
            assert "fused=True" in str(e), "%s: %s" % (name, e)
        else:
            raise AssertionError("fused=True accepted %s" % name)
        opt = make()
        named = [("p%d" % i, q) for i, q in enumerate(q for g in opt.param_groups for q in g["params"])]
        opt = DistributedOptimizer(opt, named_parameters=named, fused=1)
        assert opt._ps is None, "fused=1 with %s did not fall back" % name


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    shared = os.environ.get("B200_SHARED_GPU") == "1"
    local = 0 if shared else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    backend = "gloo" if shared else "nccl"
    controller = create_elastic_controller(batch_size=32, num_epochs=1, dataset_size=3200, backend=backend)
    assert dist.get_world_size() == world
    sgd = dict(lr=0.05, momentum=0.0, nesterov=False)
    mom = dict(lr=0.05, momentum=0.9, nesterov=False)
    nes = dict(lr=0.05, momentum=0.9, nesterov=True)
    adam = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, amsgrad=False)
    ams = dict(lr=1e-3, betas=(0.85, 0.99), eps=1e-8, amsgrad=True)
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    grid_pass = n_sm * 16 * 256 * 4  # floats one grid-stride pass of the 128-bit reduce kernel covers
    runs = [
        ("sgd", "SGD", sgd, {}),
        ("momentum", "SGD", mom, {}),
        ("nesterov", "SGD", nes, {}),
        ("adam", "Adam", adam, dict(steps=4)),
        ("amsgrad", "Adam", ams, dict(steps=4)),
        ("long_slice", "Adam", adam, dict(steps=2, sizes=[world * grid_pass + 5, 7])),
        ("op_sum", "SGD", nes, dict(opt_kw=dict(op=Sum))),
        ("predivide", "Adam", adam, dict(opt_kw=dict(gradient_predivide_factor=2.0))),
        ("reproduce_q10", "SGD", mom, dict(opt_kw=dict(reproduce_q10=True))),
        ("fixed_global_batch", "Adam", ams, dict(passes=2, opt_kw=dict(fixed_global_batch_size=True,
                                                                         backward_passes_per_step=2))),
        ("warmup_adam", "Adam", adam,
         dict(steps=4, sched=lambda o: torch.optim.lr_scheduler.LambdaLR(o, lambda k: k / 3.0))),
        ("warmup_momentum", "SGD", mom,
         dict(sched=lambda o: torch.optim.lr_scheduler.LambdaLR(o, lambda k: k / 2.0))),
        ("steplr", "SGD", nes, dict(sched=lambda o: torch.optim.lr_scheduler.StepLR(o, step_size=1, gamma=0.5))),
        ("onecycle", "SGD", mom,
         dict(raise_at=0, sched=lambda o: torch.optim.lr_scheduler.OneCycleLR(o, max_lr=0.1, total_steps=10))),
        ("momentum_by_hand", "SGD", mom, dict(raise_at=1, set_hp=(1, {"momentum": 0.5}))),
        ("betas_by_hand", "Adam", adam, dict(raise_at=1, set_hp=(1, {"betas": (0.8, 0.999)}))),
        ("clamp_edit", "Adam", adam, dict(edit=0)),
        ("clamp_edit_momentum", "SGD", mom, dict(edit=0)),
        ("resume", "Adam", ams, dict(steps=3, resume=True)),
        ("broadcast", "SGD", nes, dict(steps=2, start_different=True, controller=controller)),
        ("explicit_sync", "Adam", adam, dict(explicit_sync=True)),
    ]
    os.environ["WORKER_NUM"] = str(2 * world)  # fixed_global_batch: two backward passes per rank per update
    failed = []
    for name, kind, hp, kw in runs:
        try:
            scenario(name, kind, hp, dev, **kw)
        except Exception:
            failed.append(name)
            print("SCENARIO FAILED %s (world %d, rank %d):\n%s" % (name, world, rank, traceback.format_exc()[-2500:]),
                  flush=True)
        dist.barrier()
    try:
        refusals(dev)
    except Exception:
        failed.append("refusals")
        print("SCENARIO FAILED refusals (rank %d):\n%s" % (rank, traceback.format_exc()[-2500:]), flush=True)
    torch.cuda.synchronize()
    everywhere = [None] * world
    dist.all_gather_object(everywhere, failed)
    failed = sorted({f for fl in everywhere for f in fl})
    if rank == 0:
        if failed:
            print("mgpu_fused_allreduce_check FAILED: world=%d scenarios=%s" % (world, ",".join(failed)), flush=True)
        else:
            print("mgpu_fused_allreduce_check ok: world=%d scenarios=%d" % (world, len(runs)), flush=True)
    dist.destroy_process_group()
    sys.exit(1 if failed else 0)


if __name__ == "__main__":
    main()
