"""The drop-in API path bench.py times, checked against references over several Adam steps.

bench.py's api_path_leg builds PSGroup(1, "Adam", ADAM_ARGS), a PSClient that keeps pulled dense parameters on the
device, DeepFMLayersModel() -- 76 Embedding layers over the 38 dac_ctr groups at full size, the tower in eager torch --
and ParameterServerTrainer over them, and times train_minibatch on B = 32768 batches (seeds 1234 + p): as one CUDA
graph per minibatch, eagerly with the trainer's batched lookups, and with one lookup per layer call.  The trainer's
own tests compare those paths with each other; every leg here checks each step t against outside references:
  1. the dedup: the ids pushed for every table == the oracle's first-occurrence dedup of its group, exactly, and
     the (unique ids, inverse) of every dedup the step ran (the batched lookups' one bounded dedup shared by the deep
     and wide families, or the 76 per-layer hashed ones);
  2. the returned loss, the pushed dense gradients and the pushed row gradients within the float64 tower
     reference's bound (oracle/tower_oracle.py) of the state the step started from;
  3. the oracle's Adam (step t, lr 1e-3) applied to the pushed gradients, from the pre-step param / m / v, bit for
     bit on every pushed row of the 76 tables and on the 6 dense parameters; sampled rows outside the batch
     untouched; train_minibatch returns version t and the shard holds version = step = t;
  4. the model's dense tensors after the step == the PS's pre-step dense parameters bit for bit: what _get_model
     (eager) or _pull_dense_into_model (inside the captured graph) wrote into them.
Batches are conditioned as in test_gpu_engine_bench_path.py: dense rows of samples with a pre-activation within
1e-4 * M of a ReLU kink are redrawn against the state the step will start from.

The first step is the init handshake: its _get_model finds the shard uninitialised and pushes the model's own
tensors (PushModel, server.go:209-221), with the worker's version -1.  The reference keeps the shard's version at 0
then (model.go:84-86 only takes a version >= 1) and counts no optimizer step, so the first push is Adam step 1 with
zero slots from the model's initial values, and leaves version 1; this test pins that.

The torch tower's batch reductions run in cuBLAS and torch kernels whose summation order is theirs; the bound is
taken with the device's SM count, as for the hand-written towers, and holds with room: on an H100 80GB HBM3 (132
SMs, 400 W power limit) the worst err / bound over all legs and steps was loss 0.0016, grads 0.0082, gsum_wide 0.018,
gsum_deep 0.019.
"""
import types

import numpy as np
import pytest
import torch

from bench import ADAM_ARGS
from oracle import ps_oracle as O
from oracle import tower_oracle as T
from tests.test_gpu_engine_bench_path import (BENCH_B, BETA1, BETA2, DEV, EPS, FULL_SCAN_ROWS, LR, SAMPLE_ROWS,
                                              _check_dedup, _condition, _dense, _n_sm, _oracle_dedup, _rows, _tables)

pytestmark = pytest.mark.gpu
# the model's dense parameters in the order of the tower reference's flat layout (T.flatten)
DENSE_NAMES = ["tower.dense_linear.weight", "tower.dnn.0.weight", "tower.dnn.0.bias", "tower.dnn.1.weight",
               "tower.dnn.1.bias", "tower.dnn_logit.weight"]


def _layout(model, B):
    """What the engine test's helpers read from an engine, for the model's tables and dense parameters."""
    G = len(model.deep)
    params = [(n, tuple(p.shape)) for n, p in model.named_parameters()]
    assert [n for n, _ in params] == DENSE_NAMES, params
    o = T.layout(G)
    flat_views = [(o["wd"], T.ND), (o["w1"], T.H1 * o["in"]), (o["b1"], T.H1), (o["w2"], T.H2 * T.H1),
                  (o["b2"], T.H2), (o["w3"], T.H2)]
    assert [n for _, n in flat_views] == [int(np.prod(s)) for _, s in params]
    return types.SimpleNamespace(G=G, B=B, D=T.D, device=DEV, params=params, flat_views=flat_views,
                                 wide_names=[layer.embedding_weight_name for layer in model.wide],
                                 deep_names=[layer.embedding_weight_name for layer in model.deep],
                                 rows=[layer.input_dim for layer in model.deep])


def _record(group, monkeypatch):
    """Wrap the group's push_rows / push_dense / unique and the per-layer ops.unique so that every call appends to
    the returned log ("rows" | "dense", table name, ids, n_dev, values) or ("unique", segments, bounds, uniq, inv,
    n_unique).
    The wrappers keep tensor references only -- no host read, no sync -- so they run inside a CUDA-graph capture
    too; the tensors recorded there are the graph's own, and every replay rewrites them."""
    from elasticdl_b200 import ops

    log = []

    def pushes(fn, kind, dense):
        def call(items):
            items = list(items)
            names = {group.lookup(n)[0]: n for n in group.tables if group.lookup(n)[2] == dense}
            log.extend((kind, names[tid], ids, n_dev, values) for tid, _, ids, n_dev, values in items)
            return fn(items)
        return call

    def uniques(fn):
        def call(ids, n_seg=1, bounds=None):
            out = fn(ids, n_seg, bounds=bounds) if bounds is not None else fn(ids, n_seg)
            log.append(("unique", n_seg, bounds) + tuple(out))
            return out
        return call

    monkeypatch.setattr(group, "push_rows", pushes(group.push_rows, "rows", False))
    monkeypatch.setattr(group, "push_dense", pushes(group.push_dense, "dense", True))
    monkeypatch.setattr(group, "unique", uniques(group.unique))
    monkeypatch.setattr(ops, "unique", uniques(ops.unique))
    return log


def _pushed(log):
    """({table: (ids, values [n, dim])} of the row pushes, cut at n_dev (or all ids), {name: values} of the dense
    pushes); device tensors.  Every table is pushed once."""
    rows, dense = {}, {}
    for kind, name, ids, n_dev, values in (e for e in log if e[0] != "unique"):
        assert name not in rows and name not in dense, "%s pushed twice in one step" % name
        if kind == "dense":
            dense[name] = values
        else:
            n = ids.numel() if n_dev is None else int(n_dev[0])
            rows[name] = (ids[:n], values.reshape(ids.numel(), -1)[:n])
    return rows, dense


def _pre_state(group, lay, model, dedup, sample, t):
    """What step t starts from: param / m / v of the batch's unique rows of every table (oracle order) and of a fixed
    sample of every table's rows, the dense parameters and their slots, the shard state.  Before the first step the
    PS holds no dense parameters: the handshake of that step pushes the model's initial tensors, with zero slots."""
    tabs = {name: (_rows(group, name, dedup[g][0]), _rows(group, name, sample[g])) for name, g, _ in _tables(lay)}
    if t == 1:
        dense = {}
        for name, p in model.named_parameters():
            p0 = p.detach().cpu().numpy().reshape(-1).copy()
            dense[name] = (p0, np.zeros_like(p0), np.zeros_like(p0))
    else:
        dense = _dense(group, lay)
    return tabs, dense, group.snapshot()


def _check_dedups(log, dedup, lay, batched, what):
    """Check 1, on the dedups the step ran: the batched lookups run ONE dedup of all 38 groups, bounded by the layers'
    input_dim, shared by the deep and wide layers; the per-layer path one hashed dedup per layer call (deep layers
    first, then wide, as the model calls them)."""
    G, B = lay.G, lay.B
    calls = [e[1:] for e in log if e[0] == "unique"]
    if batched:
        assert len(calls) == 1, "%s: %d dedups, the batched lookups run one" % (what, len(calls))
        (n_seg, bounds, uniq, inv, n_unique), = calls
        assert n_seg == G and bounds is not None and list(bounds) == lay.rows, (what, n_seg, bounds)
        n = n_unique.cpu().numpy()
        uniq, inv = uniq.view(G, B).cpu().numpy(), inv.view(G, B).cpu().numpy()
        _check_dedup([(uniq[g, :n[g]], inv[g]) for g in range(G)], dedup, what + " batched dedup")
    else:
        assert len(calls) == 2 * G, "%s: %d dedups, the per-layer path runs one per layer" % (what, len(calls))
        got = []
        for i, (n_seg, bounds, uniq, inv, n_unique) in enumerate(calls):
            assert n_seg == 1 and bounds is None and uniq.numel() == B, (what, i, n_seg, bounds, uniq.numel())
            got.append((uniq[:int(n_unique[0])].cpu().numpy(), inv.cpu().numpy()))
        _check_dedup(got, dedup + dedup, what + " per-layer dedup (deep layers, then wide)")


def _check_step(group, lay, model, t, loss, version, log, dedup, ref, pre, sample, batched, what):
    """Checks 1-4 of step t (1-based count of pushes this group has seen)."""
    G, B, D = lay.G, lay.B, lay.D
    tabs, dense0, snap0 = pre
    # the shard before the step: not initialised before the handshake; version = step = t - 1 after it
    assert snap0 == [(t - 1, t - 1, t > 1)], (what, snap0)
    assert version == t, (what, version)
    rows, dense = _pushed(log)
    # 1. dedup: every dedup the step ran, and the ids pushed for every table
    _check_dedups(log, dedup, lay, batched, what)
    assert sorted(rows) == sorted(lay.wide_names + lay.deep_names), (what, sorted(rows))
    assert sorted(dense) == sorted(DENSE_NAMES), (what, sorted(dense))
    for name, g, fam in _tables(lay):
        n_dev = [e[3] for e in log if e[0] == "rows" and e[1] == name][0]
        assert (n_dev is not None) == batched, "%s: %s pushed with n_dev %r" % (what, name, n_dev)
        ids = rows[name][0].cpu().numpy()
        assert len(ids) == len(dedup[g][0]), "%s: %s pushed %d ids, oracle %d" % (what, name, len(ids), len(dedup[g][0]))
        assert np.array_equal(ids, dedup[g][0]), "%s: %s pushed ids != the oracle's dedup of group %d" % (what, name, g)
    # 4. the model's dense tensors hold the pre-step dense parameters
    for name, p in model.named_parameters():
        assert np.array_equal(p.detach().cpu().numpy().reshape(-1), dense0[name][0]), (
            "%s: the model's %s != the PS's pre-step value" % (what, name))
    # 2. loss, pushed dense and row gradients within the float64 reference's bound
    gsum_w = torch.zeros((G, B), dtype=torch.float32, device=DEV)
    gsum_d = torch.zeros((G, B, D), dtype=torch.float32, device=DEV)
    for g in range(G):
        n = len(dedup[g][0])
        gsum_w[g, :n] = rows[lay.wide_names[g]][1].reshape(n)
        gsum_d[g, :n] = rows[lay.deep_names[g]][1].reshape(n, D)
    got = {"loss": loss, "grads": T.flatten([dense[n] for n in DENSE_NAMES], G), "gsum_wide": gsum_w,
           "gsum_deep": gsum_d}
    worst = T.check(got, ref, families=("loss", "grads", "gsum_wide", "gsum_deep"), label=what, n_sm=_n_sm())
    # 3. push: oracle Adam (step t, lr 1e-3) on the pushed gradients, from the pre-step state, bit for bit
    for name, g, fam in _tables(lay):
        u = dedup[g][0]
        (p0, m0, v0), sample0 = tabs[name]
        want = [x.copy() for x in (p0, m0, v0)]
        O.np_adam(rows[name][1].cpu().numpy().copy(), *want, LR, t, BETA1, BETA2, EPS)
        for kind, a, b in zip(("param", "m", "v"), _rows(group, name, u), want):
            assert np.array_equal(a, b), "%s: %s %s of the pushed rows != oracle Adam (max |diff| %g)" % (
                what, name, kind, float(np.abs(a - b).max()))
        keep = ~np.isin(sample[g], u)
        for kind, a, b in zip(("param", "m", "v"), _rows(group, name, sample[g]), sample0):
            assert np.array_equal(a[keep], b[keep]), "%s: %s %s of a row outside the batch changed" % (what, name, kind)
    dense1 = _dense(group, lay)
    for name in DENSE_NAMES:
        want = [x.copy() for x in dense0[name]]
        O.np_adam(dense[name].reshape(-1).cpu().numpy().copy(), *want, LR, t, BETA1, BETA2, EPS)
        for kind, a, b in zip(("param", "m", "v"), dense1[name], want):
            assert np.array_equal(a, b), "%s: dense %s %s != oracle Adam (max |diff| %g)" % (
                what, name, kind, float(np.abs(a - b).max()))
    assert group.snapshot() == [(t, t, True)], what
    return worst


# leg: (batched lookups, CUDA graph, steps, table initializer).  bench.py's three api_path legs on its zero tables,
# and the graphed leg again on uniform tables: with zero tables step 1's FM and deep inputs are all zero
LEGS = {"graphed": (True, True, 5, "zero"), "batched": (True, False, 3, "zero"), "per_layer": (False, False, 3, "zero"),
        "graphed-uniform": (True, True, 4, "uniform")}
GRAPH_WARMUP = 2  # step 1 learns the lookup plan on the per-layer path; the capture must be a batched step


@pytest.mark.parametrize("leg", list(LEGS))
def test_api_path_matches_references_over_adam_steps(leg, monkeypatch):
    """bench.py's api_path configuration -- B = 32768, the 38 dac_ctr groups at full size, 76 Embedding layers, its
    batches -- a few steps through one of its legs, every step checked against the oracle's dedup, the float64 tower
    reference, the oracle's Adam and the PS's pre-step dense parameters; and the path every step took asserted."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, DeepFMLayersModel, synthetic_batch

    batched, graphed, n_steps, initializer = LEGS[leg]
    B = BENCH_B
    # torch's default, and what bench.py runs with: fp32 GEMMs without TF32
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    try:
        client = PSClient(group)
        client.dense_output = "torch"
        torch.manual_seed(7)
        model = DeepFMLayersModel(initializer=initializer).to(DEV)
        trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
            get_model_steps=1, batched_embedding_lookups=batched, cuda_graph=graphed, cuda_graph_warmup=GRAPH_WARMUP))
        lay = _layout(model, B)
        assert lay.rows == GROUP_ROWS
        log = _record(group, monkeypatch)
        rng = np.random.RandomState(11)
        sample = [np.arange(r) if r <= FULL_SCAN_ROWS else np.sort(rng.choice(r, SAMPLE_ROWS, replace=False))
                  for r in GROUP_ROWS]
        graph_log, graph_state, worst = None, None, {}
        for t in range(1, n_steps + 1):
            what = "%s step %d" % (leg, t)
            ids, dense, labels = synthetic_batch(B, 1234 + t - 1, DEV, "zipf")
            dedup = _oracle_dedup(ids)
            pre = _pre_state(group, lay, model, dedup, sample, t)
            ref = _condition(group, lay, ids, dense, labels, seed=t,
                             dense_params={name: v[0] for name, v in pre[1].items()})
            # the path this step takes: step 1 runs per layer (and learns the plan), then the plan is used
            if not batched:
                assert trainer._lookup_plan is False, what
            elif t == 1:
                assert trainer._lookup_plan is None, what
            else:
                plan = trainer._lookup_plan
                assert plan and sorted((k, dim, len(m)) for k, dim, m in plan) == [(B, 1, lay.G), (B, T.D, lay.G)], what
            del log[:]
            accepted, version, loss = trainer.train_minibatch(DeepFMLayersModel.features_of(ids, dense), labels)
            torch.cuda.synchronize()
            group.check()
            assert accepted, what
            if graphed:
                assert trainer.graph_fallback_reason is None, (what, trainer.graph_fallback_reason)
                if t <= GRAPH_WARMUP:
                    assert trainer._graph_state is None, what
                elif t == GRAPH_WARMUP + 1:  # captured, then replayed once
                    assert isinstance(trainer._graph_state, dict) and log, what
                    graph_state, graph_log = trainer._graph_state, list(log)
                else:  # replayed: no Python of the step ran, the tensors the capture recorded hold this step's values
                    assert trainer._graph_state is graph_state and not log, what
                    log.extend(graph_log)
            step_worst = _check_step(group, lay, model, t, loss, version, log, dedup, ref, pre, sample,
                                     batched and t > 1, what)
            for fam, r in step_worst.items():
                worst[fam] = max(worst.get(fam, 0.0), r)
        print("%s: worst err/bound per family over %d steps: %s" % (
            leg, n_steps, ", ".join("%s %.3g" % kv for kv in sorted(worst.items()))))
    finally:
        group.close()
