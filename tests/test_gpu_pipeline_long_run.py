"""The one-shard lookahead pipeline over long runs, checked against the float64 towers and the oracle's Adam.

On one shard a lookahead step prepares the next one beside its row push (DeepFMPSEngine.tail_prep): it pulls the
dense parameters and runs the next step's tower prologue, which clears the other plan's accumulator set over the
live rows recorded when that set was last filled (_acc_rows).  That is only right while every row outside a set's
recorded live rows is exactly 0: entering the pipeline clears both sets whole (_zero_accs), and every tail keeps it.

Batches that make a wrong clear visible: "W" gives every group min(B, rows) distinct ids (n_unique as large as it
can be), "N" draws every group from at most 4 ids.  The plans alternate, so SEQUENCE gives each accumulator set
W -> N -> W -> W and ends on N W N: a clear over too few rows (the counts of the wrong plan or step) leaves stale
gradients inside a later W batch's live rows, and one over too many wipes rows the running step still pushes.

Every training step is checked as test_gpu_engine_bench_path.py checks bench.py's step (the dedup exactly, the float64
tower bound, the oracle's Adam bit for bit on the pushed rows, rows outside the batch untouched, the loss ring), and
every lookahead step also against the pipeline's state (_check_pipeline_state): the set it trained holds nothing at
or past its batch's n_unique; the set the next step accumulates into holds exactly what the prologue writes (0, and
DCN's L2 terms) over its whole buffer; the dense parameters pulled for the next step are what the PS holds; the
other plan holds the next batch's dedup.  The legs: bench.py's headline and host feeder at its configuration;
predict(), evaluate(), eager step(), step(ev=) (bench.py's event-timed pass), step_graph and a restart after
set_dense in the middle of a run, for the four dac_ctr models; a dense write without a restart (one step stale,
DESIGN.md section 10); the event-timed pass at bench.py's configuration and its kernel report; and three mutations
of the engine that these checks must catch.
"""
import numpy as np
import pytest
import torch

from oracle import tower_oracle as T
from tests import test_gpu_dcn_tower as DCN
from tests import test_gpu_engine_evaluate as EV
from tests import test_gpu_wide_deep_tower as WD
from tests import test_gpu_xdeepfm_tower as XD
from tests.test_gpu_engine_bench_path import (BENCH_B, DEV, EDGE_ROWS, FULL_SCAN_ROWS, SAMPLE_ROWS, _check_dedup,
                                              _check_push, _check_step, _condition, _n_sm, _oracle_dedup,
                                              _plan_dedup, _pre_state)
from tests.test_gpu_step_head import _dense as _ps_dense

pytestmark = pytest.mark.gpu
SEQUENCE = "WWNNWWWWNWN"  # set 0 trains W N W W N N, set 1 W N W W W (step 10: a W between two N)
SMALL_B = 4096


def _batch(kind, B, seed, rows):
    """[ids int64 [G, B], dense, labels] on the device: synthetic_batch's ("Z"), its ids replaced by min(B, rows)
    distinct ids per group, each present, shuffled ("W"), or by draws from at most 4 ids per group ("N")."""
    from elasticdl_b200.workloads.deepfm import synthetic_batch

    ids, dense, labels = synthetic_batch(B, seed, DEV, "zipf", group_rows=rows)
    if kind == "Z":
        return [ids, dense, labels]
    gen = torch.Generator(device=DEV).manual_seed(seed)
    for g, r in enumerate(rows):
        pool = torch.randperm(r, generator=gen, device=DEV)[:min(B, r) if kind == "W" else min(4, r)]
        n = pool.numel()
        if kind == "W":
            pick = torch.cat([torch.arange(n, device=DEV), torch.randint(0, n, (B - n,), generator=gen, device=DEV)])
            pick = pick[torch.randperm(B, generator=gen, device=DEV)]
        else:
            pick = torch.randint(0, n, (B,), generator=gen, device=DEV)
        ids[g] = pool[pick]
    return [ids, dense, labels]


def _check_xdeepfm_step(group, eng, t, p, dedup, ref, pre, sample, label):
    """Checks 1-4 of step t against the xDeepFM reference, its CIN masks the kernel's own bits inside the tau window
    (test_gpu_xdeepfm_tower.py)."""
    G, B, D = eng.G, eng.B, eng.D
    what = "%s step %d" % (label, t)
    _check_dedup(_plan_dedup(eng.plans[p], G, B), dedup, what + " dedup")
    inputs, ref = ref
    ref = XD.reference_with_kernel_masks(inputs, ref, eng.scratch, what)
    got = {"loss": eng.loss_buf, "grads": eng.flat_grads, "gsum_wide": eng.gsum_w.view(G, B),
           "gsum_deep": eng.gsum_d.view(G, B, D)}
    XD.X.check(got, ref, families=tuple(got), label=what, n_sm=_n_sm())
    _check_push(group, eng, t, dedup, pre, sample, what)


def _logits_check(oracle, ref_of=lambda ref: ref):
    def check(logits, ref, what):
        oracle.check({"logits": logits}, ref_of(ref), families=("logits",), label=what, n_sm=_n_sm())
    return check


# model -> (condition: the batch's float64 reference from the PS state, redrawing dense rows near a ReLU kink;
#           check_step: checks 1-4 of a step against it; check_logits: predict()'s logits against it)
MODELS = {
    "deepfm": (_condition, _check_step, _logits_check(T)),
    "dcn": (lambda group, eng, ids, dense, labels, seed: DCN._condition(group, eng, ids, dense, labels, seed),
            DCN._check_step, _logits_check(DCN.R)),
    "wide_deep": (lambda group, eng, ids, dense, labels, seed: WD._condition(group, eng, ids, dense, labels, seed),
                  WD._check_step, _logits_check(WD.T)),
    "xdeepfm": (lambda group, eng, ids, dense, labels, seed: XD._condition(group, eng, ids, dense, labels, seed),
                _check_xdeepfm_step, _logits_check(XD.X, lambda ref: ref[1])),
}


def _prologue_outputs(eng, model):
    """What the tower prologue leaves in a set's gradients and loss: 0, but DCN's CrossNet L2 (2 * L2 * w on the
    cross kernels, as the kernel rounds it, and L2 * |w|^2)."""
    grads, loss = torch.zeros_like(eng.flat_grads), 0.0
    if model == "dcn":
        lay = DCN.R.layout(eng.G)
        cw = eng.flat_params[lay["cw"]:lay["cb"]]
        grads[lay["cw"]:lay["cb"]] = cw * float(np.float32(2) * np.float32(DCN.R.L2))
        loss = DCN.R.L2 * float((cw.double() ** 2).sum())
    return grads, loss


def _check_pipeline_state(group, eng, model, dedup, what):
    """The pipeline after a lookahead step (synchronised) that trained on the batch of `dedup`."""
    G, B, D = eng.G, eng.B, eng.D
    assert eng._ready == eng.tail_prep, what
    if not eng.tail_prep:  # xDeepFM: one accumulator set, every step prepares itself
        assert len(eng._accs) == 1, what
        return
    # the set this step trained: nothing at or past its batch's live rows
    dead = torch.arange(B, device=DEV).unsqueeze(0) >= torch.tensor([len(u) for u, _ in dedup], device=DEV).unsqueeze(1)
    for name, x in (("gsum_w", eng.gsum_w.view(G, B)), ("gsum_d", eng.gsum_d.view(G, B, D))):
        bad = int(torch.count_nonzero(x[dead]))
        assert bad == 0, "%s: %d values of the trained set's %s at or past n_unique are not 0" % (what, bad, name)
    # the set the next step accumulates into, over all G * B rows: what the prologue leaves
    nxt = eng._accs[eng._plan_acc[eng.cur]]
    assert nxt["gsum_w"] is not eng.gsum_w, what
    for name in ("gsum_w", "gsum_d"):
        bad = int(torch.count_nonzero(nxt[name]))
        assert bad == 0, "%s: %d values of the next step's %s are not 0" % (what, bad, name)
    grads, loss = _prologue_outputs(eng, model)
    assert torch.equal(nxt["flat_grads"], grads), "%s: the next step's gradients are not the prologue's (max |diff| %g)" % (
        what, float((nxt["flat_grads"] - grads).abs().max()))
    assert float(nxt["loss_buf"]) == pytest.approx(loss, rel=1e-5, abs=0), (what, float(nxt["loss_buf"]), loss)
    # the dense parameters the next step trains on
    ps = _ps_dense(group, eng)
    for (name, _), (off, n) in zip(eng.params, eng.flat_views):
        assert torch.equal(eng.flat_params[off:off + n], ps[off:off + n]), "%s: pulled %s != the PS's" % (what, name)


def _write_dense(group, eng, seed):
    """Dense parameters on the PS: half of what it holds plus seeded noise."""
    torch.cuda.synchronize()
    gen = torch.Generator(device=DEV).manual_seed(seed)
    now = group.pull_dense([n for n, _ in eng.params])
    group.set_dense([(n, torch.as_tensor(now[n], device=DEV) * 0.5
                      + 0.02 * torch.randn(tuple(now[n].shape), generator=gen, device=DEV)) for n, _ in eng.params])


def _run(model, rows, B, script, feed="device", fresh="W", seed=0, fresh_seed=None, label=""):
    """A fresh group and engine (bench.py's Adam and narrow id transport, `model` over `rows`, batch B) driven
    through `script`, every training step checked.  Tokens: "W" / "N", a lookahead step on such a batch (the next
    lookahead batch loaded beside it), on the graphed pipeline (feed "device": prepare_packed + step_ahead_graph)
    or through host_feeder(3, lookahead=True) (feed "host", lookahead steps only).  Between them:
      predict, evaluate   forward only on the loaded batch; the pipeline goes on;
      step, step_ev, graph   step(), step(ev=) behind a spin kernel, or capture() + step_graph() on a fresh int64
                          batch of kind `fresh`; the pipeline restarts (prepare_packed of the loaded batch);
      set_dense           new dense parameters on the PS, and a restart;
      write               new dense parameters on the PS, no restart: the next step trains on the ones pulled
                          before the write and pushes onto the PS's (one step stale, DESIGN.md section 10).
    The first lookahead step after anything but a lookahead step must enter the pipeline again (_zero_accs, then
    its own pull and prologue).  Returns (kernel_report of the step(ev=) calls, the engine's push kernel names)."""
    from bench import ADAM_ARGS
    from elasticdl_b200.common import evaluation_utils as EU
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, eval_metrics_fn, pack_batch, packed_views

    condition, check_step, check_logits = MODELS[model]
    kinds = [tok for tok in script if tok in ("W", "N")]
    ahead = [_batch(kind, B, seed + i, rows) for i, kind in enumerate(kinds + ["W"] if kinds else [])]
    fresh_seed = seed + 1000 if fresh_seed is None else fresh_seed
    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    try:
        eng = DeepFMPSEngine(group, B, group_rows=rows, id_transport="narrow", model=model)
        assert eng.tower_kind == "tile" and eng.row_source == "table", (eng.tower_kind, eng.row_source)
        assert eng.tail_prep == (model != "xdeepfm")
        G = eng.G
        rng = np.random.RandomState(11)
        sample = [np.arange(r) if r <= FULL_SCAN_ROWS else np.sort(rng.choice(r, SAMPLE_ROWS, replace=False))
                  for r in rows]
        entries, zero_accs = [0], eng._zero_accs

        def counted_zero_accs():
            entries[0] += 1
            zero_accs()

        eng._zero_accs = counted_zero_accs
        if feed == "host":  # batch 1 is conditioned before it is packed, later ones in the static buffer
            condition(group, eng, *ahead[0], seed=1)
            src = [(pack_batch(*(x.cpu() for x in b), pin=True, widths=eng.widths),) for b in ahead]
            feeder = eng.host_feeder(3, lookahead=True)
            for s in src[:2]:
                feeder.submit(*s)
                torch.cuda.synchronize()
        t = k = 0  # pushes so far; the lookahead batch loaded (or to load)
        started, stale, ev, uniq = feed == "host", False, {}, []
        for i, tok in enumerate(script):
            what = "%s %s#%d" % (label, tok, i)
            if tok in ("W", "N"):
                ids, dense, labels = ahead[k]
                kw = {}
                if stale:  # the write is not seen yet: the step trains on what the last one pulled
                    assert eng._ready, what
                    kw["dense_params"] = {name: eng.flat_params[off:off + n].clone()
                                          for (name, _), (off, n) in zip(eng.params, eng.flat_views)}
                    ps = _ps_dense(group, eng)
                    assert all(not torch.equal(eng.flat_params[off:off + n], ps[off:off + n])
                               for off, n in eng.flat_views), what
                ref = condition(group, eng, ids, dense, labels, seed=seed + i, **kw)
                if started:
                    packed_views(eng.s_packed[eng.cur], G, B, eng.widths)[1].copy_(dense)
                else:
                    eng.prepare_packed(pack_batch(ids, dense, labels, widths=eng.widths))
                    started = True
                    assert not eng._ready, what  # a new pipeline pulls what the PS holds now
                dedup = _oracle_dedup(ids)
                pre = _pre_state(group, eng, dedup, sample)
                p, ready, n0 = eng.cur, eng._ready, entries[0]
                if feed == "device":
                    eng.step_ahead_graph(pack_batch(*ahead[k + 1], widths=eng.widths))
                else:
                    if k + 2 < len(src):
                        feeder.submit(*src[k + 2])
                        torch.cuda.synchronize()
                    feeder.run_next()
                torch.cuda.synchronize()
                group.check()
                t, k, stale = t + 1, k + 1, False
                check_step(group, eng, t, p, dedup, ref, pre, sample, what)
                _check_dedup(_plan_dedup(eng.plans[eng.cur], G, B), _oracle_dedup(ahead[k][0]),
                             what + " next-batch dedup")
                assert entries[0] == n0 + (eng.tail_prep and not ready), (what, "pipeline entry", ready, entries, n0)
                _check_pipeline_state(group, eng, model, dedup, what)
                continue
            assert feed == "device", "interleavings run on the graphed pipeline"
            if tok in ("predict", "evaluate"):
                ids, dense, labels = ahead[k]
                ref = condition(group, eng, ids, dense, labels, seed=seed + i)
                if started:
                    packed_views(eng.s_packed[eng.cur], G, B, eng.widths)[1].copy_(dense)
                if tok == "predict":
                    logits = eng.predict(ids, dense)
                else:
                    metrics, y = EU.EvaluationMetrics(eval_metrics_fn()), EV._eval_labels(B, i)
                    logits = eng.evaluate(ids, dense, y, metrics)
                torch.cuda.synchronize()
                check_logits(logits, ref, what)
                if tok == "evaluate":
                    EV._assert_summary(metrics.get_evaluation_summary(), EV._oracle_summary([logits], [y], 0.5))
                assert group.snapshot() == [(t, t, True)], what
            elif tok in ("step", "step_ev", "graph"):
                ids, dense, labels = _batch(fresh, B, fresh_seed + t, rows)
                ref = condition(group, eng, ids, dense, labels, seed=seed + i)
                dedup = _oracle_dedup(ids)
                pre = _pre_state(group, eng, dedup, sample)
                if tok == "graph":
                    eng.capture()
                p = eng.cur
                if tok == "step":
                    eng.step(ids, dense, labels)
                elif tok == "step_ev":
                    torch.cuda._sleep(4_000_000)
                    eng.step(ids, dense, labels, ev=ev)
                    uniq.append(sum(len(u) for u, _ in dedup))
                else:
                    eng.step_graph(ids, dense, labels)
                torch.cuda.synchronize()
                group.check()
                t += 1
                check_step(group, eng, t, p, dedup, ref, pre, sample, what)
                started = False  # the step deduplicated into the plan the loaded batch was in
            elif tok in ("write", "set_dense"):  # set_dense: the next lookahead step starts a new pipeline
                _write_dense(group, eng, seed + i)
                stale, started = tok == "write", started and tok == "write"
                continue
            else:
                raise ValueError(tok)
            assert not eng._ready, what  # the next lookahead step enters the pipeline again
        return (eng.kernel_report(ev, uniq) if ev else {}), eng.push_names
    finally:
        group.close()


@pytest.mark.parametrize("feed", ["device", "host"])
def test_bench_pipeline_over_a_long_mixed_run(feed):
    """bench.py's configuration -- B = 32768, the 38 dac_ctr groups at full size, Adam, narrow ids -- through its
    headline feed (device buffers) or its host feeder (pinned buffers), SEQUENCE's W / N batches."""
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS

    _run("deepfm", GROUP_ROWS, BENCH_B, SEQUENCE, feed=feed, label="bench " + feed)


INTERLEAVED = ["W", "W", "N", "step", "N", "W", "predict", "W", "W", "evaluate", "N", "W", "step_ev", "N", "N",
               "graph", "N", "W", "set_dense", "W", "W"]


@pytest.mark.parametrize("model", ["deepfm", "dcn", "wide_deep", "xdeepfm"])
def test_pipeline_interleaved_with_everything_else(model):
    """B = 4096 over EDGE_ROWS (2 to 2e6 rows per group): a graphed lookahead run with predict(), evaluate(), an
    eager step(), step(ev=), step_graph and a restart after set_dense in it, each once; every lookahead step after
    them checked, the first one entering the pipeline again.  The eager steps that overwrite the loaded plan's
    dedup come before an N batch, so a set they filled whole is cleared by the entry, not by the N batch's prologue.
    xDeepFM prepares every step at its head."""
    _run(model, EDGE_ROWS, SMALL_B, INTERLEAVED, seed=300, label=model)


def test_dense_write_without_restart_is_one_step_stale():
    """set_dense between two lookahead steps, no prepare_packed: the next step trains on the dense parameters the
    step before it pulled and pushes its gradients onto what the PS holds; the step after it trains on the write."""
    _run("deepfm", EDGE_ROWS, SMALL_B, ["W", "W", "N", "write", "N", "W", "W", "W", "W"], seed=500, label="write")


def test_event_timed_eager_pass_at_bench_configuration():
    """bench.py's eager pass with CUDA-event pairs -- step(ev=) behind torch.cuda._sleep, the one-call tower on the
    table records -- on its batches (seeds 1234 + p), three checked steps; then kernel_report over the names
    bench.py reads."""
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS

    report, push_names = _run("deepfm", GROUP_ROWS, BENCH_B, ["step_ev"] * 3, fresh="Z", fresh_seed=1234,
                              label="step(ev)")
    assert set(report) == {"unique", "tower_fwd_bwd", *push_names}, sorted(report)
    for name, r in report.items():
        assert r["launches"] == 3 and r["ms"] > 0 and r["bytes"] > 0 and r["gbs"] > 0, (name, r)


def _other_plan_counts(orig):
    def _prepare_next(self, a, q, st):
        orig(self, a, q, st)
        # clamped: plan q's counts are unset before its first dedup
        torch.clamp(self.plans[q]["n_unique"], 0, self.B, out=self._acc_rows[self._plan_acc[self.cur]])
    return _prepare_next


def _half_counts(orig):
    def _prepare_next(self, a, q, st):
        s = self._plan_acc[q]
        if not hasattr(self, "_half_rows"):
            self._half_rows = [torch.zeros_like(r) for r in self._acc_rows]
        full = self._acc_rows[s]
        torch.div(full, 2, rounding_mode="floor", out=self._half_rows[s])
        self._acc_rows[s] = self._half_rows[s]
        try:
            orig(self, a, q, st)
        finally:
            self._acc_rows[s] = full
    return _prepare_next


MUTATIONS = ["none", "records_other_plan_counts", "clears_half_the_rows", "enters_without_clearing"]


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutations_are_caught(mutation, monkeypatch):
    """SEQUENCE at B = 4096 over EDGE_ROWS passes as the engine is ("none") and fails a check under each mutation
    of it: _prepare_next recording the other plan's counts (read while the next batch's dedup rewrites them) or
    handing the tail prologue half of the recorded counts, or no _zero_accs on entering the pipeline.  Both sets
    start at 0, so the last is only visible after a step outside the pipeline filled one: an eager step on a W
    batch, then the pipeline restarts on an N batch."""
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    script = list(SEQUENCE[:2]) + ["step"] + list(SEQUENCE[2:])
    if mutation == "none":
        _run("deepfm", EDGE_ROWS, SMALL_B, script, seed=700, label="unmutated")
        return
    if mutation == "enters_without_clearing":
        monkeypatch.setattr(DeepFMPSEngine, "_zero_accs", lambda self: None)
    else:
        wrap = _other_plan_counts if mutation == "records_other_plan_counts" else _half_counts
        monkeypatch.setattr(DeepFMPSEngine, "_prepare_next", wrap(DeepFMPSEngine._prepare_next))
    with pytest.raises(AssertionError) as caught:
        _run("deepfm", EDGE_ROWS, SMALL_B, script, seed=700, label="mutation " + mutation)
    print("%s caught: %s" % (mutation, str(caught.value).splitlines()[0]))
