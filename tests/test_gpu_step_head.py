"""On one GPU a lookahead step prepares the next one beside its own row push -- dense pull and tower prologue, the
prologue zeroing the other plan's accumulator set (DeepFMPSEngine.tail_prep) -- so the next step opens with its
tower.  It must train as the step that pulls and zeroes at its head: same losses and dense parameters over Adam
steps, through the eager and the graphed lookahead pipelines, with predict() between steps and a new pipeline
(prepare / prepare_packed) started from dense parameters set on the PS; the accumulators named on the engine are
the last step's; and the step ends with what it pulled for the next one equal to what the PS holds."""
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

ADAM = "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;"
ROWS = [7, 300, 5000, 40000]
B = 2048
STEPS = 8


def _batches(n):
    from elasticdl_b200.workloads.deepfm import synthetic_batch

    return [synthetic_batch(B, 100 + i, torch.device("cuda", 0), group_rows=ROWS) for i in range(n)]


def _dense(group, eng):
    """The PS's dense parameters in the engine's flat layout (its padding left at 0)."""
    flat = torch.zeros_like(eng.flat_params)
    for (name, _), (off, n) in zip(eng.params, eng.flat_views):
        flat[off:off + n] = group.pull_dense([name])[name].reshape(-1)
    return flat


def _set_dense(group, eng):
    torch.cuda.synchronize()
    group.set_dense([(name, torch.full_like(p, 0.01 * (k % 7 - 3))) for k, (name, p) in enumerate(eng.params)])


def _train(model, tail_prep, feed, batches):
    """Losses of STEPS steps and the dense parameters after them."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch

    group = PSGroup(1, "Adam", ADAM, device=0)
    try:
        eng = DeepFMPSEngine(group, B, group_rows=ROWS, model=model)
        assert eng.tail_prep == (model != "xdeepfm")  # xDeepFM's prologue also rewrites the CIN's scratch
        eng.tail_prep = eng.tail_prep and tail_prep
        losses, grads = [], []
        if feed == "graph":
            src = [pack_batch(*b, widths=eng.widths) for b in batches]
            eng.prepare_packed(src[0])
            for t in range(STEPS):
                eng.step_ahead_graph(src[t + 1])
                losses.append(float(eng.loss_buf))
                grads.append(eng.flat_grads.clone())
                if t == 3:
                    eng.predict(batches[t][0], batches[t][1])
                if t == 5:  # a new pipeline from dense parameters set on the PS
                    _set_dense(group, eng)
                    eng.prepare_packed(src[t + 1])
        else:
            eng.prepare(batches[0][0])
            for t in range(STEPS):
                _, dense, labels = batches[t]
                losses.append(float(eng.step_ahead(dense, labels, batches[t + 1][0])))
                assert float(eng.loss_buf) == losses[-1]
                grads.append(eng.flat_grads.clone())
                if t == 3:
                    eng.predict(batches[t][0], dense)
                if t == 5:
                    _set_dense(group, eng)
                    eng.prepare(batches[t + 1][0])
        torch.cuda.synchronize()
        group.check()
        if eng.tail_prep:  # what the last step pulled for the next one is what the PS holds
            for off, n in eng.flat_views:
                assert torch.equal(eng.flat_params[off:off + n], _dense(group, eng)[off:off + n])
        return losses, torch.stack(grads).cpu(), _dense(group, eng).cpu()
    finally:
        group.close()


@pytest.mark.parametrize("feed", ["eager", "graph"])
@pytest.mark.parametrize("model", ["deepfm", "dcn", "wide_deep", "xdeepfm"])
def test_tail_pull_trains_as_the_head_pull(model, feed):
    batches = _batches(STEPS + 1)
    got_loss, got_grads, got_dense = _train(model, True, feed, batches)
    want_loss, want_grads, want_dense = _train(model, False, feed, batches)
    # the two runs differ only in the order of the tower's float atomics
    assert got_loss == pytest.approx(want_loss, rel=1e-4, abs=1e-6), (model, feed)
    assert torch.allclose(got_grads, want_grads, rtol=1e-3, atol=1e-7), (model, feed)
    assert torch.allclose(got_dense, want_dense, rtol=1e-4, atol=1e-6), (model, feed)
