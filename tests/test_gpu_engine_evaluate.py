"""Forward-only evaluate() of the engines (DeepFMPSEngine for its four models, FrappeDeepFMEngine hashed and
bounded, CensusWideDeepEngine) and EvaluationMetrics on the drop-in trainer's evaluation result.

After a few training steps: evaluate()'s logits equal predict()'s bit for bit (where predict() exists); the
summary equals oracle/metrics_oracle.py fed the same logits and the same torch.sigmoid probabilities (a numpy
sigmoid can differ by an ulp at a threshold); every dense parameter, every table row and every shard version is
bitwise unchanged (hashed tables may gain the rows evaluate()'s pulls create).  Two engines on two streams add to
one shared AUC."""
import types

import numpy as np
import pytest
import torch

from elasticdl_b200.common import evaluation_utils as EU
from elasticdl_b200.ps import PSGroup
from elasticdl_b200.workloads import census as C
from elasticdl_b200.workloads import deepfm as DF
from elasticdl_b200.workloads import frappe as FR
from elasticdl_b200.workloads.census_features import synthetic_raw_batch
from oracle import metrics_oracle as MO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
ADAM = ("Adam", "learning_rate=0.01;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")


def _eval_labels(B, seed):
    """0 / 1 labels with some 0.7: positive for the AUC, 0 for the accuracy's int cast."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.tensor([0.0, 1.0, 0.7], device=DEV)[torch.randint(0, 3, (B,), generator=g, device=DEV)]


def _oracle_summary(logits, labels, logit_threshold):
    """The oracle's summary of eval_metrics_fn() fed the engine's logits and torch.sigmoid of them."""
    acc = MO.MeanMetric(lambda y, lg: (lg.reshape(-1) > logit_threshold).astype(np.int32)
                        == y.reshape(-1).astype(np.int32))
    lg = np.concatenate([t.cpu().numpy() for t in logits])
    probs = np.concatenate([torch.sigmoid(t).cpu().numpy() for t in logits])
    y = np.concatenate([t.cpu().numpy() for t in labels])
    acc.update(y, lg)
    return {"logits": {"accuracy": acc.result()}, "probs": {"auc": float(MO.auc(y, probs))}}


def _assert_summary(got, want):
    assert got["logits"]["accuracy"] == want["logits"]["accuracy"]
    assert got["probs"]["auc"] == pytest.approx(want["probs"]["auc"], rel=0, abs=1e-12)
    assert 0.0 <= got["probs"]["auc"] <= 1.0


def _assert_same(before, after):
    assert before.keys() == after.keys()
    for k in before:
        assert torch.equal(before[k], after[k]), k


# ------------------------------------------------------------------ DeepFM engine, four models
ROWS = [7, 11, 1000, 5000]


def _deepfm_state(group, eng):
    out = group.pull_dense([n for n, _ in eng.params])
    for names in (eng.wide_names, eng.deep_names):
        for n, r in zip(names, ROWS):
            out[n] = group.pull_rows([(n, torch.arange(r, device=DEV))])[0]
    return out


@pytest.mark.parametrize("model", ["deepfm", "dcn", "wide_deep", "xdeepfm"])
def test_deepfm_engine_evaluate(model):
    B = 512
    group = PSGroup(1, *ADAM, device=0)
    eng = DF.DeepFMPSEngine(group, B, group_rows=ROWS, model=model)
    for s in range(3):
        eng.step(*DF.synthetic_batch(B, 100 + s, DEV, "zipf", group_rows=ROWS))
    torch.cuda.synchronize()
    state, versions = _deepfm_state(group, eng), group.snapshot()
    metrics = EU.EvaluationMetrics(DF.eval_metrics_fn())
    logits, labels = [], []
    for s in range(2):
        ids, dense, _ = DF.synthetic_batch(B, 200 + s, DEV, "zipf", group_rows=ROWS)
        want = eng.predict(ids, dense).clone()
        y = _eval_labels(B, s)
        got = eng.evaluate(ids, dense, y, metrics)
        torch.cuda.synchronize()
        assert torch.equal(got, want)
        logits.append(got.clone())
        labels.append(y)
    group.check()
    _assert_summary(metrics.get_evaluation_summary(), _oracle_summary(logits, labels, 0.5))
    _assert_same(state, _deepfm_state(group, eng))
    assert group.snapshot() == versions
    group.close()


# ------------------------------------------------------------------ frappe engine
def _frappe_state(group, hashed):
    out = group.pull_dense(FR.DENSE_NAMES)
    for n in (FR.DEEP_NAME, FR.WIDE_NAME):
        if hashed:  # the rows that exist now
            for s in range(group.n_shards):
                ids = group.table_ids(n, s)
                out[(n, s)] = (ids, group.pull_rows([(n, ids)])[0])
        else:
            out.update(group.pull_dense([n]))
    return out


def _assert_frappe_same(before, group, hashed):
    for k, v in before.items():
        if isinstance(v, tuple):  # hashed: the same rows (sorted by id) hold the same values
            ids, rows = v
            order = torch.argsort(ids)
            assert torch.equal(group.pull_rows([(k[0], ids[order])])[0], rows[order]), k
        else:
            assert torch.equal(group.pull_dense([k])[k], v), k


@pytest.mark.parametrize("hashed", [True, False])
def test_frappe_engine_evaluate(hashed):
    B = 1000
    group = PSGroup(2, *ADAM, device=0)
    eng = FR.FrappeDeepFMEngine(group, B, 0.01, input_dim=None if hashed else FR.INPUT_DIM, seed=3,
                                expected_rows=1 << 14)
    for s in range(3):
        eng.step(*FR.synthetic_frappe_batch(B, 10 + s, DEV, pad_fraction=0.3))
    torch.cuda.synchronize()
    state, versions = _frappe_state(group, hashed), group.snapshot()
    metrics = EU.EvaluationMetrics(FR.eval_metrics_fn())
    logits, labels = [], []
    for s in range(2):
        ids, _ = FR.synthetic_frappe_batch(B, 50 + s, DEV, pad_fraction=0.3, zipf_s=0.8)  # new ids for hashed
        want = eng.predict(ids)
        y = _eval_labels(B, s)
        got = eng.evaluate(ids, y, metrics)
        assert got.data_ptr() == eng.tower.logits.data_ptr()
        torch.cuda.synchronize()
        assert torch.equal(got, want)
        logits.append(got.clone())
        labels.append(y)
    eng.check()
    _assert_summary(metrics.get_evaluation_summary(), _oracle_summary(logits, labels, 0.0))
    _assert_frappe_same(state, group, hashed)
    assert group.snapshot() == versions
    group.close()


def test_two_frappe_engines_on_two_streams_share_one_auc():
    B = 4096
    group = PSGroup(1, *ADAM, device=0)
    ea = FR.FrappeDeepFMEngine(group, B, 0.01, input_dim=FR.INPUT_DIM, seed=5)
    eb = FR.FrappeDeepFMEngine(group, B, 0.01, input_dim=FR.INPUT_DIM, register=False)
    auc = EU.AUC()
    metrics = [EU.EvaluationMetrics({"probs": {"auc": auc}}) for _ in range(2)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(2)]
    batches = [FR.synthetic_frappe_batch(B, 70 + w, DEV) for w in range(2)]
    main = torch.cuda.current_stream()
    logits = []
    for eng, m, st, (ids, y) in zip((ea, eb), metrics, streams, batches):
        st.wait_stream(main)
        with torch.cuda.stream(st):
            logits.append(eng.evaluate(ids, y, m))
    for st in streams:
        main.wait_stream(st)
    probs = np.concatenate([torch.sigmoid(lg).cpu().numpy() for lg in logits])
    y = np.concatenate([b[1].cpu().numpy() for b in batches])
    got, want = auc.confusion(), MO.auc_confusion(y, probs)
    for g, w in zip(got[:4], want[:4]):
        assert np.array_equal(g.astype(np.int64), w)
    assert metrics[0].get_evaluation_summary()["probs"]["auc"] == pytest.approx(float(MO.auc(y, probs)), abs=1e-12)
    group.close()


# ------------------------------------------------------------------ census engine
def test_census_engine_evaluate():
    B = 700
    group = PSGroup(2, *ADAM, device=0)
    eng = C.CensusWideDeepEngine(group, B, 0.01, seed=2)
    for s in range(3):
        numeric, strings, _, _ = synthetic_raw_batch(B, 30 + s, DEV)
        eng.step(numeric, strings, _eval_labels(B, 90 + s).round())
    loss = eng.tower.loss.clone()
    torch.cuda.synchronize()
    names = [n for n, _ in C.PARAMS]
    state, versions = group.pull_dense(names), group.snapshot()
    metrics = EU.EvaluationMetrics(C.eval_metrics_fn())
    logits, labels = [], []
    for s in range(2):
        numeric, strings, _, _ = synthetic_raw_batch(B, 60 + s, DEV)
        y = _eval_labels(B, s)
        got = eng.evaluate(numeric, strings, y, metrics)
        ids, _ = eng.transform(numeric, strings)
        ref = C.census_tower(ids.to(torch.int32).contiguous(), y, eng.flat)  # the training kernel's logits
        assert torch.equal(got, ref["logits"])
        logits.append(got.clone())
        labels.append(y)
    eng.check()
    assert torch.equal(eng.tower.loss, loss)  # the step's buffers are not evaluate()'s
    _assert_summary(metrics.get_evaluation_summary(), _oracle_summary(logits, labels, 0.5))
    _assert_same(state, group.pull_dense(names))
    assert group.snapshot() == versions
    group.close()


# ------------------------------------------------------------------ drop-in trainer
class _FrappeWithProbs(FR.FrappeDeepFM):
    """The torch twin with the outputs the reference's frappe models return: {"logits", "probs"}."""

    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        bce = torch.nn.BCEWithLogitsLoss()
        self.loss = lambda labels, outputs: bce(outputs["logits"], labels)

    def forward(self, features):
        logits = super().forward(features)
        return {"logits": logits, "probs": torch.sigmoid(logits).reshape(-1, 1)}


def test_dropin_trainer_evaluation_result():
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    B = 256
    group = PSGroup(1, "SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", device=0)
    model = _FrappeWithProbs(0.1, input_dim=FR.INPUT_DIM).to(DEV)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(cuda_graph=False))
    for s in range(3):
        accepted, _, _ = trainer.train_minibatch(*FR.synthetic_frappe_batch(B, 300 + s, DEV, pad_fraction=0.3))
        assert accepted
    for s in range(2):
        ids, _ = FR.synthetic_frappe_batch(B, 400 + s, DEV, pad_fraction=0.3)
        trainer.evaluate_minibatch(ids, _eval_labels(B, s))
    result = trainer.get_evaluation_result()
    metrics = EU.EvaluationMetrics(FR.eval_metrics_fn())
    metrics.update_evaluation_metrics(result[EU.MODEL_OUTPUT], result[EU.LABEL])
    logits = [o["logits"] for o in result[EU.MODEL_OUTPUT]]
    probs = np.concatenate([o["probs"].cpu().numpy() for o in result[EU.MODEL_OUTPUT]])
    y = np.concatenate(result[EU.LABEL])
    want = _oracle_summary(logits, [torch.from_numpy(v) for v in result[EU.LABEL]], 0.0)
    want["probs"]["auc"] = float(MO.auc(y, probs))  # the model's own torch.sigmoid probabilities
    _assert_summary(metrics.get_evaluation_summary(), want)
    group.close()
