"""CPU tests of oracle/metrics_oracle.py (Keras AUC, MeanMetricWrapper, Accuracy, MeanSquaredError) and of the
host arithmetic of elasticdl_b200/common/evaluation_utils.py that does not need a device."""
import numpy as np
import pytest
import scipy.stats

from elasticdl_b200.common import evaluation_utils as EU
from oracle import metrics_oracle as MO


def _acc_fn(labels, outputs):  # evaluation_service_test.py:37-39: tf.equal of the int32 casts
    return np.equal(outputs.astype(np.int32), labels.astype(np.int32))


def test_reference_evaluation_service_vector():
    """elasticdl/python/tests/evaluation_service_test.py:76-94: two reports -> acc 0.25, acc_fn 0.25, mse 10.125."""
    reports = [(np.array([[1], [6], [3]], np.float32), np.array([[1], [0], [3]], np.float32)),
               (np.array([[4], [5], [6], [7], [8]], np.float32), np.array([[7], [8], [9], [10], [11]], np.float32))]
    metrics = {"acc": MO.MeanMetric(MO.accuracy), "mse": MO.MeanMetric(MO.mean_squared_error),
               "acc_fn": MO.MeanMetric(_acc_fn)}
    for outputs, labels in reports:
        for m in metrics.values():
            m.update(labels, outputs)
    assert metrics["acc"].result() == pytest.approx(0.25)
    assert metrics["acc_fn"].result() == pytest.approx(0.25)
    assert metrics["mse"].result() == pytest.approx(10.125)


def test_update_in_uneven_chunks_equals_one_update():
    """evaluation_service_test.py:183-193: the AUC of 1234 predictions is the same fed whole or in chunks; the
    counts are exact, so the chunks may be uneven."""
    rng = np.random.RandomState(0)
    labels = rng.randint(0, 2, 1234)
    preds = rng.random_sample(1234).astype(np.float32)
    whole = MO.auc_confusion(labels, preds)
    cuts = [0, 1, 7, 500, 501, 999, 1234]
    parts = [MO.auc_confusion(labels[a:b], preds[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
    for i in range(4):
        assert np.array_equal(whole[i], sum(p[i] for p in parts))
    acc_whole, acc_parts = MO.MeanMetric(MO.accuracy), MO.MeanMetric(MO.accuracy)
    acc_whole.update(labels, preds > 0.5)
    for a, b in zip(cuts[:-1], cuts[1:]):
        acc_parts.update(labels[a:b], preds[a:b] > 0.5)
    assert acc_whole.result() == acc_parts.result()


@pytest.mark.parametrize("T", [2, 3, 200, 1000])
def test_auc_equals_mann_whitney_inside_buckets(T):
    """With every prediction strictly inside a threshold bucket, the ROC points are the bucket boundaries and the
    trapezoid sum is the Mann-Whitney AUC (ties count 1/2) over the bucket indices -- independent of how the
    Keras formula is recalled."""
    rng = np.random.RandomState(T)
    thr = MO.thresholds(T).astype(np.float64)
    n = 4000
    k = rng.randint(1, T, n)  # bucket k lies in (thr[k-1], thr[k])
    preds = ((thr[k - 1] + thr[k]) / 2).astype(np.float32)
    assert np.all((preds > MO.thresholds(T)[k - 1]) & (preds < MO.thresholds(T)[k]))
    labels = (rng.random_sample(n) < 0.2 + 0.6 * k / T).astype(np.float32)
    pos, neg = k[labels != 0], k[labels == 0]
    want = scipy.stats.mannwhitneyu(pos, neg).statistic / (len(pos) * len(neg))
    assert MO.auc(labels, preds, T) == pytest.approx(want, rel=1e-12, abs=1e-12)
    assert MO.auc(labels, preds, T, dtype=np.float32) == pytest.approx(want, rel=1e-5)


def test_auc_edge_values():
    rng = np.random.RandomState(1)
    p = rng.random_sample(100).astype(np.float32)
    assert MO.auc([], np.zeros(0, np.float32)) == 0.0
    assert MO.auc(np.ones(100), p) == 0.0
    assert MO.auc(np.zeros(100), p) == 0.0
    y = (np.arange(100) % 2).astype(np.float32)
    assert MO.auc(y, np.where(y != 0, 0.9, 0.1).astype(np.float32)) == 1.0
    assert MO.auc(y, np.full(100, 0.3, np.float32)) == 0.5
    with pytest.raises(ValueError):
        MO.auc(y, np.where(y != 0, 1.5, 0.1).astype(np.float32))


def test_fractional_labels_are_positive_for_auc_and_zero_for_accuracy():
    y = np.array([0.7, 0.0, 0.7, 0.0], np.float32)
    p = np.array([0.9, 0.1, 0.8, 0.2], np.float32)
    assert MO.auc(y, p) == 1.0
    m = MO.MeanMetric(lambda labels, logits: (logits > 0.5).astype(np.int32) == labels.astype(np.int32))
    m.update(y, p)
    assert m.result() == 0.5  # 0.7 truncates to 0: only the two negatives match


def test_product_thresholds_and_formula_match_the_oracle():
    for T in (2, 3, 200, 8192):
        assert np.array_equal(EU.auc_thresholds(T), MO.thresholds(T))
    rng = np.random.RandomState(2)
    labels = rng.randint(0, 2, 5000)
    preds = rng.random_sample(5000).astype(np.float32)
    tp, fp, tn, fn, _ = MO.auc_confusion(labels, preds)
    assert EU.auc_from_counts(tp, fp, tn, fn) == MO.auc_result(tp, fp, tn, fn)
    assert EU.auc_from_counts(*[np.zeros(200)] * 4) == 0.0
