"""Numpy restatement of the Keras metrics the reference's evaluation uses -- TEST INFRASTRUCTURE.

- `auc_confusion`: tf.keras.metrics.AUC's update, written as Keras writes it: the [T, n] matrix of
  `predictions > thresholds` (fp32 against the fp32 thresholds), labels cast to bool, and the four reductions
  tp / fp / tn / fn.  Predictions that are NaN or outside [0, 1] (Keras asserts) are counted, not compared.
- `auc_result`: AUC.result() for the ROC curve with interpolation summation, in float64 or in the float32
  arithmetic TensorFlow runs it in (float32 count variables, float32 divisions and sums).
- `MeanMetric`: tf.keras.metrics.MeanMetricWrapper (float32 casts, squeezable dimensions, total / count) with
  `accuracy` and `mean_squared_error`.

Parity status: TensorFlow is not part of the reference tree, so the AUC arithmetic here is third-party arithmetic
recalled from Keras 2.5 (`metrics_utils.update_confusion_matrix_variables` and `AUC.result`), as the FTRL
arithmetic of ps_oracle is.  Pinned independently of that recollection by tests/test_oracle_eval_metrics.py:
  - the Mann-Whitney identity: predictions strictly inside threshold buckets give the Mann-Whitney AUC
    (ties = 1/2) over the bucket indices, computed with scipy.stats;
  - the edge values: empty, single-class (0.0, div_no_nan), perfect separation (1.0), all predictions equal (0.5);
  - the reference's own vector of elasticdl/python/tests/evaluation_service_test.py:76-94 for Accuracy,
    MeanSquaredError and a plain accuracy lambda (MeanMetricWrapper).
"""
import numpy as np

EPSILON = 1e-7  # keras.backend.epsilon()


def thresholds(num_thresholds):
    """AUC.__init__: [0 - eps] + [(i + 1) / (T - 1) for i < T - 2] + [1 + eps], as fp32 constants."""
    T = int(num_thresholds)
    if T < 2:
        raise ValueError("`num_thresholds` must be > 1.")
    return np.array([0.0 - EPSILON] + [(i + 1) * 1.0 / (T - 1) for i in range(T - 2)] + [1.0 + EPSILON],
                    dtype=np.float32)


def auc_confusion(labels, predictions, num_thresholds=200):
    """(tp, fp, tn, fn) int64 [T] and the number of invalid predictions, from the literal comparison matrix."""
    y = np.asarray(labels, dtype=np.float32).reshape(-1) != 0  # cast(cast(y_true, float32), bool)
    p = np.asarray(predictions, dtype=np.float32).reshape(-1)
    assert y.shape == p.shape, (y.shape, p.shape)
    ok = (p >= 0) & (p <= 1)
    y, p = y[ok], p[ok]
    thr = thresholds(num_thresholds)
    pred_is_pos = p[None, :] > thr[:, None]  # [T, n]
    label_is_pos = np.broadcast_to(y[None, :], pred_is_pos.shape)
    tp = np.sum(label_is_pos & pred_is_pos, axis=1, dtype=np.int64)
    fp = np.sum(~label_is_pos & pred_is_pos, axis=1, dtype=np.int64)
    tn = np.sum(~label_is_pos & ~pred_is_pos, axis=1, dtype=np.int64)
    fn = np.sum(label_is_pos & ~pred_is_pos, axis=1, dtype=np.int64)
    return tp, fp, tn, fn, int(np.sum(~ok))


def auc_result(tp, fp, tn, fn, dtype=np.float64):
    """AUC.result(), ROC + interpolation summation, in `dtype` (np.float32: TensorFlow's arithmetic)."""
    tp, fp, tn, fn = (np.asarray(v).astype(dtype) for v in (tp, fp, tn, fn))

    def div_no_nan(a, b):
        out = np.zeros_like(a)
        np.divide(a, b, out=out, where=b != 0)
        return out

    recall = div_no_nan(tp, tp + fn)
    fp_rate = div_no_nan(fp, fp + tn)
    heights = (recall[:-1] + recall[1:]) / dtype(2.0)
    return np.sum((fp_rate[:-1] - fp_rate[1:]) * heights, dtype=dtype)


def auc(labels, predictions, num_thresholds=200, dtype=np.float64):
    tp, fp, tn, fn, invalid = auc_confusion(labels, predictions, num_thresholds)
    if invalid:
        raise ValueError("%d predictions are NaN or outside [0, 1]" % invalid)
    return auc_result(tp, fp, tn, fn, dtype)


def accuracy(y_true, y_pred):
    assert y_true.shape == y_pred.shape, (y_true.shape, y_pred.shape)
    return (y_true == y_pred).astype(np.float32)


def mean_squared_error(y_true, y_pred):
    return np.mean(np.square(y_pred - y_true), axis=-1)


class MeanMetric:
    """MeanMetricWrapper(fn): float32 casts, remove_squeezable_dimensions, total / count (float64 here)."""

    def __init__(self, fn):
        self.fn, self.total, self.count = fn, 0.0, 0

    def update(self, y_true, y_pred):
        y_true = np.asarray(y_true, dtype=np.float32)
        y_pred = np.asarray(y_pred, dtype=np.float32)
        if y_pred.ndim - y_true.ndim == 1 and y_pred.shape[-1] == 1:
            y_pred = y_pred[..., 0]
        elif y_true.ndim - y_pred.ndim == 1 and y_true.shape[-1] == 1:
            y_true = y_true[..., 0]
        values = np.asarray(self.fn(y_true, y_pred)).astype(np.float32)
        self.total += float(np.sum(values, dtype=np.float64))
        self.count += values.size

    def result(self):
        return self.total / self.count if self.count else 0.0
