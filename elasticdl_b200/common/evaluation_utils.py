"""Evaluation metrics of the reference's master (elasticdl/python/common/evaluation_utils.py:20-94), on the GPU.

- AUC: tf.keras.metrics.AUC with its defaults (ROC curve, interpolation summation, Keras' thresholds).  One
  launch of b200_metrics_auc_update (csrc/eval_metrics.cu) adds a batch to a histogram over the threshold
  buckets; result() derives the confusion counts from it and applies Keras' formula in float64.
- MeanMetricWrapper, Accuracy, MeanSquaredError: Keras' semantics with torch ops on the device.
- EvaluationMetrics: the reference's class, fed device tensors or numpy arrays.

The state of every metric is a device tensor: an update launches kernels on the current stream and reads nothing
back; result() reads the state once.  Inputs may be torch tensors (on the metric's device or on the host) or
numpy arrays, which are copied to the metric's device.

Counts are exact int64 (AUC) and the totals float64 (MeanMetricWrapper), where Keras keeps float32 variables that
stop being exact above 2^24 per count (DESIGN.md section 4, waived divergences).
"""
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib

MODEL_OUTPUT = "output"  # MetricsDictKey.MODEL_OUTPUT (elasticdl/python/common/constants.py)
LABEL = "label"  # MetricsDictKey.LABEL
EPSILON = 1e-7  # keras.backend.epsilon()


def _device(device):
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != "cuda":
        raise ValueError("metrics keep their state on a CUDA device, not %s" % device)
    return device if device.index is not None else torch.device("cuda", torch.cuda.current_device())


def _as_float(x, device):
    """x (torch tensor, numpy array or array-like) as a float32 tensor on `device` (Keras casts both y_true and
    y_pred to float32); a tensor on another CUDA device is refused."""
    if isinstance(x, torch.Tensor):
        if x.is_cuda and x.device != device:
            raise ValueError("a tensor on %s was fed to a metric on %s" % (x.device, device))
        return x.detach().to(device=device, dtype=torch.float32)
    return torch.as_tensor(np.asarray(x), dtype=torch.float32, device=device)


class Metric:
    """What EvaluationMetrics accepts as a metric without wrapping it (tf.keras.metrics.Metric's interface)."""

    def update_state(self, y_true, y_pred):
        raise NotImplementedError

    def result(self):
        raise NotImplementedError

    def reset_states(self):
        raise NotImplementedError


def auc_thresholds(num_thresholds):
    """Keras AUC's default thresholds, float32 [T]: -eps, (i + 1) / (T - 1) for i < T - 2, 1 + eps."""
    T = int(num_thresholds)
    return np.array([0.0 - EPSILON] + [(i + 1) * 1.0 / (T - 1) for i in range(T - 2)] + [1.0 + EPSILON],
                    dtype=np.float32)


def auc_from_counts(tp, fp, tn, fn):
    """Keras' ROC AUC with interpolation summation from the confusion counts [T] of the T thresholds, in float64:
    recall = div_no_nan(tp, tp + fn), fpr = div_no_nan(fp, fp + tn), sum of (fpr[i] - fpr[i+1]) times the mean of
    recall[i] and recall[i+1]."""
    tp, fp, tn, fn = (np.asarray(v, dtype=np.float64) for v in (tp, fp, tn, fn))

    def div_no_nan(a, b):
        return np.divide(a, b, out=np.zeros_like(a), where=b != 0)

    recall, fpr = div_no_nan(tp, tp + fn), div_no_nan(fp, fp + tn)
    return float(np.sum((fpr[:-1] - fpr[1:]) * ((recall[:-1] + recall[1:]) / 2.0)))


class AUC(Metric):
    """tf.keras.metrics.AUC(num_thresholds) with its defaults: the ROC curve, interpolation summation, Keras'
    thresholds.  The state is one int64 tensor on `device` (the current CUDA device by default): hist [2][T + 1]
    (the prediction counts per threshold bucket of negatives and of positives, include/b200_metrics.h) followed by
    the count of invalid predictions.  The kernel adds to it with 64-bit atomics, so updates from several streams
    (several engines on one device) may share one AUC; multi-rank runs can all-reduce `state`."""

    def __init__(self, num_thresholds=200, name="auc", device=None):
        T = int(num_thresholds)
        if T <= 1:
            raise ValueError("`num_thresholds` must be > 1.")
        if T > _lib.METRICS_MAX_THRESHOLDS:
            raise ValueError("`num_thresholds` must be <= %d, not %d" % (_lib.METRICS_MAX_THRESHOLDS, T))
        self.num_thresholds, self.name = T, name
        self.device = _device(device)
        self.lib = _lib.lib()
        self.thresholds = torch.from_numpy(auc_thresholds(T)).to(self.device)
        self.state = torch.zeros(2 * (T + 1) + 1, dtype=torch.int64, device=self.device)

    def update_state(self, y_true, y_pred):
        """Add a batch: labels and predictions of the same number of elements ([B] or [B, 1]).  A label is
        positive iff it is non-zero; a prediction must lie in [0, 1] (result() raises otherwise)."""
        labels = _as_float(y_true, self.device).reshape(-1).contiguous()
        preds = _as_float(y_pred, self.device).reshape(-1).contiguous()
        if labels.numel() != preds.numel():
            raise ValueError("%d labels for %d predictions" % (labels.numel(), preds.numel()))
        T = self.num_thresholds
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream().cuda_stream
            rc = self.lib.b200_metrics_auc_update(preds.data_ptr(), labels.data_ptr(), preds.numel(),
                                                  self.thresholds.data_ptr(), T, self.state.data_ptr(),
                                                  self.state[2 * (T + 1):].data_ptr(), ctypes.c_void_p(st))
        _lib.check_call(rc, "b200_metrics_auc_update", self.lib.b200_metrics_last_error)

    def confusion(self):
        """(tp, fp, tn, fn) uint64 [T] and the number of invalid predictions, from one read of the state."""
        T = self.num_thresholds
        s = self.state.cpu().numpy().view(np.uint64)
        hist = s[:2 * (T + 1)].reshape(2, T + 1)
        at_least = np.cumsum(hist[:, ::-1], axis=1)[:, ::-1]  # at_least[c, k] = sum over buckets >= k
        tp, fp = at_least[1, 1:], at_least[0, 1:]  # threshold i: buckets > i
        return tp, fp, at_least[0, 0] - fp, at_least[1, 0] - tp, int(s[-1])

    def result(self):
        """The AUC as a Python float; 0.0 for an empty or single-class state.  ValueError if any prediction was
        NaN or outside [0, 1] (Keras asserts on these)."""
        tp, fp, tn, fn, invalid = self.confusion()
        if invalid:
            raise ValueError("%s: %d predictions were NaN or outside [0, 1]" % (self.name, invalid))
        return auc_from_counts(tp, fp, tn, fn)

    def reset_states(self):
        self.state.zero_()

    def merge_state(self, *others):
        """Add the counts of other AUC states of the same thresholds and device."""
        for o in others:
            if not isinstance(o, AUC) or o.num_thresholds != self.num_thresholds or o.device != self.device:
                raise ValueError("merge_state needs AUC states of %d thresholds on %s"
                                 % (self.num_thresholds, self.device))
            self.state += o.state


def _squeeze(y_pred, y_true):
    """Keras' remove_squeezable_dimensions: drop a trailing 1 of the operand whose rank is one higher."""
    diff = y_pred.dim() - y_true.dim()
    if diff == 1 and y_pred.shape[-1] == 1:
        y_pred = y_pred.squeeze(-1)
    elif diff == -1 and y_true.shape[-1] == 1:
        y_true = y_true.squeeze(-1)
    return y_pred, y_true


class MeanMetricWrapper(Metric):
    """tf.keras.metrics.MeanMetricWrapper: the mean of fn(y_true, y_pred) over every value it returned.  Labels and
    predictions are cast to float32 and a trailing 1 is squeezed off the one of higher rank; fn runs on the device
    and the sum of its values (cast to float32, summed in float64) and their count stay there.  Unlike AUC's
    atomics, these are plain in-place adds: updates from several streams must be ordered by the caller."""

    def __init__(self, fn, name=None, device=None):
        self.fn = fn
        self.name = name if name is not None else getattr(fn, "__name__", "mean_metric_wrapper")
        self.device = _device(device)
        self.total = torch.zeros((), dtype=torch.float64, device=self.device)
        self.count = torch.zeros((), dtype=torch.int64, device=self.device)

    def update_state(self, y_true, y_pred):
        y_pred, y_true = _squeeze(_as_float(y_pred, self.device), _as_float(y_true, self.device))
        values = torch.as_tensor(self.fn(y_true, y_pred), device=self.device).to(torch.float32)
        self.total += values.sum(dtype=torch.float64)
        self.count += values.numel()

    def result(self):
        """total / count as a Python float, 0.0 for an empty state."""
        total, count = torch.stack([self.total, self.count.to(torch.float64)]).tolist()
        return total / count if count else 0.0

    def reset_states(self):
        self.total.zero_()
        self.count.zero_()


def accuracy(y_true, y_pred):
    """tf.keras.metrics.accuracy: 1.0 where the values are equal."""
    if y_true.shape != y_pred.shape:
        raise ValueError("shapes %s and %s are incompatible" % (tuple(y_true.shape), tuple(y_pred.shape)))
    return (y_true == y_pred).to(torch.float32)


def mean_squared_error(y_true, y_pred):
    """tf.keras.losses.mean_squared_error: the mean over the last axis of (y_pred - y_true)^2."""
    return torch.square(y_pred - y_true).mean(-1)


class Accuracy(MeanMetricWrapper):
    def __init__(self, name="accuracy", device=None):
        super().__init__(accuracy, name, device)


class MeanSquaredError(MeanMetricWrapper):
    def __init__(self, name="mean_squared_error", device=None):
        super().__init__(mean_squared_error, name, device)


def zoo_eval_metrics(logit_threshold):
    """The eval_metrics_fn of the reference's CTR models: accuracy of `logits > logit_threshold` against the labels
    truncated to int, and the AUC of the probabilities."""
    def acc(labels, predictions):
        return (predictions.reshape(-1) > logit_threshold).int() == labels.reshape(-1).int()

    return {"logits": {"accuracy": acc}, "probs": {"auc": AUC()}}


def _concat(parts):
    """Per-minibatch outputs or labels (arrays / tensors) joined along axis 0."""
    if all(isinstance(p, torch.Tensor) for p in parts):
        return torch.cat([p.detach() for p in parts])
    return np.concatenate([p.detach().cpu().numpy() if isinstance(p, torch.Tensor) else np.asarray(p) for p in parts])


def _is_parts(x):
    return isinstance(x, (list, tuple)) and len(x) > 0 and all(isinstance(p, (np.ndarray, torch.Tensor, dict))
                                                               for p in x)


def _by_output(model_outputs):
    """{output name: outputs} from a dict (a value may be a list of per-minibatch parts, as a worker collects
    them), or from what ParameterServerTrainer.get_evaluation_result()[MODEL_OUTPUT] holds: a list of per-minibatch
    outputs, each an array / tensor or a dict of them."""
    if _is_parts(model_outputs):
        if isinstance(model_outputs[0], dict):
            return {k: _concat([o[k] for o in model_outputs]) for k in model_outputs[0]}
        return {MODEL_OUTPUT: _concat(model_outputs)}
    if isinstance(model_outputs, dict):
        return {k: _concat(v) if _is_parts(v) else v for k, v in model_outputs.items()}
    return {MODEL_OUTPUT: model_outputs}


class EvaluationMetrics:
    """The reference's EvaluationMetrics.  metrics_dict: {metric_name: metric} for a model with one output, or
    {output_name: {metric_name: metric}}; a metric that is not a Metric (a plain callable(labels, outputs)) is
    wrapped in MeanMetricWrapper, in place.  Updates take each batch whole: the reference's 500-row chunks were a
    TensorFlow memory workaround and do not change exact counts."""

    def __init__(self, metrics_dict):
        if not metrics_dict:
            raise ValueError("Evaluation metrics dictionary must not be empty.")
        first_metrics = list(metrics_dict.values())[0]
        if isinstance(first_metrics, dict):
            self._model_have_multiple_outputs = True
            self._metrics_dict = metrics_dict
        else:
            self._model_have_multiple_outputs = False
            self._metrics_dict = {MODEL_OUTPUT: metrics_dict}
        for metrics in self._metrics_dict.values():
            for metric_name, metric in metrics.items():
                if not isinstance(metric, Metric):
                    metrics[metric_name] = MeanMetricWrapper(metric, name=metric_name)

    def update_evaluation_metrics(self, model_outputs, labels):
        """model_outputs: {output name: outputs} (an output without metrics is skipped), a single output, or
        ParameterServerTrainer.get_evaluation_result()[MODEL_OUTPUT]; labels: an array / tensor, or a list of
        per-minibatch labels (get_evaluation_result()[LABEL])."""
        outputs = _by_output(model_outputs)
        if _is_parts(labels):
            labels = _concat(labels)
        for key, out in outputs.items():
            for metric_inst in self._metrics_dict.get(key, {}).values():
                metric_inst.update_state(labels, out)

    def get_evaluation_summary(self):
        if self._model_have_multiple_outputs:
            return {output_name: {metric_name: metric_inst.result() for metric_name, metric_inst in metrics.items()}
                    for output_name, metrics in self._metrics_dict.items()}
        return {metric_name: metric_inst.result()
                for metric_name, metric_inst in self._metrics_dict[MODEL_OUTPUT].items()}

    def reset_metric_states(self):
        """Resets all of the metric state variables."""
        for metrics in self._metrics_dict.values():
            for metric_inst in metrics.values():
                metric_inst.reset_states()
