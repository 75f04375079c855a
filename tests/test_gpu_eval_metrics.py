"""The AUC kernel (csrc/eval_metrics.cu, include/b200_metrics.h) and the metrics of
elasticdl_b200/common/evaluation_utils.py against oracle/metrics_oracle.py.

Counts are compared bit for bit with the oracle's literal [T, n] comparison matrix: random probabilities mixed
with every threshold, the fp32 values one ulp either side of it, 0.0 and 1.0, labels in {0, 1, 0.7}, n at the warp
and CTA edges and past several grid-stride passes, T in {2, 3, 200, 8192}.  Then the refusals, invalid
predictions, graph capture, an update shared by two streams, merge_state, and EvaluationMetrics on the reference's
own vector."""
import ctypes

import numpy as np
import pytest
import torch

from elasticdl_b200 import _lib
from elasticdl_b200.common import evaluation_utils as EU
from oracle import metrics_oracle as MO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
PER_CTA = 2048  # B200_METRICS_MIN_PER_CTA: the samples below which the grid is one CTA


def _data(n, T, seed):
    """float32 probabilities in [0, 1] with a third of them at a threshold, one ulp either side, 0.0 or 1.0, and
    labels in {0, 1, 0.7}."""
    rng = np.random.RandomState(seed)
    p = rng.random_sample(n).astype(np.float32)
    thr = MO.thresholds(T)
    special = np.concatenate([thr, np.nextafter(thr, np.float32(-np.inf)), np.nextafter(thr, np.float32(np.inf)),
                              np.array([0.0, 1.0], np.float32)])
    special = special[(special >= 0) & (special <= 1)]
    pick = rng.random_sample(n) < 1.0 / 3.0
    p[pick] = special[rng.randint(0, special.size, int(pick.sum()))]
    y = np.array([0.0, 1.0, 0.7], np.float32)[rng.randint(0, 3, n)]
    return y, p


def _oracle_counts(y, p, T):
    """The oracle's confusion counts, summed over chunks (the counts are additive, as
    tests/test_oracle_eval_metrics.py checks)."""
    tot = [np.zeros(T, np.int64) for _ in range(4)] + [0]
    chunk = max(256, (1 << 24) // T)
    for a in range(0, max(len(p), 1), chunk):
        c = MO.auc_confusion(y[a:a + chunk], p[a:a + chunk], T)
        tot = [t + v for t, v in zip(tot, c)]
    return tot


def _check_counts(auc, y, p, T):
    got = auc.confusion()
    want = _oracle_counts(y, p, T)
    for name, g, w in zip(("tp", "fp", "tn", "fn"), got[:4], want[:4]):
        assert np.array_equal(g.astype(np.int64), w), (name, np.nonzero(g.astype(np.int64) != w)[0][:10])
    assert got[4] == want[4]


def _ns(T):
    edges = [1, 31, 32, 33, PER_CTA, PER_CTA + 1]
    if T == 8192:  # the literal [T, n] oracle is the cost here
        return edges + [65537]
    if T == 2:
        return edges + [(1 << 20) + 3, 5_000_011]  # 5 M: several passes of any grid (<= 2048 threads per SM x 4)
    return edges + [(1 << 20) + 3]


@pytest.mark.parametrize("T,n", [(T, n) for T in (2, 3, 200, 8192) for n in _ns(T)])
def test_counts_bit_exact(T, n):
    y, p = _data(n, T, seed=T * 7 + n % 1000)
    auc = EU.AUC(num_thresholds=T)
    auc.update_state(torch.from_numpy(y).to(DEV), torch.from_numpy(p).to(DEV).reshape(-1, 1))
    _check_counts(auc, y, p, T)
    assert auc.result() == pytest.approx(float(MO.auc(y, p, T)), rel=0, abs=1e-12)


def test_numpy_inputs_and_accumulation():
    T = 200
    y, p = _data(10000, T, seed=5)
    auc = EU.AUC()
    for a, b in ((0, 1), (1, 4000), (4000, 4000), (4000, 10000)):  # includes an empty update
        auc.update_state(y[a:b], p[a:b])
    _check_counts(auc, y, p, T)


def test_invalid_predictions_raise_until_reset():
    auc = EU.AUC()
    p = torch.tensor([0.5, float("nan"), -0.1, 1.5, -0.0, 1.0], device=DEV)
    y = torch.tensor([1.0, 1.0, 0.0, 0.0, 0.0, 1.0], device=DEV)
    auc.update_state(y, p)
    with pytest.raises(ValueError, match="3 predictions"):
        auc.result()
    tp, fp, tn, fn, invalid = auc.confusion()
    assert invalid == 3 and tp[0] + fn[0] == 2 and fp[0] + tn[0] == 1  # -0.0 is a valid negative
    auc.reset_states()
    assert auc.result() == 0.0
    auc.update_state(y[[0, 4]], p[[0, 4]])
    assert auc.result() == 1.0


def test_refusals():
    lib = _lib.lib()
    for T in (0, 1):
        with pytest.raises(ValueError, match="num_thresholds"):
            EU.AUC(num_thresholds=T)
    with pytest.raises(ValueError):
        EU.AUC(num_thresholds=_lib.METRICS_MAX_THRESHOLDS + 1)
    EU.AUC(num_thresholds=_lib.METRICS_MAX_THRESHOLDS)  # the limit itself is accepted
    buf = torch.zeros(2 * (_lib.METRICS_MAX_THRESHOLDS + 2) + 1, dtype=torch.int64, device=DEV)
    x = torch.full((8,), 0.5, device=DEV)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    thr = torch.zeros(_lib.METRICS_MAX_THRESHOLDS + 1, device=DEV)
    for T, n in ((1, 8), (_lib.METRICS_MAX_THRESHOLDS + 1, 8), (200, -1), (200, 1 << 31)):
        before = lib.b200_metrics_launch_count()
        rc = lib.b200_metrics_auc_update(x.data_ptr(), x.data_ptr(), n, thr.data_ptr(), T, buf.data_ptr(),
                                         buf[-1:].data_ptr(), st)
        assert rc == _lib.EINVAL, (T, n, rc)
        assert lib.b200_metrics_launch_count() == before
        assert lib.b200_metrics_last_error()
    # n = 0 launches nothing and leaves the state alone, even with null inputs
    before = lib.b200_metrics_launch_count()
    assert lib.b200_metrics_auc_update(None, None, 0, thr.data_ptr(), 200, buf.data_ptr(), buf[-1:].data_ptr(), st) == 0
    assert lib.b200_metrics_launch_count() == before
    torch.cuda.synchronize()
    assert int(buf.abs().sum()) == 0
    with pytest.raises(ValueError, match="labels for"):
        EU.AUC().update_state(x[:3], x)


def test_graph_replay_adds_k_times():
    T, n, k = 200, 50_000, 3
    y, p = _data(n, T, seed=11)
    sy, sp = torch.from_numpy(y).to(DEV), torch.from_numpy(p).to(DEV)
    auc = EU.AUC()
    torch.cuda.synchronize()
    before = _lib.lib().b200_metrics_launch_count()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        auc.update_state(sy, sp)
    assert _lib.lib().b200_metrics_launch_count() == before + 1
    for _ in range(k):
        graph.replay()
    torch.cuda.synchronize()
    got = auc.confusion()
    want = _oracle_counts(y, p, T)
    for g, w in zip(got[:4], want[:4]):
        assert np.array_equal(g.astype(np.int64), k * w)


def test_two_streams_share_one_state_and_merge_state():
    T = 200
    parts = [_data(300_000, T, seed=20 + i) for i in range(2)]
    auc = EU.AUC()
    streams = [torch.cuda.Stream(device=DEV) for _ in parts]
    dev_parts = [(torch.from_numpy(y).to(DEV), torch.from_numpy(p).to(DEV)) for y, p in parts]
    main = torch.cuda.current_stream()
    for s, (y, p) in zip(streams, dev_parts):
        s.wait_stream(main)
        with torch.cuda.stream(s):
            for _ in range(4):
                auc.update_state(y, p)
    for s in streams:
        main.wait_stream(s)
    y = np.concatenate([parts[0][0]] * 4 + [parts[1][0]] * 4)
    p = np.concatenate([parts[0][1]] * 4 + [parts[1][1]] * 4)
    _check_counts(auc, y, p, T)
    # merge_state: the same as one state fed both parts
    a, b = EU.AUC(), EU.AUC()
    a.update_state(*dev_parts[0])
    b.update_state(*dev_parts[1])
    a.merge_state(b)
    _check_counts(a, np.concatenate([parts[0][0], parts[1][0]]), np.concatenate([parts[0][1], parts[1][1]]), T)
    with pytest.raises(ValueError):
        a.merge_state(EU.AUC(num_thresholds=10))


def test_evaluation_metrics_reference_vector():
    """elasticdl/python/tests/evaluation_service_test.py:76-94 through EvaluationMetrics: numpy reports, device
    state, acc 0.25, acc_fn 0.25, mse 10.125; reset clears them."""
    metrics = EU.EvaluationMetrics({
        "acc": EU.Accuracy(), "mse": EU.MeanSquaredError(),
        "acc_fn": lambda labels, outputs: outputs.to(torch.int32) == labels.to(torch.int32)})
    metrics.update_evaluation_metrics({EU.MODEL_OUTPUT: np.array([[1], [6], [3]], np.float32)},
                                      np.array([[1], [0], [3]], np.float32))
    metrics.update_evaluation_metrics({EU.MODEL_OUTPUT: np.array([[4], [5], [6], [7], [8]], np.float32)},
                                      np.array([[7], [8], [9], [10], [11]], np.float32))
    s = metrics.get_evaluation_summary()
    assert s["acc"] == pytest.approx(0.25) and s["acc_fn"] == pytest.approx(0.25)
    assert s["mse"] == pytest.approx(10.125)
    metrics.reset_metric_states()
    assert metrics.get_evaluation_summary() == {"acc": 0.0, "mse": 0.0, "acc_fn": 0.0}


def test_evaluation_metrics_outputs_and_squeeze():
    """Multiple outputs: an output without metrics is skipped; [B, 1] predictions against [B] labels are squeezed
    (Keras' remove_squeezable_dimensions); lists of per-minibatch parts are joined."""
    rng = np.random.RandomState(3)
    y = rng.randint(0, 2, 1000).astype(np.float32)
    logits = rng.randn(1000).astype(np.float32)
    probs = torch.sigmoid(torch.from_numpy(logits).to(DEV)).reshape(-1, 1)
    metrics = EU.EvaluationMetrics(EU.zoo_eval_metrics(0.0))
    metrics.update_evaluation_metrics({"logits": torch.from_numpy(logits[:400]).to(DEV), "probs": probs[:400],
                                       "other": probs[:400]}, torch.from_numpy(y[:400]).to(DEV))
    metrics.update_evaluation_metrics({"logits": [logits[400:700], logits[700:]],
                                       "probs": [probs[400:700], probs[700:]]}, [y[400:700], y[700:]])
    s = metrics.get_evaluation_summary()
    acc = MO.MeanMetric(lambda labels, lg: (lg.reshape(-1) > 0).astype(np.int32) == labels.reshape(-1).astype(np.int32))
    acc.update(y, logits)
    assert s["logits"]["accuracy"] == acc.result()
    assert s["probs"]["auc"] == pytest.approx(float(MO.auc(y, probs.cpu().numpy())), rel=0, abs=1e-12)
    m = EU.Accuracy()
    m.update_state(torch.ones(5, device=DEV), torch.ones((5, 1), device=DEV))
    assert m.result() == 1.0
