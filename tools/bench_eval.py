#!/usr/bin/env python
"""Evaluation metrics on the GPU (elasticdl_b200/common/evaluation_utils.py), one JSON line per measurement:
  (a) at B in --batches: auc_update_call, one AUC.update_state call (Python, ctypes and one
      b200_metrics_auc_update launch); auc_kernel, the launch alone, 50 of them captured in one CUDA graph and
      replayed, with algorithmic bytes 8 B (one fp32 prediction and one fp32 label per sample) and the rate;
  (b) keras_torch: the same update as Keras computes it, written in torch: the [T, B] broadcast comparison
      `preds > thresholds`, the label matrix and the four reductions tp / fp / tn / fn;
  (c) engine: the dac_ctr DeepFM engine (bench.py's tile tower, Zipf batches) at --engine-batch: predict() alone
      against evaluate() with eval_metrics_fn(), and the metrics' share of an evaluation step.
Times are CUDA events around --reps calls on one stream after --warmup calls (a device synchronise ends each
window).  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
GRAPHED = 50  # AUC updates per captured graph in (a)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def time_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def keras_update(thr, labels, preds, counts):
    """Keras' update_confusion_matrix_variables in torch: [T, B] comparisons and four reductions."""
    pred_is_pos = preds.reshape(1, -1) > thr.reshape(-1, 1)
    label_is_pos = (labels.reshape(1, -1) != 0).expand_as(pred_is_pos)
    counts[0] += (label_is_pos & pred_is_pos).sum(1)
    counts[1] += (~label_is_pos & pred_is_pos).sum(1)
    counts[2] += (~label_is_pos & ~pred_is_pos).sum(1)
    counts[3] += (label_is_pos & ~pred_is_pos).sum(1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="32768,262144,1048576")
    ap.add_argument("--engine-batch", type=int, default=32768)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures on a CUDA device; none is visible")
    from elasticdl_b200.common import evaluation_utils as EU

    dev = torch.device("cuda", 0)
    name, power = card()
    base = {"gpu": name, "power_limit": power, "reps": args.reps}
    g = torch.Generator(device=dev).manual_seed(0)
    for B in [int(b) for b in args.batches.split(",")]:
        preds = torch.sigmoid(torch.randn(B, generator=g, device=dev))
        labels = (torch.rand(B, generator=g, device=dev) < 0.25).float()
        auc = EU.AUC()
        ms = time_ms(lambda: auc.update_state(labels, preds), args.reps, args.warmup)
        print(json.dumps(dict(base, what="auc_update_call", B=B, thresholds=200, ms=ms)), flush=True)
        # the kernel without the Python call: GRAPHED updates captured in one CUDA graph, replayed
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            for _ in range(GRAPHED):
                auc.update_state(labels, preds)
        ms_g = time_ms(graph.replay, max(10, args.reps // GRAPHED), 2) / GRAPHED
        print(json.dumps(dict(base, what="auc_kernel", B=B, thresholds=200, ms=ms_g, bytes=8 * B,
                              gbs=8 * B / (ms_g * 1e-3) / 1e9)), flush=True)
        counts = torch.zeros((4, 200), dtype=torch.int64, device=dev)
        ms_k = time_ms(lambda: keras_update(auc.thresholds, labels, preds, counts), args.reps, args.warmup)
        print(json.dumps(dict(base, what="keras_torch", B=B, thresholds=200, ms=ms_k, over_update_call=ms_k / ms,
                              over_kernel=ms_k / ms_g)),
              flush=True)

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads import deepfm as DF

    B = args.engine_batch
    group = PSGroup(1, "Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", device=0)
    eng = DF.DeepFMPSEngine(group, B)
    ids, dense, labels = DF.synthetic_batch(B, 1, dev, "zipf")
    eng.step(ids, dense, labels)
    metrics = EU.EvaluationMetrics(DF.eval_metrics_fn())
    ms_p = time_ms(lambda: eng.predict(ids, dense), args.reps, args.warmup)
    ms_e = time_ms(lambda: eng.evaluate(ids, dense, labels, metrics), args.reps, args.warmup)
    metrics.get_evaluation_summary()
    group.check()
    print(json.dumps(dict(base, what="engine", model="deepfm", B=B, predict_ms=ms_p, evaluate_ms=ms_e,
                          metrics_share=(ms_e - ms_p) / ms_e)), flush=True)
    group.close()


if __name__ == "__main__":
    main()
