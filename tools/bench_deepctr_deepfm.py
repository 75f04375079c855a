#!/usr/bin/env python
"""deepctr's DeepFM estimator (workloads/deepctr_deepfm.py) on the parameter-server step: batch 64 (the zoo's
batch_size) and 65536, one worker, the graphed engine step over its two groups (Adagrad and Ftrl, two shards each),
prints one JSON line per batch with
  - engine ms/step (wall time per step) and samples/s,
  - the tower's time from CUDA events (its five launches alone, repeated),
  - the tower's achieved FLOP/s from the DNN's 419 KFLOP per sample (forward + backward of 117-256-128-64-1, the
    FM and linear terms not counted) and its share of the 3xTF32 bound (3 x those FLOP at the data sheet's
    495 TFLOP/s dense TF32),
  - the card's name and power limit, read in the same run.
Usage: python tools/bench_deepctr_deepfm.py [--steps N] [--warmup W] [--batches ...]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticdl_b200.ps import PSGroup  # noqa: E402
from elasticdl_b200.workloads import deepctr_deepfm as M  # noqa: E402

DEV = torch.device("cuda", 0)
MACS = 117 * 256 + 256 * 128 + 128 * 64 + 64  # forward MACs per sample (71 K)
FLOP_PER_SAMPLE = 2 * (3 * MACS - 117 * 256 + 104 * 256)  # forward, data (dx of the 104 sparse columns), weight
TF32_PEAK = 495e12  # H100 SXM data sheet, dense TF32


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def data(B, n, seed):
    return [(d / 1e4, s, y) for d, s, y in (M.synthetic_batch(B, seed + k, DEV) for k in range(n))]


def engine_run(B, steps, warmup):
    (lt, la), (dt, da) = M.optimizers()
    eng = M.DeepctrDeepfmEngine(PSGroup(2, dt, da, device=0), PSGroup(2, lt, la, device=0), B, seed=1)
    d = data(B, 2, 100)
    for i in range(warmup):
        eng.replay(*d[i % 2])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        eng.replay(*d[i % 2])
    torch.cuda.synchronize()
    dt_s = time.perf_counter() - t0
    eng.check()
    return 1e3 * dt_s / steps, steps * B / dt_s, eng


def tower_ms(eng, dense, labels, reps):
    t = eng.tower
    for _ in range(3):
        t.launch(eng.ids, dense, labels, eng.flat)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        t.launch(eng.ids, dense, labels, eng.flat)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batches", type=int, nargs="+", default=[64, 65536])
    args = ap.parse_args()
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    for B in args.batches:
        ms, sps, eng = engine_run(B, args.steps, args.warmup)
        row = dict(card, batch=B, engine_ms_per_step=round(ms, 4), samples_per_s=round(sps))
        dense, _, labels = data(B, 1, 5)[0]
        tms = tower_ms(eng, dense, labels, max(args.steps, 20))
        flops = FLOP_PER_SAMPLE * B
        row.update(tower_ms=round(tms, 4), tower_tflops=round(flops / tms / 1e9, 2),
                   share_of_3xtf32_bound=round(3 * flops / TF32_PEAK / (tms * 1e-3), 4),
                   bound="3xTF32 compute: 3 x %.2f GFLOP at 495 TFLOP/s (data sheet)" % (flops / 1e9))
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
