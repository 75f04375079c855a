#!/usr/bin/env python
"""deepctr's WDL (workloads/deepctr_wdl.py) on the parameter-server step: batch 32 (the reference tutorial's
minibatch), 4096 and 65536, with 1 and 4 worker threads (each its own client view and stream, the graphed engine
step), prints one JSON line per point with
  - engine ms/step (wall time per step of one worker) and samples/s (all workers),
  - the tower's time from CUDA events (its five launches alone, repeated, one worker),
  - the tower's achieved FLOP/s from the DNN's 419 KFLOP per sample (forward + backward of 117-256-128-64-1) and
    its share of the 3xTF32 bound (3 x those FLOP at the data sheet's 495 TFLOP/s dense TF32),
  - the drop-in ParameterServerTrainer's ms/step over the torch twin with cuda_graph=True (1 worker),
  - the card's name and power limit, read in the same run.
Usage: python tools/bench_deepctr_wdl.py [--steps N] [--warmup W] [--batches ...] [--workers ...]"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticdl_b200.ps import PSGroup  # noqa: E402
from elasticdl_b200.workloads import deepctr_wdl as M  # noqa: E402

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
    out = []
    for s in range(n):
        dense, strings, labels = M.synthetic_batch(B, seed + s, DEV)
        out.append((dense / 1e4, strings, labels))  # as the tests: raw counts saturate p
    return out


def engine_run(B, workers, steps, warmup):
    opt_type, opt_args, lr = M.optimizer()
    group = PSGroup(2, opt_type, opt_args, device=0)
    engines = [M.DeepctrWdlEngine(group, B, lr, seed=1, register=(w == 0)) for w in range(workers)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(workers)]
    d = [data(B, 2, 100 * (w + 1)) for w in range(workers)]
    for e, s, dd in zip(engines, streams, d):
        with torch.cuda.stream(s):
            for i in range(warmup):
                e.replay(*dd[i % 2])
    torch.cuda.synchronize()

    def run(w):
        with torch.cuda.stream(streams[w]):
            for i in range(steps):
                engines[w].replay(*d[w][i % 2])
        streams[w].synchronize()

    t0 = time.perf_counter()
    threads = [threading.Thread(target=run, args=(w,)) for w in range(workers)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    for e in engines:
        e.check()
    return 1e3 * dt / steps, workers * steps * B / dt, engines[0]


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


def dropin_ms(B, steps, warmup):
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    opt_type, opt_args, lr = M.optimizer()
    group = PSGroup(1, opt_type, opt_args, device=0)
    twin = M.DeepctrWdl(lr=lr).to(DEV)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(twin, client, args=types.SimpleNamespace(cuda_graph=True))
    transform = M.transform(DEV)
    feats = []
    for dense, strings, labels in data(B, 2, 7):
        ids, _ = transform(dense, strings)
        feats.append(({"ids": ids.long(), "dense": dense}, labels))
    for i in range(warmup):
        trainer.train_minibatch(*feats[i % 2])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        trainer.train_minibatch(*feats[i % 2])
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps, trainer.graph_fallback_reason


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 4096, 65536])
    ap.add_argument("--workers", type=int, nargs="+", default=[1, 4])
    args = ap.parse_args()
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    for B in args.batches:
        for workers in args.workers:
            ms, sps, eng = engine_run(B, workers, args.steps, args.warmup)
            row = dict(card, batch=B, workers=workers, engine_ms_per_step=round(ms, 4), samples_per_s=round(sps))
            if workers == 1:
                dense, _, labels = data(B, 1, 5)[0]
                tms = tower_ms(eng, dense, labels, max(args.steps, 20))
                flops = FLOP_PER_SAMPLE * B
                row.update(tower_ms=round(tms, 4), tower_tflops=round(flops / tms / 1e9, 2),
                           share_of_3xtf32_bound=round(3 * flops / TF32_PEAK / (tms * 1e-3), 4),
                           bound="3xTF32 compute: 3 x %.1f GFLOP at 495 TFLOP/s (data sheet)" % (flops / 1e9))
                dms, why = dropin_ms(B, max(args.steps // 2, 5), args.warmup)
                row.update(dropin_ms_per_step=round(dms, 3), dropin_graph_fallback=why)
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
