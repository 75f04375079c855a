#!/usr/bin/env python
"""census_dnn_model and heart_functional_api (workloads/fc_dnn.py) on the parameter-server step: per model, batch
64, 4096 and 65536, with 1 and 4 worker threads (each its own client view and stream, the graphed engine step),
prints one JSON line with
  - engine ms/step (wall time per step of one worker) and samples/s (all workers),
  - the tower kernel's time from CUDA events (one worker's tower launch alone, repeated),
  - the drop-in ParameterServerTrainer's ms/step over the torch twin with cuda_graph=True (1 worker),
  - the card's name and power limit, read in the same run.
Usage: python tools/bench_fc_dnn.py [--steps N] [--warmup W] [--models ...] [--batches ...]"""
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
from elasticdl_b200.workloads import fc_dnn as M  # noqa: E402

DEV = torch.device("cuda", 0)


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def batches(L, B, n, seed):
    out = []
    for s in range(n):
        if L is not M.HEART:
            numeric, strings = M.synthetic_census_batch(B, seed + s, DEV)
            labels = (torch.rand(B, generator=torch.Generator(device=DEV).manual_seed(seed + s), device=DEV)
                      < 0.25).float()
        else:
            numeric, strings, labels = M.synthetic_heart_batch(B, seed + s, DEV)
        out.append((numeric, strings, labels))
    return out


def engine_run(L, B, workers, steps, warmup):
    opt_type, opt_args, lr = L.optimizer
    group = PSGroup(2, opt_type, opt_args, device=0)
    engines = [M.FeatureColumnDNNEngine(group, L, B, lr, seed=1, register=(w == 0)) for w in range(workers)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(workers)]
    data = [batches(L, B, 2, 100 * (w + 1)) for w in range(workers)]
    for e, s, d in zip(engines, streams, data):
        with torch.cuda.stream(s):
            for i in range(warmup):
                e.replay(*d[i % 2])
    torch.cuda.synchronize()

    def run(w):
        with torch.cuda.stream(streams[w]):
            for i in range(steps):
                engines[w].replay(*data[w][i % 2])
        streams[w].synchronize()

    threads = [threading.Thread(target=run, args=(w,)) for w in range(workers)]
    t0 = time.perf_counter()
    [t.start() for t in threads]
    [t.join() for t in threads]
    wall = time.perf_counter() - t0
    for e in engines:
        e.check()
    tower_ms = None
    if workers == 1:
        e = engines[0]
        numeric, strings, labels = data[0][0]
        with torch.cuda.stream(streams[0]):
            e.step(numeric, strings, labels)  # the step's dedup and rows for this batch
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            n = max(steps, 10)
            a.record()
            for _ in range(n):
                e.tower.launch(numeric, e.ids, strings, e.inv, e.n_unique, e.rows, labels, e.flat)
            b.record()
            b.synchronize()
        tower_ms = a.elapsed_time(b) / n
    group.close()
    return 1e3 * wall / steps, workers * B * steps / wall, tower_ms


def dropin_run(L, B, steps, warmup):
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    opt_type, opt_args, lr = L.optimizer
    group = PSGroup(1, opt_type, opt_args, device=0)
    twin = M.FeatureColumnDNN(L).to(DEV)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(twin, client, args=types.SimpleNamespace(cuda_graph=True))
    transform = L.transform(DEV)
    data = [(M.twin_features(L, n, s, transform), y) for n, s, y in batches(L, B, 2, 7)]
    for i in range(warmup + 4):
        trainer.train_minibatch(*data[i % 2])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        trainer.train_minibatch(*data[i % 2])
    torch.cuda.synchronize()
    ms = 1e3 * (time.perf_counter() - t0) / steps
    graphed = isinstance(trainer._graph_state, dict)
    group.close()
    return ms, graphed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--models", nargs="*", default=list(M.LAYOUTS))
    ap.add_argument("--batches", nargs="*", type=int, default=[64, 4096, 65536])
    args = ap.parse_args()
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    for model in args.models:
        L = M.layout_of(model)
        for B in args.batches:
            dropin_ms, graphed = dropin_run(L, B, args.steps, args.warmup)
            for workers in (1, 4):
                ms, sps, tower_ms = engine_run(L, B, workers, args.steps, args.warmup)
                row = dict(model=model, batch=B, workers=workers, engine_ms_per_step=round(ms, 4),
                           samples_per_s=round(sps), tower_ms=None if tower_ms is None else round(tower_ms, 4),
                           dropin_ms_per_step=round(dropin_ms, 4) if workers == 1 else None,
                           dropin_graphed=graphed if workers == 1 else None, steps=args.steps, **card)
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
