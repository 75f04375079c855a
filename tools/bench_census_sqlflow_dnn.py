#!/usr/bin/env python
"""census_model_sqlflow's DNNClassifier (workloads/fc_dnn.py CENSUS_SQLFLOW_DNN: eight 64 x 16 tables kept as
dense PS parameters, Adam() defaults) on the parameter-server step, at batch 64, 4096 and 65536 on two shards.
Prints one JSON line per batch with
  - the engine's ms/step and samples/s, graphed (replay) and eager (step), one worker,
  - the tower kernel's time from CUDA events (the engine's tower launch alone, repeated),
  - the drop-in ParameterServerTrainer's ms/step and samples/s over the torch twin (its tables kept as
    DenseTableEmbedding by ParameterServerModelHandler) with cuda_graph=True,
  - the card's name and power limit, read in the same run.
Every time is the wall clock over `--steps` steps ending in a device synchronise, after `--warmup` steps.
Usage: python tools/bench_census_sqlflow_dnn.py [--steps N] [--warmup W] [--batches ...]"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticdl_b200.common.model_handler import ParameterServerModelHandler  # noqa: E402
from elasticdl_b200.ps import PSGroup  # noqa: E402
from elasticdl_b200.workloads import fc_dnn as M  # noqa: E402

DEV = torch.device("cuda", 0)
L = M.CENSUS_SQLFLOW_DNN


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def batches(B, n, seed):
    out = []
    for s in range(n):
        numeric, strings = M.synthetic_census_batch(B, seed + s, DEV)
        labels = (torch.rand(B, generator=torch.Generator(device=DEV).manual_seed(seed + s), device=DEV)
                  < 0.25).float()
        out.append((numeric, strings, labels))
    return out


def timed(fn, steps, warmup):
    """ms per call of fn(i) over `steps` calls after `warmup`, ending in a device synchronise."""
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        fn(i)
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0) / steps


def engine_run(B, steps, warmup):
    opt_type, opt_args, lr = L.optimizer
    group = PSGroup(2, opt_type, opt_args, device=0)
    eng = M.FeatureColumnDNNEngine(group, L, B, lr, seed=1)
    data = batches(B, 2, 100)
    graphed = timed(lambda i: eng.replay(*data[i % 2]), steps, warmup)
    eager = timed(lambda i: eng.step(*data[i % 2]), steps, warmup)
    numeric, strings, labels = data[0]
    eng.step(numeric, strings, labels)  # the step's dedup and rows for this batch
    tower = timed(lambda i: eng.tower.launch(numeric, eng.ids, strings, eng.inv, eng.n_unique, eng.rows, labels,
                                             eng.flat), max(steps, 10), 2)
    eng.check()
    group.close()
    return graphed, eager, tower


def dropin_run(B, steps, warmup):
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    opt_type, opt_args, _ = L.optimizer
    group = PSGroup(2, opt_type, opt_args, device=0)
    twin = ParameterServerModelHandler().get_model_to_train(M.FeatureColumnDNN(L)).to(DEV)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(twin, client, args=types.SimpleNamespace(cuda_graph=True))
    transform = L.transform(DEV)
    data = [(M.twin_features(L, n, s, transform), y) for n, s, y in batches(B, 2, 7)]
    ms = timed(lambda i: trainer.train_minibatch(*data[i % 2]), steps, warmup + 4)
    graphed = isinstance(trainer._graph_state, dict)
    group.check()
    group.close()
    return ms, graphed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batches", nargs="*", type=int, default=[64, 4096, 65536])
    args = ap.parse_args()
    card = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit()}
    for B in args.batches:
        graphed, eager, tower = engine_run(B, args.steps, args.warmup)
        dropin, dropin_graphed = dropin_run(B, args.steps, args.warmup)
        row = dict(model=L.name, batch=B, engine_graphed_ms_per_step=round(graphed, 4),
                   engine_graphed_samples_per_s=round(1e3 * B / graphed), engine_eager_ms_per_step=round(eager, 4),
                   engine_eager_samples_per_s=round(1e3 * B / eager), tower_ms=round(tower, 4),
                   dropin_ms_per_step=round(dropin, 4), dropin_samples_per_s=round(1e3 * B / dropin),
                   dropin_graphed=dropin_graphed, steps=args.steps, **card)
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
