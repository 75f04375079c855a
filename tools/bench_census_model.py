#!/usr/bin/env python
"""BASELINE.json configs[2] as the reference defines it: the census wide & deep model
(model_zoo/census_wide_deep_model/wide_deep_functional_api.py) from raw Adult-shaped rows, async, 1 and 4 workers.

Per configuration (workers 1 / 4 as threads on cloned views, each on its own stream; batch 64 -- the reference's
CI value, scripts/client_test.sh -- 4096 and 65536; SGD lr 0.1 and Adam lr 3e-4) one JSON line with:
  - engine_ms_per_step / engine_samples_per_s: CensusWideDeepEngine.replay (the whole step as one CUDA graph:
    pull -> census_transform -> tower -> push), wall time over all workers' steps ending in a synchronize;
  - tower_ms: the census tower kernel alone, CUDA events around `--tower-reps` launches on one stream;
  - dropin_ms_per_step / dropin_samples_per_s: ParameterServerTrainer(cuda_graph=True) over the torch twin
    CensusWideDeep on the same raw batches (dropin_path says whether it ran graphed or eagerly, and why);
  - the card's name and power limit, read in the same run.
At batch 64 the step is launch-bound: its time is a latency, not a share of any roof."""
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

OPTS = {"sgd": ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", 0.1),
        "adam": ("Adam", "learning_rate=0.0003;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", 3e-4)}
N_BATCHES = 4


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def batches(w, B, dev):
    from elasticdl_b200.workloads.census_features import synthetic_raw_batch

    out = []
    for s in range(N_BATCHES):
        numeric, strings, _, _ = synthetic_raw_batch(B, 1000 * w + s, dev)
        gen = torch.Generator(device=dev).manual_seed(7 * w + s)
        out.append((numeric, strings, (torch.rand(B, generator=gen, device=dev) < 0.24).float()))
    return out


def run_threads(workers, steps, fn, streams):
    """fn(w, s) for s < steps in each of `workers` threads on its own stream; wall seconds of the timed loops."""
    barrier = threading.Barrier(workers + 1)
    errors = []

    def loop(w):
        try:
            with torch.cuda.stream(streams[w]):
                barrier.wait()
                for s in range(steps):
                    fn(w, s)
                streams[w].synchronize()
                barrier.wait()
        except Exception as e:  # noqa: BLE001
            errors.append((w, repr(e)))
            barrier.abort()

    threads = [threading.Thread(target=loop, args=(w,)) for w in range(workers)]
    [t.start() for t in threads]
    try:
        barrier.wait()
        t0 = time.perf_counter()
        barrier.wait()
        wall = time.perf_counter() - t0
    except threading.BrokenBarrierError:
        wall = float("nan")
    [t.join() for t in threads]
    if errors:
        raise RuntimeError(errors)
    return wall


def engine_arm(opt, workers, B, steps, data, dev):
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.census import CensusWideDeepEngine

    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(1, opt_type, opt_args, device=0)
    engines = [CensusWideDeepEngine(group, B, lr, seed=1, register=(w == 0)) for w in range(workers)]
    streams = [torch.cuda.Stream(device=dev) for _ in range(workers)]
    for w, (e, s) in enumerate(zip(engines, streams)):
        with torch.cuda.stream(s):
            e.capture()
            for k in range(3):
                e.replay(*data[w][k % N_BATCHES])
    torch.cuda.synchronize()
    wall = run_threads(workers, steps, lambda w, s: engines[w].replay(*data[w][s % N_BATCHES]), streams)
    for e in engines:
        e.check()
    version = group.snapshot()[0][0]
    # the tower alone on one stream
    e = engines[0]
    ids = e.transform(*data[0][0][:2])[0]
    labels = data[0][0][2]
    reps = max(20, steps)
    for _ in range(5):
        e.tower.launch(ids, labels, e.flat, False)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        e.tower.launch(ids, labels, e.flat, False)
    t1.record()
    torch.cuda.synchronize()
    tower_ms = t0.elapsed_time(t1) / reps
    loss = float(e.tower.loss)
    group.close()
    return {"engine_ms_per_step": 1e3 * wall / steps, "engine_samples_per_s": workers * steps * B / wall,
            "tower_ms": tower_ms, "ps_version": version, "engine_last_loss": loss}


def dropin_arm(opt, workers, B, steps, data, dev):
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.census import CensusWideDeep
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    opt_type, opt_args, lr = OPTS[opt]
    torch.manual_seed(0)
    group = PSGroup(1, opt_type, opt_args, device=0)
    models = [CensusWideDeep(lr, optimizer=opt).to(dev) for _ in range(workers)]
    for m in models[1:]:
        m.load_state_dict(models[0].state_dict())
    trainers, streams = [], []
    for w in range(workers):
        client = PSClient(group if w == 0 else group.clone_view())
        client.dense_output = "torch"
        s = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(s):
            tr = ParameterServerTrainer(models[w], client, args=types.SimpleNamespace(get_model_steps=1, cuda_graph=True))
            for k in range(6):
                numeric, strings, labels = data[w][k % N_BATCHES]
                tr.train_minibatch((numeric, strings), labels)
            s.synchronize()
        trainers.append(tr)
        streams.append(s)

    def one(w, s):
        numeric, strings, labels = data[w][s % N_BATCHES]
        trainers[w].train_minibatch((numeric, strings), labels)

    wall = run_threads(workers, steps, one, streams)
    why = trainers[0].graph_fallback_reason
    group.close()
    return {"dropin_ms_per_step": 1e3 * wall / steps, "dropin_samples_per_s": workers * steps * B / wall,
            "dropin_path": "graphed" if why is None else "eager (%s)" % why}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--batches", default="64,4096,65536")
    ap.add_argument("--workers", default="1,4")
    ap.add_argument("--opts", default="sgd,adam")
    ap.add_argument("--no-dropin", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_census_model.py measures on a CUDA device; none is available")
    dev = torch.device("cuda", 0)
    name, power = card()
    for B in [int(b) for b in args.batches.split(",")]:
        for workers in [int(w) for w in args.workers.split(",")]:
            data = [batches(w, B, dev) for w in range(workers)]
            for opt in args.opts.split(","):
                row = {"config": "census wide&deep from raw rows, async %s lr %g, %d worker(s), batch %d"
                                 % (opt, OPTS[opt][2], workers, B),
                       "gpu": name, "power_limit": power, "steps_per_worker": args.steps}
                row.update(engine_arm(opt, workers, B, args.steps, data, dev))
                if not args.no_dropin:
                    row.update(dropin_arm(opt, workers, B, args.steps, data, dev))
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
