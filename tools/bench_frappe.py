#!/usr/bin/env python
"""The frappe DeepFM model the reference's own tests train (model_zoo/deepfm_edl_embedding, deepfm_functional_api)
on one worker, async.

Per configuration (batch 64 -- the reference's CI value, scripts/client_test.sh -- 4096, 32768 and 262144;
hashed tables (input_dim=None) or bounded ones (input_dim=5383); SGD lr 0.1 or Adam lr 1e-3) one JSON line with:
  - engine_ms_per_step / engine_samples_per_s: FrappeDeepFMEngine.replay (the whole step as one CUDA graph), wall
    time over `--steps` steps ending in a synchronize;
  - eager_ms: the eager step's parts between CUDA events (pull_dense, dedup, pull, tower, push), median over steps;
  - tower_bytes: the tower's algorithmic bytes (ids, inv, labels, logits, the U unique rows read once and their
    gradients written once, the dense parameters and gradients) beside its time.  At these sizes the tower is
    latency-bound, not bandwidth-bound: its time is a latency, not a share of any roof;
  - dropin_ms_per_step / dropin_samples_per_s: ParameterServerTrainer(cuda_graph=True) over the torch twin
    FrappeDeepFM on the same batches (dropin_path says whether it ran graphed or eagerly, and why);
  - the card's name and power limit, read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OPTS = {"sgd": ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", 0.1),
        "adam": ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", 1e-3)}
N_BATCHES = 4


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
    except Exception:  # noqa: BLE001
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def timed(steps, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for s in range(steps):
        fn(s)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def engine_arm(opt, hashed, B, steps, data):
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.frappe import INPUT_DIM, FrappeDeepFMEngine

    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(1, opt_type, opt_args, device=0)
    eng = FrappeDeepFMEngine(group, B, lr, input_dim=None if hashed else INPUT_DIM, seed=1, expected_rows=1 << 16)
    for k in range(3):
        eng.replay(*data[k % N_BATCHES])
    wall = timed(steps, lambda s: eng.replay(*data[s % N_BATCHES]))
    eng.check()
    # the eager step's parts
    parts = {}
    for s in range(max(10, min(steps, 50))):
        ev = {}
        eng.step(*data[s % N_BATCHES], ev=ev)
        torch.cuda.synchronize()
        names = ["start", "pull_dense", "dedup", "pull", "tower", "push"]
        for a, b in zip(names, names[1:]):
            parts.setdefault(b, []).append(ev[a][0].elapsed_time(ev[b][0]))
    U = int(eng.n_unique.item())
    eng.check()
    loss = float(eng.tower.loss)
    group.close()
    # ids 8 + inv 4 per occurrence, label 4 + logit 4 per sample, U rows of 65 floats read and written once,
    # the dense parameters read and their gradients written
    tower_bytes = B * 10 * 12 + B * 8 + U * 65 * 4 * 2 + 41089 * 4 * 2
    return {"engine_ms_per_step": 1e3 * wall / steps, "engine_samples_per_s": steps * B / wall,
            "eager_ms": {k: round(statistics.median(v), 4) for k, v in parts.items()},
            "n_unique": U, "tower_bytes": tower_bytes, "engine_last_loss": loss}


def dropin_arm(opt, hashed, B, steps, data):
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer
    from elasticdl_b200.workloads.frappe import INPUT_DIM, FrappeDeepFM

    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(1, opt_type, opt_args, device=0)
    model = FrappeDeepFM(lr, input_dim=None if hashed else INPUT_DIM, optimizer=opt).cuda()
    client = PSClient(group)
    client.dense_output = "torch"
    tr = ParameterServerTrainer(model, client, args=types.SimpleNamespace(get_model_steps=1, cuda_graph=True))
    for k in range(6):
        tr.train_minibatch(*data[k % N_BATCHES])
    wall = timed(steps, lambda s: tr.train_minibatch(*data[s % N_BATCHES]))
    why = tr.graph_fallback_reason
    group.close()
    return {"dropin_ms_per_step": 1e3 * wall / steps, "dropin_samples_per_s": steps * B / wall,
            "dropin_path": "graphed" if why is None else "eager (%s)" % why}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--batches", default="64,4096,32768,262144")
    ap.add_argument("--tables", default="hashed,bounded")
    ap.add_argument("--opts", default="sgd,adam")
    ap.add_argument("--no-dropin", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_frappe.py measures on a CUDA device; none is available")
    from elasticdl_b200.workloads.frappe import synthetic_frappe_batch

    dev = torch.device("cuda", 0)
    name, power = card()
    for B in [int(b) for b in args.batches.split(",")]:
        data = [synthetic_frappe_batch(B, 1000 + s, dev, pad_fraction=0.3) for s in range(N_BATCHES)]
        steps = max(20, min(args.steps, args.steps * 4096 // B)) if B > 4096 else args.steps
        for tables in args.tables.split(","):
            for opt in args.opts.split(","):
                row = {"config": "frappe DeepFM, %s tables, async %s lr %g, 1 worker, batch %d"
                                 % (tables, opt, OPTS[opt][2], B),
                       "gpu": name, "power_limit": power, "steps": steps}
                row.update(engine_arm(opt, tables == "hashed", B, steps, data))
                if not args.no_dropin:
                    row.update(dropin_arm(opt, tables == "hashed", B, steps, data))
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
