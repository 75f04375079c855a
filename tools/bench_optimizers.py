#!/usr/bin/env python
"""Times one push of every optimizer kind at the DeepFM shapes bench.py trains: 76 tables (38 id groups x (wide dim 1
+ deep dim 8), bench.py's row counts), the unique ids of one B = 32768 Zipf batch per group, b200ps_push_rows
replayed from a CUDA graph.  Each kind runs on a fresh single-shard group with the same ids and gradients.

    python tools/bench_optimizers.py [--batch 32768] [--iters 200]

Prints one JSON line per kind: us per push (CUDA events over the replays, median of 5 timed blocks) and the effective
GB/s of the push's algorithmic bytes -- per unique row: its id (8 B), its gradient row, and its record (param and
slots) read and written -- next to Adam's, the existing kind with two slots."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import measured_peak  # noqa: E402

KINDS = {  # name: (opt_type, opt_args, slots)
    "sgd": ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", 0),
    "adam": ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", 2),
    "amsgrad": ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=true;", 3),
    "rmsprop": ("RMSprop", "learning_rate=0.001;rho=0.9;momentum=0.0;epsilon=1e-07;centered=false;", 1),
    "rmsprop_momentum": ("RMSprop", "learning_rate=0.001;rho=0.9;momentum=0.9;epsilon=1e-07;centered=false;", 2),
    "rmsprop_centered": ("RMSprop", "learning_rate=0.001;rho=0.9;momentum=0.0;epsilon=1e-07;centered=true;", 2),
    "rmsprop_centered_momentum": ("RMSprop", "learning_rate=0.001;rho=0.9;momentum=0.9;epsilon=1e-07;centered=true;",
                                  3),
    "adadelta": ("Adadelta", "learning_rate=1.0;rho=0.95;epsilon=1e-07;", 2),
    "adamax": ("Adamax", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;", 2),
    "nadam": ("Nadam", "learning_rate=0.002;beta_1=0.9;beta_2=0.999;epsilon=1e-07;", 2),
}


def time_kind(name, rows, uniq, grads, iters, dev):
    from elasticdl_b200.ps import PSGroup

    ot, oa, n_slots = KINDS[name]
    group = PSGroup(1, ot, oa, device=dev.index, track_rows=False)
    try:
        tids = []
        for g, r in enumerate(rows):
            tids.append(group.register_table("w%d" % g, 1, "zero", r))
            tids.append(group.register_table("d%d" % g, 8, "zero", r))
        group.commit()
        items = []
        for g, u in enumerate(uniq):
            items.append((tids[2 * g], u.numel(), u, None, grads[g][0]))
            items.append((tids[2 * g + 1], u.numel(), u, None, grads[g][1]))
        group.push_begin(0.0, [0])  # step 1: every per-push scalar is that of a real push
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            group.push_rows(items)  # warm-up outside the capture
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            group.push_rows(items)
        for _ in range(10):
            graph.replay()
        times = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(iters):
                graph.replay()
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1) * 1e3 / iters)
        group.check()
        n = sum(u.numel() for u in uniq)
        nbytes = n * (8 + 4 * (1 + 8) + 2 * 4 * (1 + 8) * (1 + n_slots))
        us = float(np.median(times))
        return {"kind": name, "slots": n_slots, "us_per_push": us, "gbs": nbytes / (us * 1e-6) / 1e9,
                "unique_rows": n, "bytes": nbytes, "us_blocks": times}
    finally:
        group.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--kinds", default=",".join(KINDS))
    args = ap.parse_args()
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, synthetic_batch

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ids, _, _ = synthetic_batch(args.batch, 1, dev, "zipf", group_rows=GROUP_ROWS)
    gen = torch.Generator(device=dev).manual_seed(2)
    uniq, grads = [], []
    for g in range(len(GROUP_ROWS)):
        u = torch.unique(ids[g])
        uniq.append(u.contiguous())
        grads.append((torch.randn((u.numel(), 1), generator=gen, device=dev),
                      torch.randn((u.numel(), 8), generator=gen, device=dev)))
    peak, peak_kind = measured_peak()
    res = {k: time_kind(k, GROUP_ROWS, uniq, grads, args.iters, dev) for k in args.kinds.split(",")}
    adam = res.get("adam")
    for k, r in res.items():
        r["hbm_frac"] = r["gbs"] / peak
        r["peak_kind"] = peak_kind
        if adam is not None:
            r["us_vs_adam"] = r["us_per_push"] / adam["us_per_push"]
        r["gpu"] = torch.cuda.get_device_name(dev)
        print(json.dumps(r))


if __name__ == "__main__":
    main()
