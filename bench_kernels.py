#!/usr/bin/env python
"""Kernel-level roofline sweep of the PS kernels (not the driver's bench: see bench.py).

For each kernel: algorithmic bytes (SURVEY.md 8d) / CUDA-event time on the launching stream,
against MEASURED_PEAKS.json:hbm_gbs.  Working sets exceed the 50 MB L2 (5.5 M-row tables,
ResNet-50-sized dense parameter), ids are unique and uniformly random.  One JSON line per case.
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from bench import measured_peak  # noqa: E402

ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")
SGD = ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;")


def timeit(fn, iters=20, warmup=3):
    """Average device time of one call: `iters` calls captured into ONE CUDA graph and replayed between two
    events (launching them eagerly from Python leaves the GPU idle between kernels shorter than the ~20 us
    of host work per call, and the event pair then measures the host)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(iters):
            fn()
    g.replay()
    torch.cuda.synchronize()
    ms = []
    for _ in range(3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b) / iters)
    return sorted(ms)[1]


def main():
    from elasticdl_b200.ps import PSGroup

    peak, kind = measured_peak()
    dev = torch.device("cuda", 0)
    rows = 5_549_416
    out = []
    only = os.environ.get("BK_ONLY", "")  # e.g. "adam:8" -> one optimizer / dim (tuning sweeps)
    sizes = [int(x) for x in os.environ.get("BK_SIZES", "122000,1000000,4000000").split(",")]  # unique ids per launch
    for opt_name, opt, S in (("adam", ADAM, 2), ("sgd", SGD, 0)):
        if only and not only.startswith(opt_name):
            continue
        group = PSGroup(1, *opt, device=0, track_rows=True)
        for dim in (8, 1, 64):
            if only and ":" in only and int(only.split(":")[1]) != dim:
                continue
            name = "t%d" % dim
            tid = group.register_table(name, dim, "zero", rows)
            group.commit()
            for U in sizes:
                pools = []
                for p in range(3):  # rotate id sets so consecutive launches touch different rows
                    ids = torch.randperm(rows, device=dev)[:U].contiguous()
                    pools.append(ids)
                outbuf = torch.empty((U, dim), device=dev)
                grads = torch.randn((U, dim), device=dev) * 1e-3
                state = {"i": 0}

                def pull():
                    ids = pools[state["i"] % 3]
                    state["i"] += 1
                    arr, n = group.make_segs([(tid, U, ids, None, outbuf)])
                    group.lib.b200ps_pull_rows(group._h, arr, n, group._stream())

                def push():
                    ids = pools[state["i"] % 3]
                    state["i"] += 1
                    arr, n = group.make_segs([(tid, U, ids, None, grads)])
                    group.lib.b200ps_push_rows(group._h, arr, n, group._stream())

                group.push_begin(0.001, [0])
                ms_pull = timeit(pull)
                ms_push = timeit(push)
                b_pull = U * (8 + 8 * dim)
                b_push = U * (8 + 4 * dim + (1 + S) * 8 * dim)
                for kname, ms, nb in (("pull_rows", ms_pull, b_pull), ("push_rows_" + opt_name, ms_push, b_push)):
                    if kname == "pull_rows" and opt_name == "sgd":
                        continue
                    line = {"kernel": kname, "dim": dim, "unique_ids": U, "table_rows": rows, "us": ms * 1e3,
                            "algorithmic_bytes": nb, "gbs": nb / ms / 1e6, "frac_of_peak": nb / ms / 1e6 / peak,
                            "peak": peak, "peak_kind": kind, "record_bytes": 4 * ((dim * (S + 1) + 3) // 4 * 4)}
                    print(json.dumps(line), flush=True)
                    out.append(line)
        group.check()
        if only:
            group.close()
            continue
        # dense fused update, ResNet-50-sized parameter (25.6 M fp32)
        n = 25_600_000
        group.register_dense("resnet50_flat", (n,), 0)
        group.commit()
        g = [torch.randn(n, device=dev) * 1e-3 for _ in range(8)]
        for R in (1, 2, 8):
            def dense():
                group.push_dense_reduce("resnet50_flat", g[:R], scale=1.0 / R)
            group.push_begin(0.001, [0])
            ms = timeit(dense)
            nb = n * 4 * (R + 2 * (1 + S))
            line = {"kernel": "push_dense_reduce_" + opt_name, "numel": n, "replicas": R, "us": ms * 1e3,
                    "algorithmic_bytes": nb, "gbs": nb / ms / 1e6, "frac_of_peak": nb / ms / 1e6 / peak, "peak": peak,
                    "peak_kind": kind}
            print(json.dumps(line), flush=True)
        group.close()
        del g
        torch.cuda.empty_cache()
    if only:
        return
    # unique / segment_sum at scale
    from elasticdl_b200 import ops

    for k, hi in ((1_245_184, 5_549_416), (8_000_000, 100_000_000)):
        ids = torch.randint(0, hi, (k,), device=dev)
        ms = timeit(lambda: ops.unique(ids, 1))
        uniq, inv, nu = ops.unique(ids, 1)
        U = int(nu.item())
        nb = k * 12 + U * 8
        print(json.dumps({"kernel": "unique(1 persistent kernel)", "k": k, "unique": U, "us": ms * 1e3,
                          "algorithmic_bytes": nb, "gbs": nb / ms / 1e6, "frac_of_peak": nb / ms / 1e6 / peak}), flush=True)
        vals = torch.randn((k, 8), device=dev)
        ms = timeit(lambda: ops.segment_sum(vals, inv, 1, k, 8))
        nb = k * 36 + U * 32
        print(json.dumps({"kernel": "segment_sum_dim8", "k": k, "unique": U, "us": ms * 1e3,
                          "algorithmic_bytes": nb, "gbs": nb / ms / 1e6, "frac_of_peak": nb / ms / 1e6 / peak}), flush=True)


if __name__ == "__main__":
    main()
