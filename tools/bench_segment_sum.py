"""Time b200ps_segment_sum at the drop-in trainer path's shape: 38 segments of 32768 ids at dims 8 and 1, launched
without a group handle as ops.GatherRows' backward launches it, with the inverse index of a real dedup of the
benchmark's Zipf batch.  One or more builds of libb200ps.so take turns inside every round, so that clock and
neighbour drift hit them alike.

    python tools/bench_segment_sum.py [--lib PATH ...] [--rounds R] [--iters N]

Prints one JSON line: per library and dim the median, min and max microseconds per call over the rounds (CUDA
events around N back-to-back calls), the GPU's name and its power limit."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from elasticdl_b200 import _lib, ops
    from elasticdl_b200 import build as _build
    from elasticdl_b200.workloads.deepfm import synthetic_batch

    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", help="libb200ps.so to time (default: the in-tree build)")
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    paths = args.lib or [_build.LIB]
    libs = []
    for p in paths:
        h = ctypes.CDLL(os.path.abspath(p))
        h.b200ps_segment_sum.restype, h.b200ps_segment_sum.argtypes = _lib.SYMBOLS["b200ps_segment_sum"]
        libs.append(h)

    dev = torch.device("cuda", 0)
    T, k = 38, 32768
    ids, _, _ = synthetic_batch(k, 1, dev, "zipf")
    _, inv, _ = ops.unique(ids.reshape(-1), T)
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    times = {}
    outs = {}
    for dim in (8, 1):
        vals = torch.randn((T * k, dim), device=dev)
        bufs = [torch.empty_like(vals) for _ in libs]
        for h, out in zip(libs, bufs):  # warm-up, and the outputs every build must agree on
            for _ in range(20):
                assert h.b200ps_segment_sum(None, vals.data_ptr(), inv.data_ptr(), T, k, dim, out.data_ptr(), stream) == 0
        torch.cuda.synchronize()
        outs[dim] = [float((b - bufs[0]).abs().max()) for b in bufs]
        for _ in range(args.rounds):
            for j, (h, out) in enumerate(zip(libs, bufs)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    h.b200ps_segment_sum(None, vals.data_ptr(), inv.data_ptr(), T, k, dim, out.data_ptr(), stream)
                e1.record()
                e1.synchronize()
                times.setdefault((paths[j], dim), []).append(e0.elapsed_time(e1) * 1000.0 / args.iters)
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": smi, "shape": {"T": T, "k": k}, "rounds": args.rounds, "iters": args.iters,
           "max_abs_diff_vs_first_lib": {str(d): v for d, v in outs.items()}, "us_per_call": {}}
    for (p, dim), v in times.items():
        res["us_per_call"]["%s dim=%d" % (p, dim)] = {"median": round(statistics.median(v), 2),
                                                      "min": round(min(v), 2), "max": round(max(v), 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
