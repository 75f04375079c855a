#!/usr/bin/env python
"""Upper bounds on what each part of the benchmarked DeepFM step costs, from bench.py's own workload.

    python tools/step_ceilings.py [--rounds 7] [--replays 200] [--warmup 50] [--json OUT]

The script builds bench.py's engine (1 GPU, B = 32768, tile tower reading the table records, narrow packed ids,
the same seeds and batch pool) and captures its lookahead CUDA graph several times, each time with some nodes
left out.  A variant without a node computes wrong results: it exists to be timed only, and the difference to
"full" bounds what removing or hiding that node can save.

    full      every node
    no-head   the dense pull and the tower prologue (the tower reads the W1x and parameters left by earlier steps;
              the tile counter is reset by a fill at the end of the step so the tower still runs every tile)
    no-tail   the loss publish and the push's version bump (k_publish_loss, k_push_end)
    no-dedup  the next batch's dedup on the side stream
    no-push   the row push (k_push_flat)

The variants alternate round by round in one process, so a drift of the clock or a neighbour's load hits all of
them alike; each round times `replays` back-to-back replays with CUDA events.  The card's name, power limit and SM
clock are read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = ("full", "no-head", "no-tail", "no-dedup", "no-push")


class _SkipLib:
    """The library with some entry points replaced by no-ops that return success."""

    def __init__(self, real, skip):
        self._real, self._skip = real, set(skip)

    def __getattr__(self, name):
        if name in self._skip:
            return lambda *args: 0
        return getattr(self._real, name)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "-i", os.environ.get("LOCAL_RANK", "0"),
                              "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as e:  # the timings stand without it; say why it is missing
        return {"error": repr(e)}


def capture_variant(engine, variant, counter, grid):
    """The engine's two lookahead graphs with the nodes of `variant` left out."""
    import torch

    group = engine.group
    real_lib, real_calls = group.lib, engine.calls
    real_end, real_publish, real_unique = group.push_end, engine._publish_loss, engine._unique_into
    skip = {"no-head": ("b200ps_pull_dense",), "no-tail": ("b200_deepfm_publish_loss",),
            "no-push": ("b200ps_push_rows",)}.get(variant, ())
    try:
        group.lib = _SkipLib(real_lib, skip)
        if variant == "no-head":
            engine.calls = real_calls._replace(prologue=lambda args, st: 0)

            def publish_then_reset(loss, st):
                real_publish(loss, st)
                counter.fill_(grid)  # on the stream the publish runs on: the end of the dense branch

            engine._publish_loss = publish_then_reset
        elif variant == "no-tail":
            group.push_end = lambda sync=True: None
        elif variant == "no-dedup":
            engine._unique_into = lambda ids: None
        engine.graphs_ahead = None
        graphs = engine.capture_ahead()
    finally:
        group.lib, engine.calls = real_lib, real_calls
        for obj, name in ((group, "push_end"), (engine, "_publish_loss"), (engine, "_unique_into")):
            obj.__dict__.pop(name, None)
    torch.cuda.synchronize()
    return graphs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--pool", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--replays", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--json", default=None, help="also write the result here")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("step_ceilings.py: no CUDA device")
    from bench import ADAM_ARGS
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch, synthetic_batch

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    engine = DeepFMPSEngine(group, args.batch, tower="tile", paired=False, exchange=None, id_transport="narrow")
    assert engine.row_source == "table" and engine.model == "deepfm"
    devp = []
    for p in range(args.pool):
        ids, dense, labels = synthetic_batch(args.batch, 1234 + p, dev, "zipf")
        devp.append(pack_batch(ids, dense, labels, widths=engine.widths))
    # the tile counter follows W1x [320][16] in the scratch buffer (deepfm_tower2.cu); the grid is
    # launch_tile_tower's: two CTAs per SM, at most one per tile
    counter = engine.scratch[320 * 16:320 * 16 + 1].view(torch.int32)
    grid = min(2 * torch.cuda.get_device_properties(dev).multi_processor_count, (args.batch + 31) // 32)

    graphs = {v: capture_variant(engine, v, counter, grid) for v in VARIANTS}
    engine.graphs_ahead = graphs["full"]
    engine.prepare_packed(devp[0])
    k = 0

    def replay(v, n):
        nonlocal k
        engine.graphs_ahead = graphs[v]
        for _ in range(n):
            k += 1
            engine.step_ahead_graph(devp[k % args.pool])

    for v in VARIANTS:
        replay(v, args.warmup)
    torch.cuda.synchronize()
    info = gpu_info()
    ms = {v: [] for v in VARIANTS}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
        for v in VARIANTS:
            replay(v, 5)
            e0.record()
            replay(v, args.replays)
            e1.record()
            torch.cuda.synchronize()
            ms[v].append(e0.elapsed_time(e1) / args.replays)
    info_end = gpu_info()
    group.check()
    full = statistics.median(ms["full"])
    rows = []
    for v in VARIANTS:
        med = statistics.median(ms[v])
        rows.append({"variant": v, "median_us": 1e3 * med, "min_us": 1e3 * min(ms[v]), "max_us": 1e3 * max(ms[v]),
                     "saves_us": 1e3 * (full - med), "saves_pct": 100.0 * (full - med) / full})
    print("| variant | median µs/step | min–max µs | bound: saves µs (%) |")
    print("|---|---|---|---|")
    for r in rows:
        print("| %s | %.1f | %.1f–%.1f | %.1f (%.1f %%) |" % (r["variant"], r["median_us"], r["min_us"], r["max_us"],
                                                        r["saves_us"], r["saves_pct"]))
    out = {"gpu": info, "gpu_after": info_end, "rounds": args.rounds, "replays": args.replays, "batch": args.batch,
           "variants": rows, "ms_per_round": ms}
    print(json.dumps(out))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)
    group.close()


if __name__ == "__main__":
    main()
