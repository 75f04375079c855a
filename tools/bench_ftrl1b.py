#!/usr/bin/env python
"""BASELINE.json configs[4]: one embedding table of 1 B slots, dim 8, FTRL (lr 0.1, l1 = l2 = 0, initial
accumulator 0.1), PS shards striped over the GPUs (id % N), B = 262144 ids per push drawn over the whole
1e9 range (uniform, or Zipf 1.05), seed 99 (SURVEY.md section 8d item 5).

    python tools/bench_ftrl1b.py [--rows 1000000000] [--batch 262144] [--dist uniform|zipf]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port 29551 \
        tools/bench_ftrl1b.py

--rows defaults to 1e9 over two or more GPUs and to 5e8 on one: 1e9 records of 96 B (96 GB) exceed one H100's
80 GB, 5e8 (48 GB) leave room for the id pool, workspaces and the CUDA context.

One step per rank = unique (hashed: ids are unbounded for the dedup) -> pull rows -> synthetic gradient ->
push (FTRL fused in the row kernel, params + accumulator + linear in one 96 B record).  At N > 1 every rank
addresses all shards directly (flat kernels over peer-mapped slabs).  Rank 0 first checks one push of
rank-private ids against the oracle's FTRL (np_ftrl: TF ApplyFtrl restated, PARITY UNPINNED) bit for bit.
Prints one JSON line: pushes/s (ids/s, whole job), ms per step (max over ranks, CUDA events), algorithmic
GB/s of pull and push and their fraction of the measured HBM peak."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import measured_peak  # noqa: E402

FTRL = ("Ftrl", "learning_rate=0.1;initial_accumulator_value=0.1;l1_regularization_strength=0.0;"
                "l2_regularization_strength=0.0;l2_shrinkage_regularization_strength=0.0;beta=0.0;")


def draw_ids(n, rows, dist_kind, gen, dev):
    u = torch.rand(n, generator=gen, device=dev, dtype=torch.float64)
    if dist_kind == "zipf":
        a = 1.0 - 1.05
        ids = torch.floor(((rows ** a - 1.0) * u + 1.0).pow(1.0 / a)) - 1.0
    else:
        ids = torch.floor(u * rows)
    return ids.clamp_(0, rows - 1).to(torch.int64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=0, help="table slots (0: 1e9, or 5e8 on a single GPU)")
    ap.add_argument("--dim", type=int, default=8)
    ap.add_argument("--batch", type=int, default=262144)
    ap.add_argument("--dist", default="uniform", choices=["uniform", "zipf"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    if args.rows <= 0:
        args.rows = 1_000_000_000 if world > 1 else 500_000_000
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("NCCL_DEBUG", "WARN")
        dist.init_process_group("nccl", device_id=dev)
    from elasticdl_b200._lib import check
    from elasticdl_b200.ps import PSGroup

    group = PSGroup(world, *FTRL, device=local, local_shards=[rank] if world > 1 else None, track_rows=False)
    tid = group.register_table("big/embeddings:0", args.dim, "zero", args.rows)
    group.commit()
    lib, h = group.lib, group._h
    B, D = args.batch, args.dim
    gen = torch.Generator(device=dev).manual_seed(99 + rank)
    pool = [draw_ids(B, args.rows, args.dist, gen, dev) for _ in range(8)]
    ws = torch.zeros(lib.b200ps_unique_workspace(1, B), dtype=torch.uint8, device=dev)
    uniq = torch.empty(B, dtype=torch.int64, device=dev)
    inv = torch.empty(B, dtype=torch.int32, device=dev)
    n_u = torch.empty(1, dtype=torch.int32, device=dev)
    rows = torch.empty((B, D), dtype=torch.float32, device=dev)
    grads = torch.empty((B, D), dtype=torch.float32, device=dev)
    noise = torch.randn((B, D), generator=gen, device=dev) * 1e-2
    seg_pull = group.make_segs([(tid, B, uniq, n_u, rows)])
    seg_push = group.make_segs([(tid, B, uniq, n_u, grads)])
    st = group._stream()

    def sync():
        torch.cuda.synchronize(dev)
        if world > 1:
            dist.barrier()
            torch.cuda.synchronize(dev)

    # ---- parity: one push of rank-0-only ids against the oracle's FTRL (first touch: p = 0, accum = 0.1, linear = 0)
    parity = None
    sync()
    if rank == 0:
        from oracle import ps_oracle as O

        ids = torch.unique(draw_ids(4096, args.rows, "uniform", torch.Generator(device=dev).manual_seed(7), dev))
        g = (torch.randn((ids.numel(), D), generator=torch.Generator(device=dev).manual_seed(8), device=dev) * 0.1)
        group.push_begin(0.1, [0] * world)
        group.push_rows([(tid, ids.numel(), ids, None, g)])
        group.push_end()
        got = group.pull_rows([("big/embeddings:0", ids)])[0].cpu().numpy()
        acc = group.slot_rows("big/embeddings:0", ids, 1).cpu().numpy()
        lin = group.slot_rows("big/embeddings:0", ids, 2).cpu().numpy()
        p = np.zeros_like(got)
        a0 = np.full_like(got, 0.1)
        l0 = np.zeros_like(got)
        O.np_ftrl(g.cpu().numpy().copy(), p, a0, l0, 0.1, 0.0, 0.0, 0.0)
        ok = np.array_equal(got, p) and np.array_equal(acc, a0) and np.array_equal(lin, l0)
        parity = {"ftrl_first_push_vs_oracle": "bit-exact" if ok else "MISMATCH", "rows": int(ids.numel()),
                  "note": "oracle FTRL is restated from TF ApplyFtrl: parity unpinned"}
        if not ok:
            print(json.dumps({"parity": parity}), file=sys.stderr)
            raise SystemExit(3)
    sync()

    ev = {"unique": [], "pull": [], "push": []}

    def step(i, timed):
        ids = pool[i % len(pool)]

        def mark(name):
            if not timed:
                return None
            e = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev[name].append(e)
            e[0].record()
            return e

        e = mark("unique")
        check(lib.b200ps_unique(h, ids.data_ptr(), 1, B, uniq.data_ptr(), inv.data_ptr(), n_u.data_ptr(), ws.data_ptr(),
                                ws.numel(), st))
        if e:
            e[1].record()
        e = mark("pull")
        check(lib.b200ps_pull_rows(h, seg_pull[0], seg_pull[1], st))
        if e:
            e[1].record()
        torch.add(noise, rows, alpha=0.01, out=grads)  # synthetic gradient of the pulled rows
        group.push_begin(0.1, [0] * world)
        e = mark("push")
        check(lib.b200ps_push_rows(h, seg_push[0], seg_push[1], st))
        if e:
            e[1].record()
        group.push_end(sync=False)

    for i in range(args.warmup):
        step(i, False)
    sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        torch.cuda._sleep(2_000_000)  # keep the GPU ahead of the host: the event pairs bracket device time
        step(args.warmup + i, True)
    e1.record()
    sync()
    group.check()
    n_unique = int(n_u.item())
    per = {k: sum(a.elapsed_time(b) for a, b in v) / len(v) for k, v in ev.items()}
    step_ms = per["unique"] + per["pull"] + per["push"]
    if world > 1:
        t = torch.tensor([step_ms, per["unique"], per["pull"], per["push"]], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        step_ms, per["unique"], per["pull"], per["push"] = (float(x) for x in t.tolist())
    peak, kind = measured_peak()
    if rank == 0:
        b_pull, b_push = n_unique * (8 + 8 * D), n_unique * (8 + 4 * D + 3 * 8 * D)
        out = {"workload": "1 B-slot table, dim %d, FTRL, %d ids per push per rank, %s ids" % (D, B, args.dist),
               "rows": args.rows, "table_bytes_total": args.rows * 4 * D * 3, "n_gpus": world, "steps": args.steps,
               "ids_per_sec": world * B / (step_ms * 1e-3), "ms_per_step_device": step_ms,
               "unique_ids_per_push": n_unique, "kernels_ms": per,
               "pull_gbs": b_pull / per["pull"] / 1e6, "push_gbs": b_push / per["push"] / 1e6,
               "pull_frac_of_hbm_peak": b_pull / per["pull"] / 1e6 / peak,
               "push_frac_of_hbm_peak": b_push / per["push"] / 1e6 / peak, "peak": peak, "peak_kind": kind,
               "parity": parity,
               "note": "device time of unique + pull + push per step (CUDA events, max over ranks); at N > 1 rows of "
                       "peer shards are read / updated over NVLink (7/8 of them at N = 8), so the HBM fraction is "
                       "bounded by scattered 32 B peer accesses, not by HBM"}
        print(json.dumps(out))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
