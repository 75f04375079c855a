"""DeepFM, DCN, Wide & Deep and xDeepFM engine steps side by side: bench.py's workload (B = 32768, the 38 dac_ctr
groups, Adam, its Zipf batches, narrow packed ids, the graphed lookahead pipeline) run for DeepFMPSEngine(model=m),
m in MODELS, alternating in one process over several repeats (the order rotates from repeat to repeat).

Prints, per model, ms/step and samples/s of the graphed steps (median and spread over the repeats) and the
tower's CUDA-event time (eager steps with event pairs, each step queued behind a spin kernel as bench.py does),
plus the card's name and power limit read in the same run.  For xDeepFM also the CIN's algorithmic rate,
2 x 128 x 8 x (G^2 + 64 G) x 3 x B FLOP (forward, data and weight passes) over the tower's event time, the 3xTF32
tensor rate that implies (three TF32 products per fp32 product) against the 495 TF/s dense TF32 data-sheet peak,
and the same steps on tower="torch" (eager, same batches).  One JSON line at the end.

    python tools/bench_dcn.py [--steps 50] [--warmup 10] [--repeats 5] [--pool 8]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


MODELS = ("deepfm", "dcn", "wide_deep", "xdeepfm")
TF32_PEAK = 495e12  # H100 SXM data sheet, dense TF32


def cin_flop(G, B):
    """The CIN's algorithmic FLOP of one training step: three contractions of 2 x 128 x 8 x (G^2 + 64 G) per sample."""
    return 2 * 128 * 8 * (G * G + 64 * G) * 3 * B


def card():
    import torch

    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit"], out["max_sm_clock"] = (v.strip() for v in q.split(","))
    except (OSError, ValueError, subprocess.SubprocessError) as e:
        out["power_limit"] = "unknown (%s)" % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--pool", type=int, default=8)
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_dcn.py measures on the GPU; none is available")
    from bench import ADAM_ARGS
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch, synthetic_batch

    dev = torch.device("cuda", 0)
    B = args.batch
    models = MODELS
    groups, engines, devb, devp = {}, {}, {}, {}
    for m in models:
        groups[m] = PSGroup(1, "Adam", ADAM_ARGS, device=0)
        engines[m] = DeepFMPSEngine(groups[m], B, id_transport="narrow", model=m)
        devb[m] = [synthetic_batch(B, 1234 + p, dev, "zipf") for p in range(args.pool)]
        devp[m] = [pack_batch(*b, widths=engines[m].widths) for b in devb[m]]

    # tower time: eager steps with CUDA-event pairs, each queued behind a spin kernel (device time, not host time)
    tower_ms = {}
    for m in models:
        eng = engines[m]
        for i in range(args.warmup):
            eng.step(*devb[m][i % args.pool])
        ev = {}
        for i in range(args.steps):
            torch.cuda._sleep(4_000_000)
            eng.step(*devb[m][i % args.pool], ev=ev)
        torch.cuda.synchronize(dev)
        groups[m].check()
        tower_ms[m] = eng.kernel_report(ev, [1])["tower_fwd_bwd"]["ms"]

    # xDeepFM on the torch tower, eager, same batches: the tile tower's step must beat it
    tg = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    te = DeepFMPSEngine(tg, B, id_transport="narrow", model="xdeepfm", tower="torch")
    for i in range(2):
        te.step(*devb["xdeepfm"][i % args.pool])
    torch.cuda.synchronize(dev)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    n_torch = max(3, args.steps // 10)
    for i in range(n_torch):
        te.step(*devb["xdeepfm"][i % args.pool])
    t1.record()
    torch.cuda.synchronize(dev)
    torch_ms = t0.elapsed_time(t1) / n_torch
    tg.check()
    tg.close()

    # the graphed lookahead step, the models alternating repeat by repeat
    for m in models:
        engines[m].capture_ahead()
        engines[m].prepare_packed(devp[m][0])
    pos = {m: 0 for m in models}
    ms = {m: [] for m in models}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for r in range(args.repeats):
        for m in models[r % len(models):] + models[:r % len(models)]:
            eng = engines[m]
            for _ in range(args.warmup):
                pos[m] += 1
                eng.step_ahead_graph(devp[m][pos[m] % args.pool])
            torch.cuda.synchronize(dev)
            e0.record()
            for _ in range(args.steps):
                pos[m] += 1
                eng.step_ahead_graph(devp[m][pos[m] % args.pool])
            e1.record()
            torch.cuda.synchronize(dev)
            groups[m].check()
            ms[m].append(e0.elapsed_time(e1) / args.steps)
    info = card()
    result = {"card": info, "batch": B, "steps": args.steps, "repeats": args.repeats, "models": {}}
    for m in models:
        med = statistics.median(ms[m])
        result["models"][m] = {"ms_per_step": med, "ms_min": min(ms[m]), "ms_max": max(ms[m]),
                               "samples_per_s": B / (med * 1e-3), "tower_ms": tower_ms[m],
                               "final_loss": engines[m].loss_host(engines[m].steps - 1)}
        print("%-9s  %.4f ms/step (min %.4f, max %.4f over %d repeats)  %.3g samples/s  tower %.4f ms" % (
            m, med, min(ms[m]), max(ms[m]), args.repeats, B / (med * 1e-3), tower_ms[m]))
    print("card: %s, power limit %s, max SM clock %s" % (info["name"], info.get("power_limit"), info.get("max_sm_clock")))
    G = engines["xdeepfm"].G
    rate = cin_flop(G, B) / (tower_ms["xdeepfm"] * 1e-3)
    x = result["models"]["xdeepfm"]
    x.update({"torch_tower_ms_per_step": torch_ms, "cin_tflops": rate / 1e12, "tf32_tensor_tflops": 3 * rate / 1e12,
              "tf32_share_of_peak": 3 * rate / TF32_PEAK})
    print("xdeepfm CIN: %.1f GFLOP per step, %.1f TFLOP/s algorithmic over the tower time, %.1f TFLOP/s of TF32 "
          "products = %.1f%% of the 495 TF/s data-sheet peak; tower=\"torch\" eager step %.3f ms" % (
              cin_flop(G, B) / 1e9, rate / 1e12, 3 * rate / 1e12, 100 * 3 * rate / TF32_PEAK, torch_ms))
    for g in groups.values():
        g.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
