#!/usr/bin/env python
"""Where does the e2e step lose time against the device-resident step?  Same engine, same graphs, K steps each:
  value      step_ahead_graph on device-resident packed batches (what bench.py's `value` times)
  feeder_dev the HostFeeder fed with DEVICE batches (same Python, D2D instead of H2D copies)
  feeder_h2d the HostFeeder fed with pinned HOST batches (what bench.py's `e2e` times)
  value+dma  `value` while an unrelated stream keeps copying 4 MB pinned buffers H2D (nobody reads them)
and the per-kernel CUDA-event times of eager steps with and without that background DMA."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ADAM_ARGS  # noqa: E402
from elasticdl_b200.ps import PSGroup  # noqa: E402
from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch, synthetic_batch  # noqa: E402


def main():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    B, pool, K, W = 32768, 8, 40, 8
    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    eng = DeepFMPSEngine(group, B, tower="tile", id_transport="narrow")
    devb, devp, host = [], [], []
    for p in range(pool):
        ids, dense, labels = synthetic_batch(B, 1234 + p, dev, "zipf")
        devb.append((ids, dense, labels))
        devp.append(pack_batch(ids, dense, labels, widths=eng.widths))
        host.append(pack_batch(ids.cpu(), dense.cpu(), labels.cpu(), pin=True, widths=eng.widths))
    for i in range(3):
        eng.step(*devb[i])
    eng.capture_ahead()
    eng.prepare_packed(devp[0])
    out = {}

    def timed(fn, n=K, warm=W):
        for i in range(warm):
            fn(i)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for i in range(warm, warm + n):
            fn(i)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / n * 1e3

    out["value_us"] = timed(lambda i: eng.step_ahead_graph(devp[(i + 1) % pool]))

    # background DMA: an unrelated stream copying pinned buffers to a scratch device buffer, back to back
    bg_stream = torch.cuda.Stream(device=dev)
    scratch = torch.empty_like(devp[0])
    stop = {"n": 0}

    def bg_enqueue(n):
        with torch.cuda.stream(bg_stream):
            for j in range(n):
                scratch.copy_(host[j % pool], non_blocking=True)

    def value_dma(i):
        bg_enqueue(2)  # two 4 MB copies per step keep the link busy
        eng.step_ahead_graph(devp[(i + 1) % pool])

    out["value_with_background_h2d_us"] = timed(value_dma)
    bg_stream.synchronize()

    def value_dma1(i):
        bg_enqueue(1)  # one 4 MB copy per step: the e2e volume
        eng.step_ahead_graph(devp[(i + 1) % pool])

    out["value_with_one_h2d_per_step_us"] = timed(value_dma1)
    bg_stream.synchronize()

    for name, src in (("feeder_dev_us", devp), ("feeder_h2d_us", host)):
        feeder = eng.host_feeder(3, lookahead=True)
        feeder.started = True  # the plan of the running pipeline is already prepared
        for j in range(2):
            feeder.submit(src[j % pool])

        def fstep(i, feeder=feeder, src=src):
            feeder.submit(src[(i + 2) % pool])
            feeder.run_next()

        out[name] = timed(fstep)
        torch.cuda.synchronize()

    # per-kernel: eager steps with CUDA-event pairs, GPU kept busy in front
    def per_kernel(with_dma):
        ev = {}
        torch.cuda.synchronize()
        for i in range(12):
            torch.cuda._sleep(2_000_000)
            if with_dma:
                bg_enqueue(3)
            eng.step(*devb[i % pool], ev=ev)
        torch.cuda.synchronize()
        return {k: round(sum(a.elapsed_time(b) for a, b in v[2:]) / len(v[2:]) * 1e3, 1) for k, v in ev.items()}

    out["eager_kernels_us"] = per_kernel(False)
    out["eager_kernels_with_background_h2d_us"] = per_kernel(True)
    group.check()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
