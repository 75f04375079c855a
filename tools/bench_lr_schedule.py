"""What a learning-rate schedule costs on the step, H100.  Alternating rounds in one process, medians reported:

  * the drop-in trainer (ParameterServerTrainer, DeepFM layers model, B = 32768, Adam, args.cuda_graph) with a
    constant lr, with a per-step ExponentialDecay installed on the device (train_loop callbacks), and with the same
    schedule as a Python callable (the host sets the lr; the lr changes every step);
  * the DeepFM engine's captured step (step_graph) without and with a device schedule.

Prints one JSON object (card, power limit, ms per step)."""
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

from elasticdl_b200 import callbacks as cb  # noqa: E402
from elasticdl_b200.ps import PSGroup  # noqa: E402
from elasticdl_b200.worker.ps_client import PSClient  # noqa: E402
from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer  # noqa: E402
from elasticdl_b200.workloads.deepfm import DeepFMLayersModel, DeepFMPSEngine, pack_batch, synthetic_batch  # noqa: E402

ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    return out.splitlines()[0] if out else torch.cuda.get_device_name(0)


def trainer_legs(dev, batches, warmup):
    sched = cb.ExponentialDecay(1e-3, 1, 0.999)
    legs = {}
    for mode in ("constant", "device_schedule", "callable_schedule"):
        group = PSGroup(1, *ADAM, device=dev.index)
        client = PSClient(group)
        client.dense_output = "torch"
        model = DeepFMLayersModel().to(dev)
        trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
            get_model_steps=1, batched_embedding_lookups=True, cuda_graph=True, cuda_graph_warmup=warmup))
        callbacks = None
        if mode != "constant":
            callbacks = [cb.LearningRateScheduler(sched if mode == "device_schedule" else (lambda v: sched(v)))]
        legs[mode] = (trainer, callbacks, group)
        trainer.train_loop(batches[: warmup + 2], callbacks=callbacks)  # warm-up, capture, one replay
    return legs


def time_trainer(leg, batches, k, dev):
    trainer, callbacks, _ = leg
    torch.cuda.synchronize(dev)
    eager0 = trainer._eager_steps
    t0 = time.perf_counter()
    trainer.train_loop([batches[i % len(batches)] for i in range(k)], callbacks=callbacks)
    torch.cuda.synchronize(dev)
    return (time.perf_counter() - t0) / k * 1e3, trainer._eager_steps - eager0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32768)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    B = args.batch
    raw = [synthetic_batch(B, 100 + i, dev, "zipf") for i in range(8)]
    feats = [(DeepFMLayersModel.features_of(ids, dense), labels) for ids, dense, labels in raw]
    legs = trainer_legs(dev, feats, args.warmup)
    engines = {}
    for mode in ("constant", "device_schedule"):
        group = PSGroup(1, *ADAM, device=0)
        eng = DeepFMPSEngine(group, B, lr_schedule=cb.ExponentialDecay(1e-3, 1, 0.999) if mode != "constant" else None)
        eng.capture()
        packed = [pack_batch(ids, dense, labels, widths=eng.widths) for ids, dense, labels in raw]
        for p in packed[:3]:
            eng.step_graph(p)
        engines[mode] = (eng, packed, group)
    res = {m: [] for m in legs}
    eager = {m: 0 for m in legs}
    eng_res = {m: [] for m in engines}
    for _ in range(args.rounds):
        for m in legs:
            ms, n_eager = time_trainer(legs[m], feats, args.steps, dev)
            res[m].append(ms)
            eager[m] += n_eager
        for m, (eng, packed, _) in engines.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize(dev)
            s.record()
            for i in range(args.steps * 4):
                eng.step_graph(packed[i % len(packed)])
            e.record()
            torch.cuda.synchronize(dev)
            eng_res[m].append(s.elapsed_time(e) / (args.steps * 4))
    for _, _, g in list(legs.values()) + list(engines.values()):
        g.check()
    out = {"card": card(), "batch": B, "rounds": args.rounds, "steps_per_round": args.steps, "trainer": {}, "engine": {}}
    for m, (trainer, _, _) in legs.items():
        out["trainer"][m] = {"ms_per_step_median": statistics.median(res[m]), "ms_per_step_rounds": res[m],
                             "eager_steps_timed": eager[m], "cuda_graph": isinstance(trainer._graph_state, dict),
                             "graph_fallback_reason": trainer.graph_fallback_reason}
    for m in engines:
        out["engine"][m] = {"ms_per_step_median": statistics.median(eng_res[m]), "ms_per_step_rounds": eng_res[m]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
