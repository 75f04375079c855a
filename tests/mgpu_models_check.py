"""The Wide & Deep and DCN engines on the owner-computes exchange (torchrun, one rank per GPU; B200_SHARED_GPU=1 puts
every rank on cuda:0 as its own process).  For each model, every rank:
  - conditions its first batch on the known initial state (the engine's seeded rows and tower), so that no sample
    sits within rounding of a ReLU kink;
  - runs one eager step and, right after the tower, copies what the exchange pulled into bet_w / bet_d, the plan's
    dedup, the dense parameters and the tower's outputs;
  - checks the pulled rows against the initial rows and the tower's loss, logits, flat_grads and gsum_w / gsum_d
    against the float64 reference on those rows (oracle/wide_deep_oracle.py, oracle/dcn_oracle.py);
  - trains a few more steps, eagerly and from its CUDA graph, and the loss falls."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticdl_b200.ps import PSGroup  # noqa: E402
from oracle import dcn_oracle, wide_deep_oracle  # noqa: E402

ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")
ROWS = [11, 5000, 60000, 9, 300]
B = 2048


def _reference(model):
    """(reference(inputs...), oracle module) of a model."""
    if model == "dcn":
        return dcn_oracle.dcn_reference, dcn_oracle
    return wide_deep_oracle.wide_deep_reference, wide_deep_oracle


def _initial_rows(eng, dev, seed=7, init_std=0.01):
    """The rows DeepFMPSEngine(init_rows=True) set on creation, regenerated: (wide [G] of [r], deep [G] of [r, 8])."""
    gen = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for dim in (1, eng.D):
        out.append([torch.randn((r, dim), generator=gen, device=dev) * init_std for r in ROWS])
    return [w.reshape(-1) for w in out[0]], out[1]


def _gather_rows(wide, deep, uniq, n_unique, G):
    """bet_wide [G, B] / bet_deep [G, B, 8] of the unique ids (NaN past n_unique[g])."""
    dev = uniq.device
    bw = torch.full((G, B), float("nan"), device=dev)
    bd = torch.full((G, B, 8), float("nan"), device=dev)
    for g in range(G):
        u = int(n_unique[g])
        bw[g, :u] = wide[g][uniq[g, :u]]
        bd[g, :u] = deep[g][uniq[g, :u]]
    return bw, bd


def check_model(model, world, rank, local, dev, n_sm):
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, synthetic_batch

    ref_fn, R = _reference(model)
    group = PSGroup(world, *ADAM, device=local, local_shards=[rank])
    eng = DeepFMPSEngine(group, B, group_rows=ROWS, model=model)
    assert eng.exchange == "owner" and eng.row_source == "pull" and eng.tower_kind == "tile", (
        eng.exchange, eng.row_source, eng.tower_kind)
    G = eng.G
    ids, dense, labels = synthetic_batch(B, 60 + rank, dev, "zipf", group_rows=ROWS)
    wide0, deep0 = _initial_rows(eng, dev)
    params0 = eng.flat_params.clone()
    inv, n_unique, uniq = R.first_occurrence_inverse(ids)
    bw, bd = _gather_rows(wide0, deep0, uniq, n_unique, G)
    gen = torch.Generator(device=dev).manual_seed(90 + rank)
    for _ in range(40):
        near = R.near_relu_kink(ref_fn(inv, n_unique, bw, bd, dense, labels, params0))
        if not bool(near.any()):
            break
        dense[near] = torch.randn((int(near.sum()), R.ND), generator=gen, device=dev)
    else:
        raise AssertionError("conditioning did not converge")
    snap = {}

    def after_tower():
        for k in ("bet_w", "bet_d", "inv", "n_unique", "uniq", "flat_params", "loss_buf", "logits_buf", "flat_grads",
                  "gsum_w", "gsum_d"):
            snap[k] = getattr(eng, k).clone()

    torch.cuda.synchronize(dev)  # this rank's rows and dense parameters are set before any peer reads them
    dist.barrier()
    l0 = float(eng.step(ids, dense, labels, after_tower=after_tower))
    torch.cuda.synchronize(dev)
    group.check()
    # the exchange pulled the initial rows of this rank's unique ids (in the engine's own dedup order)
    s_inv, s_nu, s_uniq = snap["inv"].view(G, B), snap["n_unique"], snap["uniq"].view(G, B)
    bw, bd = _gather_rows(wide0, deep0, s_uniq, s_nu, G)
    got_w, got_d = snap["bet_w"].view(G, B), snap["bet_d"].view(G, B, 8)
    for g in range(G):
        u = int(s_nu[g])
        assert torch.equal(got_w[g, :u], bw[g, :u]) and torch.equal(got_d[g, :u], bd[g, :u]), (model, rank, g)
    assert torch.equal(snap["flat_params"], params0), (model, rank)
    ref = ref_fn(s_inv, s_nu, got_w, got_d, dense, labels, snap["flat_params"])
    got = {"loss": snap["loss_buf"], "logits": snap["logits_buf"], "grads": snap["flat_grads"],
           "gsum_wide": snap["gsum_w"].view(G, B), "gsum_deep": snap["gsum_d"].view(G, B, 8)}
    rs = R.check(got, ref, label="%s rank %d step 1" % (model, rank), n_sm=n_sm)
    for _ in range(20):
        l1 = float(eng.step(ids, dense, labels))
    group.check()
    assert np.isfinite(l0) and l1 < l0, (model, rank, l0, l1)
    eng.capture()
    for _ in range(5):
        l2 = float(eng.step_graph(ids, dense, labels))
    group.check()
    assert l2 < l1, (model, rank, l1, l2)
    dist.barrier()
    group.close()
    return l0, l1, l2, max(rs.values())


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    # B200_SHARED_GPU=1: every rank is a process on cuda:0 (see tests/mgpu_xchg_check.py)
    shared = os.environ.get("B200_SHARED_GPU") == "1"
    local = 0 if shared else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
    lines = []
    for model in ("wide_deep", "dcn"):
        l0, l1, l2, worst = check_model(model, world, rank, local, dev, n_sm)
        lines.append("%s loss %.4f -> %.4f -> %.4f (graph), step 1 worst err/bound %.3f" % (model, l0, l1, l2, worst))
    dist.barrier()
    print("rank %d: %s" % (rank, "; ".join(lines)))
    sys.stdout.flush()
    dist.barrier()
    if rank == 0:
        print("mgpu_models_check ok: world=%d" % world)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
