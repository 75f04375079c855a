"""Time the weighted pooled lookup of an EmbeddingBag (mode "sum", per_sample_weights): combine forward + backward
(the BET gradient and the weight gradient) through ops.SparseCombine, against torch's own
F.embedding_bag(inv, bet, offsets, "sum", per_sample_weights=w) over the same pulled rows, alternating.
B = 32768 bags, Poisson(10) ids per bag (the reference's Frappe DeepFM has 10 ids per sample), Zipf(1.05) over a
10^6-row table; dim 8 and 64.  Prep, dedup and pull run once, outside the timed window: both paths start from the same
[U, dim] rows.

    python tools/bench_weighted_lookup.py [--rounds 15] [--iters 20]

Prints one JSON line per dim with the median and spread of alternating rounds, the largest output and gradient
differences of the two paths, and the card's name and power limit."""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from elasticdl_b200 import ops  # noqa: E402
from elasticdl_b200.ps import PSGroup  # noqa: E402
from tools.bench_sparse_lookup import ROWS, card  # noqa: E402


def make_bags(B, seed=0):
    rng = np.random.default_rng(seed)
    lens = rng.poisson(10, B)
    ids = (rng.zipf(1.05, int(lens.sum())) - 1) % ROWS
    offsets = np.concatenate([[0], np.cumsum(lens)[:-1]])
    w = rng.uniform(0.0, 2.0, ids.size).astype(np.float32)
    return torch.tensor(ids).cuda(), torch.tensor(offsets).cuda(), torch.tensor(w).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--B", type=int, default=32768)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_weighted_lookup needs a GPU")
    ids, offsets, w = make_bags(a.B)
    name = card()
    group = PSGroup(1, "SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", device=0)
    for dim in (8, 64):
        fids, ws, batch, nnz = ops.bag_prep(group, ids, offsets, dim)
        uniq, inv, n = ops.unique(fids)
        u = uniq[: int(n.item())]
        group.check()
        bet = torch.randn(u.numel(), dim, device="cuda").requires_grad_(True)
        order = torch.argsort(u)
        inv_in = order[torch.searchsorted(u[order], ids)]  # each input entry's row of bet, for torch
        wl = w.clone().requires_grad_(True)
        G = torch.randn(batch, dim, device="cuda")

        def kernels():
            out = ops.SparseCombine.apply(bet, inv, ws, batch, nnz, "sum", dim, wl)
            return (out,) + torch.autograd.grad(out, [bet, wl], G)

        def torch_path():
            out = F.embedding_bag(inv_in, bet, offsets, mode="sum", per_sample_weights=wl)
            return (out,) + torch.autograd.grad(out, [bet, wl], G)

        paths = {"kernels": kernels, "torch": torch_path}
        res_k, res_t = kernels(), torch_path()  # warms every shape
        diffs = [float((x - y).detach().abs().max()) for x, y in zip(res_k, res_t)]
        times = {k: [] for k in paths}
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        for r in range(a.rounds):
            for k in (("kernels", "torch") if r % 2 == 0 else ("torch", "kernels")):
                torch.cuda.synchronize()
                ev[0].record()
                for _ in range(a.iters):
                    paths[k]()
                ev[1].record()
                torch.cuda.synchronize()
                times[k].append(ev[0].elapsed_time(ev[1]) * 1000.0 / a.iters)
        res = {"dim": dim, "B": a.B, "nnz": nnz, "n_unique": int(u.numel()), "card": name,
               "max_out_diff": diffs[0], "max_gbet_diff": diffs[1], "max_gw_diff": diffs[2]}
        for k, t in times.items():
            res[k + "_us_median"] = round(float(np.median(t)), 1)
            res[k + "_us_spread"] = [round(float(np.min(t)), 1), round(float(np.max(t)), 1)]
        print(json.dumps(res))
    group.close()


if __name__ == "__main__":
    main()
