"""Time the pooled lookup of sparse input (Embedding with a combiner on a sparse [B, L] COO input): layer forward +
backward with a PSClient pull as the lookup, the kernel path against the torch composition it replaced (kept here as
the baseline).  B = 32768 rows, Poisson(10) ids per row (the reference's Frappe DeepFM has 10 ids per sample),
Zipf(1.05) over a 10^6-row table, 5 % negative ids, 1 % empty rows; dim 8 and 64, bounded and hashed tables.

    python tools/bench_sparse_lookup.py [--rounds 15] [--iters 20] [--profile]

Prints one JSON line per shape with the median and spread of alternating rounds, the largest output difference
of the two paths over the oracle's bound, and the card's name and power limit.  --profile lists the kernels of one
call of the kernel path instead."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

from elasticdl_b200 import ops  # noqa: E402
from elasticdl_b200.layers import Embedding  # noqa: E402
from elasticdl_b200.ps import PSGroup  # noqa: E402
from elasticdl_b200.worker.ps_client import PSClient  # noqa: E402
from oracle import sparse_oracle as so  # noqa: E402

ROWS = 10 ** 6


class TorchComposition(Embedding):
    """The torch composition of safe_embedding_lookup_sparse this path replaced (the baseline)."""

    def safe_embedding_lookup_sparse(self, sparse_ids, combiner="mean"):
        sp = sparse_ids.coalesce()
        rows = sp.indices()[0]
        vals = sp.values().to(torch.int64)
        batch = sp.shape[0]
        keep = vals >= 0
        rows, vals = rows[keep], vals[keep]
        counts = torch.bincount(rows, minlength=batch)
        is_row_empty = counts == 0
        empty_rows = torch.nonzero(is_row_empty).reshape(-1)
        if empty_rows.numel():
            rows = torch.cat([rows, empty_rows])
            vals = torch.cat([vals, torch.zeros_like(empty_rows)])
            order = torch.argsort(rows, stable=True)
            rows, vals = rows[order], vals[order]
            counts = torch.bincount(rows, minlength=batch)
        k = vals.numel()
        bet, inv = self._unique_and_pull(vals)
        per_id = ops.GatherRows.apply(bet, inv, 1, k, self.output_dim)
        out = torch.zeros((batch, self.output_dim), dtype=torch.float32, device=per_id.device)
        out = out.index_add(0, rows, per_id)
        if combiner == "mean":
            out = out / counts.clamp(min=1).to(out.dtype).unsqueeze(1)
        elif combiner == "sqrtn":
            out = out / counts.clamp(min=1).to(out.dtype).sqrt().unsqueeze(1)
        return torch.where(is_row_empty.unsqueeze(1), torch.zeros_like(out), out)


def make_input(B, seed=0):
    rng = np.random.default_rng(seed)
    lens = rng.poisson(10, B)
    lens[rng.random(B) < 0.01] = 0
    rows = np.repeat(np.arange(B), lens)
    vals = (rng.zipf(1.05, rows.size) - 1) % ROWS
    vals[rng.random(rows.size) < 0.05] = -1
    cols = np.concatenate([np.arange(n) for n in lens])
    sp = torch.sparse_coo_tensor(torch.tensor(np.stack([rows, cols])), torch.tensor(vals), (B, int(lens.max())))
    return sp.coalesce().cuda(), rows, vals


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:  # the numbers are still printed, without the card
        return "unknown (%s)" % e


def one_call(layer, sp, G):
    layer.set_tape(True)
    out = layer(sp)
    bet = layer.embedding_and_ids[0].batch_embedding
    (g,) = torch.autograd.grad(out, [bet], G)
    layer.reset()
    return out, g


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=15)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--B", type=int, default=32768)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_sparse_lookup needs a GPU")
    sp, rows, vals = make_input(a.B)
    name = card()
    for dim in (8, 64):
        for bounded in (True, False):
            group = PSGroup(1, "SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", device=0)
            group.register_table("bench/embeddings:0", dim, "uniform", capacity=ROWS if bounded else None,
                                 expected_rows=2 ** 21)
            group.commit()
            client = PSClient(group)
            paths = {}
            for kind, cls in (("kernels", Embedding), ("torch", TorchComposition)):
                layer = cls(dim, input_dim=ROWS if bounded else None, combiner="mean", name="bs_%s_%d_%d" % (kind, dim, bounded))
                layer.set_embedding_weight_name("bench/embeddings:0")
                layer.set_lookup_embedding_func(client.pull_embedding_vectors)
                paths[kind] = layer
            G = torch.randn(a.B, dim, device="cuda")
            outs = {k: one_call(l, sp, G) for k, l in paths.items()}  # creates the rows, warms every shape
            if a.profile:
                from torch.profiler import ProfilerActivity, profile

                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    one_call(paths["kernels"], sp, G)
                    torch.cuda.synchronize()
                names = [e.name for e in prof.events() if e.device_type.name == "CUDA"]
                print(json.dumps({"dim": dim, "bounded": bounded, "kernels": len(names), "list": names}))
                group.close()
                continue
            out_k, g_k = outs["kernels"]
            out_t, g_t = outs["torch"]
            # both paths lie within the oracle's per-row bound of the exact result, so within twice it of each other
            _, fids, _ = so.fill(rows, vals, a.B)
            uniq, _ = so.unique_first(fids)
            absrows = client.pull_embedding_vectors("bench/embeddings:0", torch.tensor(uniq).cuda()).abs()
            bd = 2 * so.bound(rows, vals, a.B, absrows.double().cpu().numpy(), "mean")
            err = (out_k - out_t).detach().abs().double().cpu().numpy()
            diff, agree = float(err.max()), bool((err <= bd).all())
            times = {k: [] for k in paths}
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            for r in range(a.rounds):
                for k in (("kernels", "torch") if r % 2 == 0 else ("torch", "kernels")):
                    torch.cuda.synchronize()
                    ev[0].record()
                    for _ in range(a.iters):
                        one_call(paths[k], sp, G)
                    ev[1].record()
                    torch.cuda.synchronize()
                    times[k].append(ev[0].elapsed_time(ev[1]) * 1000.0 / a.iters)
            res = {"dim": dim, "bounded": bounded, "B": a.B, "nnz": int(sp.values().numel()), "card": name,
                   "max_out_diff": diff, "agree_within_bound": agree}
            for k, t in times.items():
                res[k + "_us_median"] = round(float(np.median(t)), 1)
                res[k + "_us_spread"] = [round(float(np.min(t)), 1), round(float(np.max(t)), 1)]
            print(json.dumps(res))
            group.close()


if __name__ == "__main__":
    main()
