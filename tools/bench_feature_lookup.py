"""Time the string-vocabulary lookup and the fused feature transforms (csrc/feature_ids.cu) on the GPU.

    python tools/bench_feature_lookup.py [--legs lookup,census,dac_ctr] [--rounds 9] [--iters 20] [--root DIR]

Legs:
  lookup   IndexLookup's kernel (b200feat_index_lookup) at B = 2^20 strings of W = 16 bytes over V in {8, 10^4, 10^6,
           10^7} 16-byte terms, for all-hit, half-OOV and Zipf(1.05) inputs, against the torch composition a user
           would otherwise write: b200feat_fingerprint64, torch.searchsorted over the sorted term fingerprints, a row
           gather and compare, then torch.where.  The two outputs are compared.
  census   the fused census wide & deep transform (workloads/census_features.census_transform) at B in {64, 4096,
           65536, 2^20}.
  dac_ctr  the fused dac_ctr transform (workloads/dac_ctr_features.dac_ctr_transform) at B in {4096, 2^20}.  It uses
           only API that predates IndexLookup, so with --root pointing at an older checkout the same leg times that
           checkout's kernel.

Prints the card's name and power limit, then one JSON line per shape: the median and spread (min, max) of the
per-call time over rounds of `iters` calls timed with CUDA events, and GB/s from the bytes the shapes imply (string
and numeric bytes read, slots probed -- one 16-byte slot per lookup, plus the Wv-byte term row on a hit -- and ids
written) with their share of the 3.35 TB/s HBM3 data-sheet figure.  These kernels are bounded by bytes, not
operations, so that share is the roofline figure."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np


def _args():
    p = argparse.ArgumentParser()
    p.add_argument("--legs", default="lookup,census,dac_ctr")
    p.add_argument("--rounds", type=int, default=9)
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--root", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."),
                   help="checkout whose elasticdl_b200 package is imported")
    return p.parse_args()


a = _args()
sys.path.insert(0, os.path.abspath(a.root))

import ctypes  # noqa: E402

import torch  # noqa: E402

from elasticdl_b200 import _lib  # noqa: E402

HBM = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers are still printed, without the card
        return "unknown (%s)" % e


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(rc):
    if rc:
        raise RuntimeError(_lib.lib().b200feat_last_error().decode())


def time_calls(fns, rounds, iters):
    """{name: [per-call seconds per round]}, the callables alternating round by round after a warm-up."""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for f in fns.values():
        for _ in range(3):
            f()
    out = {k: [] for k in fns}
    names = list(fns)
    for r in range(rounds):
        for k in (names if r % 2 == 0 else names[::-1]):
            torch.cuda.synchronize()
            ev[0].record()
            for _ in range(iters):
                fns[k]()
            ev[1].record()
            torch.cuda.synchronize()
            out[k].append(ev[0].elapsed_time(ev[1]) / 1e3 / iters)
    return out


def stats(ts, nbytes):
    med = float(np.median(ts))
    return {"median_us": round(med * 1e6, 2), "min_us": round(min(ts) * 1e6, 2), "max_us": round(max(ts) * 1e6, 2),
            "GBps": round(nbytes / med / 1e9, 1), "hbm_share": round(nbytes / med / HBM, 4)}


def hex_rows(vals, upper=False):
    """uint64 values -> uint8 [n, 16] of their 16 hex digits (distinct values give distinct rows)."""
    digits = np.frombuffer(b"0123456789ABCDEF" if upper else b"0123456789abcdef", dtype=np.uint8)
    shifts = np.arange(60, -4, -4, dtype=np.uint64)
    return digits[((vals[:, None] >> shifts) & np.uint64(15)).astype(np.int64)]


def leg_lookup(rounds, iters):
    lib = _lib.lib()
    B, W = 1 << 20, 16
    rng = np.random.RandomState(0)
    for V in (8, 10 ** 4, 10 ** 6, 10 ** 7):
        vals = (np.arange(V, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        terms = np.ascontiguousarray(hex_rows(vals))
        n_slots = lib.b200feat_vocab_slots(V)
        slots = np.zeros(n_slots * 2, dtype=np.int64)
        check(lib.b200feat_vocab_build(terms.ctypes.data, V, W, n_slots, slots.ctypes.data, None))
        slots_d, terms_d = torch.from_numpy(slots).cuda(), torch.from_numpy(terms).cuda()
        # the torch composition's table: sorted term fingerprints and their vocabulary positions
        tfp = torch.empty(V, dtype=torch.int64, device="cuda")
        check(lib.b200feat_fingerprint64(terms_d.data_ptr(), W, V, tfp.data_ptr(), stream()))
        sorted_fp, order = torch.sort(tfp)
        for kind in ("all_hit", "half_oov", "zipf"):
            if kind == "zipf":
                u = rng.rand(B)
                s = 1.05
                idx = np.minimum(np.floor(((V ** (1 - s) - 1.0) * u + 1.0) ** (1.0 / (1 - s))).astype(np.int64) - 1,
                                 V - 1)
                idx = rng.permutation(V)[idx]
            else:
                idx = rng.randint(V, size=B)
            x = terms[idx].copy()
            if kind == "half_oov":
                miss = rng.rand(B) < 0.5
                x[miss] = hex_rows(rng.randint(0, 1 << 62, miss.sum()).astype(np.uint64), upper=True)
                x[miss, 0] = ord("Z")  # never a lower-case hex term
            xd = torch.from_numpy(x).cuda()
            out = torch.empty(B, dtype=torch.int64, device="cuda")
            fp = torch.empty(B, dtype=torch.int64, device="cuda")

            def kernel():
                check(lib.b200feat_index_lookup(xd.data_ptr(), W, B, slots_d.data_ptr(), terms_d.data_ptr(), n_slots,
                                                V, W, 1, out.data_ptr(), stream()))

            def composition():
                check(lib.b200feat_fingerprint64(xd.data_ptr(), W, B, fp.data_ptr(), stream()))
                pos = torch.searchsorted(sorted_fp, fp).clamp_(max=V - 1)
                cand = order[pos]
                hit = (sorted_fp[pos] == fp) & (terms_d[cand] == xd).all(1)
                return torch.where(hit, cand, torch.full_like(cand, V))  # one OOV bucket: V + fp % 1

            kernel()
            ref = composition()
            torch.cuda.synchronize()
            same = bool(torch.equal(out, ref))
            hits = int((ref < V).sum())
            nbytes = B * W + B * 16 + hits * W + B * 8
            ts = time_calls({"kernel": kernel, "torch": composition}, rounds, iters)
            print(json.dumps({"leg": "index_lookup", "V": V, "inputs": kind, "B": B, "W": W, "hits": hits,
                              "outputs_equal": same, "kernel": stats(ts["kernel"], nbytes),
                              "torch_composition": stats(ts["torch"], nbytes),
                              "speedup": round(float(np.median(ts["torch"]) / np.median(ts["kernel"])), 2)}), flush=True)
            assert same, "kernel and torch composition disagree"


def leg_census(rounds, iters):
    from elasticdl_b200.workloads import census_features as C

    for ids_dtype in (torch.int32,):
        ft = C.census_transform(ids_dtype)
        for B in (64, 4096, 65536, 1 << 20):
            num, strings, _, _ = C.synthetic_raw_batch(B, 0, "cuda")
            ids = torch.empty((12, B), dtype=ids_dtype, device="cuda")
            nbytes = B * 4 * 4 + B * 8 * C.STRING_WIDTH + B * 5 * 16 + B * 12 * ids.element_size()
            ts = time_calls({"t": lambda: ft(num, strings, ids_out=ids)}, rounds, iters)
            print(json.dumps({"leg": "census_transform", "B": B, "ids": str(ids_dtype), **stats(ts["t"], nbytes)}),
                  flush=True)


def leg_dac_ctr(rounds, iters):
    from elasticdl_b200.workloads.dac_ctr_features import dac_ctr_transform, synthetic_raw_batch

    for ids_dtype in (torch.int32,):
        ft = dac_ctr_transform(ids_dtype)
        for B in (4096, 1 << 20):
            numeric, strings, _ = synthetic_raw_batch(B, 0, "cuda")
            ids = torch.empty((38, B), dtype=ids_dtype, device="cuda")
            dense = torch.empty((B, 13), dtype=torch.float32, device="cuda")
            nbytes = B * 13 * 8 + B * 26 * 8 + B * 38 * ids.element_size() + B * 13 * 4
            ts = time_calls({"t": lambda: ft(numeric, strings, ids_out=ids, dense_out=dense)}, rounds, iters)
            print(json.dumps({"leg": "dac_ctr_transform", "root": os.path.abspath(a.root), "B": B,
                              "ids": str(ids_dtype), **stats(ts["t"], nbytes)}), flush=True)


def main():
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: these are GPU timings")
    print(json.dumps({"card": card(), "device": torch.cuda.get_device_name()}), flush=True)
    for leg in a.legs.split(","):
        {"lookup": leg_lookup, "census": leg_census, "dac_ctr": leg_dac_ctr}[leg](a.rounds, a.iters)


if __name__ == "__main__":
    main()
