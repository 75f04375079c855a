"""The oracle against the reference's OWN compiled kernels (oracle/_ref) and against the vectors they produced.

* tests/golden/ref_kernel_vectors.npz was written by RUNNING the reference's kernel_api.cc (compiled unmodified,
  oracle/Makefile `ref`) -- tests/golden/gen_kernel_vectors.py.  The C restatement (ps_oracle.c) and its numpy twin
  must reproduce every output bit for bit.  Runs anywhere (the fixture is committed).
* tests/golden/ref_kernel_live.json (gen_kernel_vectors.py `live`) holds digests of what the reference kernels
  returned on further seeded inputs, the outputs of kernel_test.go's own vectors and of the bench's CPU arm with the
  reference's Adam as its row update; the oracle is held to those here, without the reference present.
Bar: bit-exact (integer compare of the fp32 patterns).
"""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import gen_kernel_vectors as G  # noqa: E402
from oracle import ps_oracle as O  # noqa: E402

F = np.float32
VEC = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_kernel_vectors.npz"))
with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_kernel_live.json")) as _f:
    LIVE = json.load(_f)


def bits(a):
    return np.ascontiguousarray(a, dtype=F).view(np.uint32)


def run_oracle_c(kind, hp, g3, p, s0, s1, s2):
    for k in range(3):
        g = np.ascontiguousarray(g3[k])
        if kind == "sgd":
            O.lib.oracle_sgd(O._f32(g), O._f32(p), hp["lr"], p.size)
        elif kind == "momentum":
            O.lib.oracle_momentum(O._f32(g), O._f32(p), O._f32(s0), hp["mu"], hp["nesterov"], hp["lr"], p.size)
        elif kind == "adam":
            O.lib.oracle_adam(O._f32(g), O._f32(p), O._f32(s0), O._f32(s1), hp["lr"], p.size, hp["step"] + k,
                              hp["beta1"], hp["beta2"], hp["eps"], O._f32(s2) if hp["ams"] else O._null_f32())
        elif kind == "adagrad":
            O.lib.oracle_adagrad(O._f32(g), O._f32(p), O._f32(s0), hp["lr"], p.size, hp["eps"])


def run_oracle_np(kind, hp, g3, p, s0, s1, s2):
    for k in range(3):
        g = g3[k]
        if kind == "sgd":
            O.np_sgd(g, p, hp["lr"])
        elif kind == "momentum":
            O.np_momentum(g, p, s0, hp["mu"], hp["nesterov"], hp["lr"])
        elif kind == "adam":
            O.np_adam(g, p, s0, s1, hp["lr"], hp["step"] + k, hp["beta1"], hp["beta2"], hp["eps"],
                      s2 if hp["ams"] else None)
        elif kind == "adagrad":
            O.np_adagrad(g, p, s0, hp["lr"], hp["eps"])


CASES = {name: (kind, hp, n) for name, kind, hp, n in G.cases()}


def test_fixture_lists_the_generator_cases():
    assert list(VEC["names"]) == [c[0] for c in G.cases()]


@pytest.mark.parametrize("runner", [run_oracle_c, run_oracle_np], ids=["c", "numpy"])
@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_reference_kernel_vectors(name, runner):
    kind, hp, n = CASES[name]
    st = {k: VEC[name + "/in_" + k].copy() for k in ("p", "s0", "s1", "s2")}
    runner(kind, hp, VEC[name + "/g"], st["p"], st["s0"], st["s1"], st["s2"])
    for k in ("p", "s0", "s1", "s2"):
        assert np.array_equal(bits(st[k]), bits(VEC[name + "/out_" + k])), (name, k)


@pytest.mark.parametrize("seed", G.LIVE_SEEDS)
def test_oracle_equals_ref_live(seed):
    """Fresh random inputs each seed, sizes that exercise the SSE body and the scalar tail."""
    want = LIVE["equals_ref_live"][str(seed)]
    for name, kind, hp, g3, base in G.live_cases(seed):
        b = [x.copy() for x in base]
        run_oracle_c(kind, hp, g3, *b)
        assert G.digest(b) == want[name], (name, base[0].size)


def test_ref_replays_kernel_test_go_vectors():
    """elasticdl/go/pkg/kernel/kernel_test.go:25-47 (SGD, exact) and :69-107 (Adam step 5, expected
    values written with the Go-side formula, compared there with tolerance 1e-4... we keep 1e-6), on what the
    reference kernels returned for them; the oracle returns the same bits."""
    ref = {k: np.array(v, dtype=np.uint32).view(F) for k, v in LIVE["kernel_test_go"].items()}
    g = np.arange(10, dtype=F) * F(0.5) + F(0.25)
    p = np.arange(10, dtype=F) * F(-0.3) + F(1.0)
    want = p - F(0.1) * g
    assert np.array_equal(bits(ref["sgd_p"]), bits(want))
    O.lib.oracle_sgd(O._f32(g), O._f32(p), 0.1, p.size)
    assert np.array_equal(bits(p), bits(ref["sgd_p"]))
    rng = np.random.default_rng(3)
    g, p0, m0, v0 = [rng.random(10).astype(F) for _ in range(4)]
    p, m, v = ref["adam_p"], ref["adam_m"], ref["adam_v"]
    em = 0.9 * m0.astype(np.float64) + 0.1 * g
    ev = 0.999 * v0.astype(np.float64) + 0.001 * g.astype(np.float64) ** 2
    ep = p0 - 0.1 * np.sqrt(1 - 0.999 ** 5) / (1 - 0.9 ** 5) * em / (np.sqrt(ev) + 1e-8)
    assert np.allclose(m, em, rtol=1e-6) and np.allclose(v, ev, rtol=1e-6) and np.allclose(p, ep, rtol=1e-5, atol=1e-6)
    po, mo, vo = p0.copy(), m0.copy(), v0.copy()
    O.lib.oracle_adam(O._f32(g), O._f32(po), O._f32(mo), O._f32(vo), 0.1, po.size, 5, 0.9, 0.999, 1e-8, O._null_f32())
    for x, y in ((po, p), (mo, m), (vo, v)):
        assert np.array_equal(bits(x), bits(y))


@pytest.mark.parametrize("dim", [1, 8])
def test_sparse_adam_rows_through_the_reference_kernel(dim):
    """The CPU arm of bench.py updates table rows with the reference's own compiled Adam (one call per row, as
    kernel.go:119-138 does through cgo): the oracle's own row update leaves the tables bit-identical to what that
    hook produced, duplicates applied sequentially, AMSGrad slot included."""
    assert G.digest(G.sparse_adam_tables(dim, None)) == LIVE["sparse_adam"][str(dim)]
