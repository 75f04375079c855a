"""Edge tests of the drop-in trainer path's client-side primitives: the dedup (k_unique / k_unique_small behind
b200ps_unique*, ops.unique, PSGroup.unique), the row gather (k_gather_rows) and the gradient segment sum
(k_segment_sum) behind b200ps_gather_rows / b200ps_segment_sum, ops.gather_rows / ops.segment_sum and
ops.GatherRows, and the trainer's batched lookups past 96 layers of one (k, dim).

Dedup results are compared exactly with oracle.ps_oracle.unique_first_occurrence per segment: uniq[:n], the whole
inverse index and n_unique.  Gathers are compared bit for bit.  Segment sums are compared with the float64 sum per
(row, column): a row that one or two values land on equals float32(a + b) exactly (the zeroed output plus one or
two float adds gives that in any order), a row of multiplicity m >= 3 lies within the recursive-summation bound
(m - 1) 2^-24 sum|x| of it whatever order the atomics take, and a row that no id maps to is exactly +0.

Shapes come from the device's SM count the way the launches size their grids.  The dedup's co-resident grid has at
most 4 blocks per SM (1 with blocks_per_sm = 1), so segment counts around 4 x SMs make the blocks walk the run slots
of more than 96 segments (the equal-runs layout).  The gather and the segment sum cap their grid at 16 blocks of 256
threads per SM of the handle (132 SMs without one), so k x chunks around one such pass makes the grid-stride loops
take a second and a fourth pass.  Every output is carved from a larger buffer filled with a sentinel (-7 for ids,
NaN for floats), so a skipped element or a write past the end shows.
"""
import ctypes
import types

import numpy as np
import pytest
import torch

from oracle import ps_oracle as O

pytestmark = pytest.mark.gpu

F32 = np.float32
TINY = float(np.finfo(F32).tiny)  # 2^-126, the smallest normal float32
SENT = -7
GUARD = 1031  # sentinel elements after every output
NULL_SMS = 132  # grid_for() without a handle
SGD = ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;")
ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")


def _lib():
    from elasticdl_b200 import _lib as L

    return L.lib()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _err():
    return _lib().b200ps_last_error().decode()


def _n_sm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


@pytest.fixture(scope="module")
def group():
    from elasticdl_b200.ps import PSGroup

    g = PSGroup(1, *SGD, device=0)
    yield g
    g.close()


# ================================================================================================== dedup
def _n_segs(name):
    s = _n_sm()
    return {"4sm-1": 4 * s - 1, "4sm+1": 4 * s + 1, "8sm+3": 8 * s + 3}.get(name) or int(name)


def _seg_ids(rng, T, k):
    """[T, k] int64.  Segment t draws from a range that cycles through one id, 7 ids, about k / 2, 10 k and 2^40
    (a third of those negative: an unbounded segment takes any int64)."""
    his = np.array([1, 7, max(k // 2, 1), 10 * k, 1 << 40], dtype=np.float64)
    hi = his[np.arange(T) % 5][:, None]
    ids = (rng.random_sample((T, k)) * hi).astype(np.int64)
    neg = (np.arange(T) % 5 == 4)[:, None] & (rng.random_sample((T, k)) < 0.3)
    return np.where(neg, -ids - 1, ids)


def _want_unique(ids):
    """Per-segment oracle: uniq padded with the sentinel past n_unique (the kernels never write there), inv, n."""
    T, k = ids.shape
    uniq = np.full((T, k), SENT, dtype=np.int64)
    inv = np.empty((T, k), dtype=np.int32)
    n = np.empty(T, dtype=np.int32)
    for t in range(T):
        u, i = O.unique_first_occurrence(ids[t])
        uniq[t, : len(u)], inv[t], n[t] = u, i, len(u)
    return uniq, inv, n


def _unique_outs(T, k):
    return (torch.full((T * k + GUARD,), SENT, dtype=torch.int64, device="cuda"),
            torch.full((T * k + GUARD,), SENT, dtype=torch.int32, device="cuda"),
            torch.full((T + GUARD,), SENT, dtype=torch.int32, device="cuda"))


def _read_unique(outs, T, k):
    ub, ib, nb = outs
    torch.cuda.synchronize()
    assert (ub[T * k:] == SENT).all() and (ib[T * k:] == SENT).all() and (nb[T:] == SENT).all(), "written past the end"
    return ub[: T * k].view(T, k).cpu().numpy(), ib[: T * k].view(T, k).cpu().numpy(), nb[:T].cpu().numpy()


def _compare_unique(got, want, what):
    for name, g, w in zip(("uniq", "inv", "n_unique"), got, want):
        bad = np.argwhere(g != w)
        assert bad.size == 0, "%s: first wrong %s at %s: %d != %d (%d wrong)" % (
            what, name, tuple(bad[0]), g[tuple(bad[0])], w[tuple(bad[0])], len(bad))


def _masked(uniq, n):
    """uniq of an entry point that allocates its own outputs: the sentinel past n_unique, as _want_unique has it."""
    u = uniq.copy()
    u[np.arange(u.shape[1])[None, :] >= n[:, None]] = SENT
    return u


_WS = {}  # one workspace per entry point, reused dirty from call to call and from shape to shape


def _ws(path, need):
    ws = _WS.get(path)
    if ws is None or ws.numel() < need:
        ws = _WS[path] = torch.zeros(need, dtype=torch.uint8, device="cuda")
    return ws


UNIQUE_PATHS = ["ops", "handle", "handle_bps1", "null_bps1"]


def _run_unique(path, group, d_ids, T, k):
    """One dedup of the [T * k] int64 ids through `path`; returns (uniq, inv, n_unique) as [T, k], [T, k], [T]."""
    from elasticdl_b200 import ops

    lib = _lib()
    if path == "ops":  # ps = NULL, blocks_per_sm 0, ops' own workspace
        u, i, n = ops.unique(d_ids, T)
        torch.cuda.synchronize()
        n = n.cpu().numpy()
        return _masked(u.view(T, k).cpu().numpy(), n), i.view(T, k).cpu().numpy(), n
    outs = _unique_outs(T, k)
    ws = _ws(path, lib.b200ps_unique_workspace(T, k))
    ptrs = (outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), ws.data_ptr(), ws.numel())
    if path == "handle":
        rc = lib.b200ps_unique(group._h, d_ids.data_ptr(), T, k, *ptrs, _stream())
    else:  # one block per SM: run slots outnumber the blocks already at moderate T
        h = group._h if path == "handle_bps1" else None
        rc = lib.b200ps_unique_bounded_ex(h, d_ids.data_ptr(), 0, T, k, None, *ptrs, 1, _stream())
    assert rc == 0, _err()
    return _read_unique(outs, T, k)


# 51 units of 1024 positions, the last one partial.  At 97 segments the full grid takes runs of 12 to 27 units (by
# the occupancy), so the last run of every segment is short; with one block per SM one run takes all 51
RAGGED_K = 51 * 1024 + 7
K_VALUES = [1, 33, 1024, 1025, 5000]
T_NAMES = ["95", "96", "97", "200", "4sm-1", "4sm+1", "8sm+3"]
UNIQUE_CASES = [(t, k) for t in T_NAMES for k in K_VALUES] + [("65535", 1), ("97", RAGGED_K)]


@pytest.mark.parametrize("segs,k", UNIQUE_CASES, ids=["T%s-k%d" % c for c in UNIQUE_CASES])
def test_unique_segment_counts_past_96_and_the_resident_grid(group, segs, k):
    """T segments of k ids through ops.unique (no handle), b200ps_unique and b200ps_unique_bounded_ex with one
    block per SM (with and without a handle), twice on the same dirty workspaces with fresh ids."""
    T = _n_segs(segs)
    rng = np.random.RandomState(T * 7 + k)
    for rep in range(2):
        ids = _seg_ids(rng, T, k)
        want = _want_unique(ids)
        d_ids = torch.from_numpy(ids).cuda().view(-1)
        for path in UNIQUE_PATHS:
            _compare_unique(_run_unique(path, group, d_ids, T, k), want, "%s, call %d" % (path, rep))
    group.check()


def test_unique_refuses_65536_segments_and_launches_nothing(group):
    from elasticdl_b200 import ops

    lib = _lib()
    T, k = 65536, 1
    d_ids = torch.arange(T, dtype=torch.int64, device="cuda")
    ws = _ws("refusal", lib.b200ps_unique_workspace(T, k))
    for h in (group._h, None):
        for fn in ("unique", "ex"):
            outs = _unique_outs(T, k)
            before = lib.b200ps_launch_count(h)
            ptrs = (outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), ws.data_ptr(), ws.numel())
            if fn == "unique":
                rc = lib.b200ps_unique(h, d_ids.data_ptr(), T, k, *ptrs, _stream())
            else:
                rc = lib.b200ps_unique_bounded_ex(h, d_ids.data_ptr(), 0, T, k, None, *ptrs, 0, _stream())
            assert rc == -1 and "bad unique shape" in _err(), (rc, _err())
            torch.cuda.synchronize()
            assert lib.b200ps_launch_count(h) == before
            assert all((o == SENT).all() for o in outs)
    with pytest.raises(ValueError, match="bad unique shape"):
        ops.unique(d_ids, T)


@pytest.mark.parametrize("T", [97, 200])
def test_unique_bounds_past_96_segments_give_the_unbounded_result(group, T):
    """PSGroup.unique drops the bounds past 96 segments and b200ps_unique_bounded ignores them (no direct-address
    arrays in the workspace): the results equal the unbounded dedup and the oracle, over dirty workspaces."""
    lib = _lib()
    k = 1025
    bounds = [(t % 7 + 1) * 50 for t in range(T)]
    arr = (ctypes.c_int64 * T)(*bounds)
    assert lib.b200ps_unique_bounded_workspace(T, k, arr) == lib.b200ps_unique_workspace(T, k)
    rng = np.random.RandomState(T)
    ws = _ws("bounded", lib.b200ps_unique_workspace(T, k))
    for rep in range(2):
        ids = np.stack([rng.randint(0, b, size=k) for b in bounds]).astype(np.int64)
        want = _want_unique(ids)
        d_ids = torch.from_numpy(ids).cuda().view(-1)
        for with_bounds in (True, False):
            u, i, n = group.unique(d_ids, T, bounds=bounds if with_bounds else None)
            n = n.cpu().numpy()
            got = (_masked(u.view(T, k).cpu().numpy(), n), i.view(T, k).cpu().numpy(), n)
            _compare_unique(got, want, "PSGroup.unique bounds=%s, call %d" % (with_bounds, rep))
        outs = _unique_outs(T, k)
        assert lib.b200ps_unique_bounded(group._h, d_ids.data_ptr(), T, k, arr, outs[0].data_ptr(), outs[1].data_ptr(),
                                         outs[2].data_ptr(), ws.data_ptr(), ws.numel(), _stream()) == 0, _err()
        _compare_unique(_read_unique(outs, T, k), want, "b200ps_unique_bounded, call %d" % rep)
    group.check()


# direct segments with a tiny, a 2^14 (shared-memory sized) and a 2^20 range, one of 3e6 ids (sparse: no probe),
# an unknown range and one past 2^30 (both hashed)
TAG_BOUNDS = [5, 16384, 0, 3_000_000, (1 << 30) + 1, 1 << 20]


def _bounded_call(group, path, ws, k, rng):
    """One bounded dedup of fresh ids over TAG_BOUNDS through `path` on `ws`, compared with the oracle."""
    lib = _lib()
    T = len(TAG_BOUNDS)
    arr = (ctypes.c_int64 * T)(*TAG_BOUNDS)
    assert ws.numel() == lib.b200ps_unique_bounded_workspace(T, k, arr) > lib.b200ps_unique_workspace(T, k)
    ids = np.stack([rng.randint(0, b, size=k) if 0 < b <= (1 << 30) else
                    rng.randint(-(1 << 40), 1 << 40, size=k) if b else rng.randint(0, 5000, size=k)
                    for b in TAG_BOUNDS]).astype(np.int64)
    want = _want_unique(ids)
    d_ids = torch.from_numpy(ids).cuda().view(-1)
    outs = _unique_outs(T, k)
    ptrs = (outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), ws.data_ptr(), ws.numel())
    if path == "bounded":
        rc = lib.b200ps_unique_bounded(group._h, d_ids.data_ptr(), T, k, arr, *ptrs, _stream())
    else:
        h = group._h if path == "ex" else None
        rc = lib.b200ps_unique_bounded_ex(h, d_ids.data_ptr(), 0, T, k, arr, *ptrs, 1, _stream())
    assert rc == 0, _err()
    _compare_unique(_read_unique(outs, T, k), want, path)
    group.check()


def _bounded_ws(k, fill):
    T = len(TAG_BOUNDS)
    need = _lib().b200ps_unique_bounded_workspace(T, k, (ctypes.c_int64 * T)(*TAG_BOUNDS))
    if fill == "zeros":
        return torch.zeros(need, dtype=torch.uint8, device="cuda")
    return torch.randint(0, 256, (need,), dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("k", [1 << 20, (1 << 20) + 1], ids=["tagged", "untagged"])
def test_unique_bounded_past_the_position_tag(group, k):
    """The direct-address position arrays carry an epoch tag while k <= 2^20 and are cleared on every call past it:
    three calls with different ids on one workspace (stale positions of the previous call would win the atomicMin),
    through b200ps_unique_bounded and b200ps_unique_bounded_ex (one block per SM, with and without a handle)."""
    rng = np.random.RandomState(k % 1000)
    ws = _bounded_ws(k, "zeros")
    for path in ("bounded", "ex", "ex_null"):
        _bounded_call(group, path, ws, k, rng)


@pytest.mark.parametrize("k", [1 << 20, (1 << 20) + 1], ids=["tagged", "untagged"])
def test_unique_bounded_on_a_workspace_of_random_bytes(group, k):
    rng = np.random.RandomState(k % 1000 + 1)
    ws = _bounded_ws(k, "random")
    _bounded_call(group, "ex", ws, k, rng)


# ================================================================================= gather and segment sum
DIMS = [1, 2, 3, 4, 5, 7, 8, 12, 16, 24, 64, 100, 128]
PATTERNS = ["distinct", "pairs_near", "pairs_far", "hot", "zipf", "scattered", "low"]
WORKS = ["pass-1", "pass", "pass+1", "3pass+17"]


def _chunk_width(dim, aligned):
    """Floats per work item of the vector class b200ps picks (dim_class): 8, 4, or 1 for any unaligned pointer."""
    if not aligned:
        return 1
    return 8 if dim % 8 == 0 else 4 if dim % 4 == 0 else 1


def _pass_items(handle):
    return 16 * (_n_sm() if handle else NULL_SMS) * 256


def _k_for(work, p, chunks):
    """Rows per segment so that k * chunks is just below, at, just past one pass of p work items, or past three."""
    return {"pass-1": (p - 1) // chunks, "pass": p // chunks, "pass+1": -(-(p + 1) // chunks),
            "3pass+17": -(-(3 * p + 17) // chunks)}[work]


def _inv_pattern(name, k, rng):
    """Inverse index of one segment of k rows, into [0, k) like a dedup's."""
    i = np.arange(k)
    if name == "distinct":
        v = rng.permutation(k)
    elif name == "pairs_near":  # every id twice, on neighbouring rows (one warp)
        v = i // 2
    elif name == "pairs_far":  # every id twice, half a segment apart (different warps)
        v = i % ((k + 1) // 2)
    elif name == "hot":  # one id for every row
        v = np.zeros(k, dtype=np.int64)
    elif name == "zipf":
        v = (rng.zipf(1.3, size=k) - 1) % k
    elif name == "scattered":  # lanes l, l + 7, l + 14, ... of each 32 rows share an id
        v = np.minimum((i // 32) * 7 + (i % 32) * 5 % 7, k - 1)
    else:  # "low": ids below k / 3 only, the rows past them are never targeted
        v = rng.randint(0, max(k // 3, 1), size=k)
    return v.astype(np.int32)


def _float_buf(n, offset):
    """(whole NaN buffer, the n floats starting `offset` floats in)."""
    buf = torch.full((offset + n + GUARD,), float("nan"), dtype=torch.float32, device="cuda")
    return buf, buf[offset: offset + n]


def _untouched(buf, offset, n):
    return bool(torch.isnan(buf[:offset]).all()) and bool(torch.isnan(buf[offset + n:]).all())


def _check_gather(got, bet, dst, what):
    """got [T * k, dim] == bet[dst] bit for bit (dst: global row of every output row)."""
    want = bet[dst]
    bad = np.argwhere(got.view(np.int32) != want.view(np.int32))
    assert bad.size == 0, "%s: first wrong gathered float at %s: %r != %r" % (what, tuple(bad[0]), got[tuple(bad[0])],
                                                                              want[tuple(bad[0])])


def _sum_refs(vals, dst, rows):
    """float64 sum, float64 sum of |x|, float32 sum (exact for one or two addends), multiplicity per output row, and
    where a subnormal addend lands."""
    v = torch.from_numpy(vals)
    d = torch.from_numpy(dst.astype(np.int64))
    z64 = torch.zeros((rows, v.shape[1]), dtype=torch.float64)
    s64 = z64.clone().index_add_(0, d, v.double())
    a64 = z64.index_add_(0, d, v.abs().double())
    s32 = torch.zeros((rows, v.shape[1]), dtype=torch.float32).index_add_(0, d, v)
    sub = (vals != 0) & (np.abs(vals) < TINY)
    has_sub = np.zeros(s32.shape, dtype=bool)
    if sub.any():
        has_sub = torch.zeros(s32.shape, dtype=torch.int32).index_add_(0, d, torch.from_numpy(sub.astype(np.int32)))
        has_sub = has_sub.numpy() > 0
    return s64.numpy(), a64.numpy(), s32.numpy(), np.bincount(dst, minlength=rows), has_sub


def _check_sum(got, refs, what):
    """Rows nobody targets: +0.  One or two addends: float32(a + b) exactly.  m >= 3: within (m - 1) 2^-24 sum|x| of
    the float64 sum (plus the float64 sum's own rounding).  NaN and inf exactly where the float64 sum has them.

    DIVERGENCE: the float reductions to global memory flush subnormal addends and results to zero on sm_90 (the
    scalar one is REDG.E.ADD.F32.FTZ.RN in SASS; the 128-bit one does the same).  A lone subnormal addend therefore
    sums to 0, and a sum that involves a subnormal addend or result is within 2^-126 per addend and per add
    (2 m 2^-126 in all) of the float64 sum instead of bit exact."""
    s64, a64, s32, m, has_sub = refs
    none = m == 0
    assert not got[none].view(np.int32).any(), "%s: a row no id maps to is not +0" % what
    nan = np.isnan(s64)
    assert np.array_equal(np.isnan(got), nan), "%s: NaN at %s, want it at %s" % (
        what, np.argwhere(np.isnan(got))[:5].tolist(), np.argwhere(nan)[:5].tolist())
    inf = np.isinf(s64)
    assert np.array_equal(got[inf], s64[inf].astype(np.float32)), "%s: inf sums differ" % what
    fin = ~(nan | inf)
    few = fin & ((m == 1) | (m == 2))[:, None]
    touched = few & (has_sub | ((s32 != 0) & (np.abs(s32) < TINY)))
    lone = touched & (m == 1)[:, None]
    assert not got[lone].any(), "%s: a lone subnormal addend was not flushed to zero" % what
    near = np.abs(got[touched] - s64[touched]) <= 2 * np.broadcast_to(m[:, None], got.shape)[touched] * TINY
    assert near.all(), "%s: subnormal sums past the flush" % what
    bad = np.argwhere(few & ~touched & (got != s32))
    assert bad.size == 0, "%s: row of %d addends at %s: %r != float32 sum %r" % (
        what, m[bad[0][0]], tuple(bad[0]), got[tuple(bad[0])], s32[tuple(bad[0])])
    many = fin & (m >= 3)[:, None]
    mm = np.broadcast_to(m[:, None], got.shape)[many].astype(np.float64)
    err = np.abs(got[many].astype(np.float64) - s64[many])
    bound = ((mm - 1) * 2.0 ** -24 + mm * 2.0 ** -52) * a64[many] + 2 * mm * TINY
    assert (err <= bound).all(), "%s: %d sums past the recursive-summation bound, worst %g of %g" % (
        what, int((err > bound).sum()), float(err.max()), float(bound[np.argmax(err)]))


def _run_gather_sum(handle, aligned, T, k, dim, vals_d, inv_d, what):
    """b200ps_gather_rows and b200ps_segment_sum into poisoned outputs (one float off unless aligned); returns both."""
    lib = _lib()
    off = 0 if aligned else 1
    n = T * k * dim
    res = []
    for fn in (lib.b200ps_gather_rows, lib.b200ps_segment_sum):
        buf, out = _float_buf(n, off)
        before = lib.b200ps_launch_count(handle)
        assert fn(handle, vals_d.data_ptr(), inv_d.data_ptr(), T, k, dim, out.data_ptr(), _stream()) == 0, _err()
        torch.cuda.synchronize()
        assert lib.b200ps_launch_count(handle) == before + 1
        assert _untouched(buf, off, n), "%s: %s wrote outside its output" % (what, fn.__name__)
        res.append(out.view(T * k, dim).cpu().numpy())
    return res


def _gather_sum_configs(di, aligned):
    """(work, T, first pattern) for the dim at index di: two work sizes at T = 1, 3 segments (past one pass for every
    fourth dim, else 3001 rows) and 97 segments of 257 rows.  Work sizes and patterns rotate with the dim, the
    alignment and the segment, so that over the dims every work size meets every pattern and both alignments."""
    a = 0 if aligned else 1
    w0, w1 = WORKS[(di + a) % 4], WORKS[(di + a + 2) % 4]
    return [(w0, 1, di % 7), (w1, 1, (di + 3) % 7), ("pass+1" if (di + a) % 4 == 0 else 3001, 3, (di + 5) % 7),
            (257, 97, di % 7)]


@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "offset1"])
@pytest.mark.parametrize("dim", DIMS)
def test_gather_and_segment_sum_every_pass_dim_and_pattern(group, dim, aligned):
    """Gather and segment sum through the handle (poisoned outputs) and through ops (no handle), on 16 B aligned
    buffers and with values / bet and out one float off (the scalar fallback: the same results).  k is sized from
    the handle's SM count and from the 132 SMs ops' grid assumes; they coincide on a 132-SM H100."""
    from elasticdl_b200 import ops

    di = DIMS.index(dim)
    chunks = dim // _chunk_width(dim, aligned)
    off = 0 if aligned else 1
    gen = torch.Generator(device="cuda").manual_seed(dim * 2 + off)
    for work, T, p0 in _gather_sum_configs(di, aligned):
        by_k = {}
        for handle in (group._h, None):
            k = work if isinstance(work, int) else _k_for(work, _pass_items(handle is not None), chunks)
            by_k.setdefault(k, []).append(handle)
        for k, handles in by_k.items():
            rng = np.random.RandomState(k * 131 + dim)
            pats = [PATTERNS[(p0 + t) % 7] for t in range(T)]
            inv = np.stack([_inv_pattern(p, k, rng) for p in pats])
            dst = (np.arange(T)[:, None] * k + inv).reshape(-1)
            _, vals_d = _float_buf(T * k * dim, off)
            vals_d.copy_(torch.randn(T * k * dim, generator=gen, device="cuda"))
            inv_d = torch.from_numpy(inv).cuda().view(-1)
            vals = vals_d.view(T * k, dim).cpu().numpy()
            refs = _sum_refs(vals, dst, T * k)
            what = "%s dim %d %s T %d k %d (%s)" % (work, dim, "aligned" if aligned else "offset", T, k,
                                                  ",".join(sorted(set(pats))))
            for handle in handles:
                if handle is None:  # ops allocates `out` itself: only values / bet carry the offset
                    g = ops.gather_rows(vals_d, inv_d, T, k, dim).cpu().numpy()
                    s = ops.segment_sum(vals_d.view(T * k, dim), inv_d, T, k, dim).cpu().numpy()
                else:
                    g, s = _run_gather_sum(handle, aligned, T, k, dim, vals_d, inv_d, what)
                _check_gather(g, vals, dst, what + (" ops" if handle is None else " handle"))
                _check_sum(s, refs, what + (" ops" if handle is None else " handle"))


SUBNORMALS = np.array([1e-45, -1e-45, TINY / 2, -TINY / 4, TINY * 0.75, 3e-44], dtype=F32)


@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "offset1"])
@pytest.mark.parametrize("dim", [1, 8, 12])
def test_gather_and_segment_sum_inf_nan_and_subnormals(group, dim, aligned):
    """Rows of ±inf, NaN, -0 and subnormals among normal values, landing alone, in pairs (one warp and two), in fives
    and on one hot row: NaN and inf where the float64 sum has them; subnormals are flushed by the atomics (see
    _check_sum), which the lone subnormal addends pin."""
    T, k = 2, 4096
    rng = np.random.RandomState(dim)
    i = np.arange(k)
    seg0 = np.where(i < 1024, i, np.where(i < 2048, 1024 + (i - 1024) // 2, 1536 + i % 1024))  # 1, 2 near, 2 far
    seg1 = np.where(i < 2000, i // 5, np.where(i < 4000, 400 + (i - 2000) % 1000, 1400))  # 5, 2 far, hot
    inv = np.stack([seg0, seg1]).astype(np.int32)
    dst = (np.arange(T)[:, None] * k + inv).reshape(-1)
    vals = rng.standard_normal((T * k, dim)).astype(F32)
    specials = np.concatenate([[np.inf, -np.inf, np.nan, -0.0], SUBNORMALS]).astype(F32)
    pick = rng.random_sample(vals.shape) < 0.05
    vals[pick] = specials[rng.randint(len(specials), size=int(pick.sum()))]
    sub_rows = rng.choice(T * k, 300, replace=False)  # whole rows of subnormals: their sums are subnormal too
    vals[sub_rows] = SUBNORMALS[rng.randint(len(SUBNORMALS), size=(300, dim))]
    refs = _sum_refs(vals, dst, T * k)
    s64, _, _, m, has_sub = refs
    assert np.isnan(s64).any() and np.isinf(s64).any()
    assert (has_sub & (m == 1)[:, None]).sum() > 50  # lone subnormal addends
    off = 0 if aligned else 1
    _, vals_d = _float_buf(T * k * dim, off)
    vals_d.copy_(torch.from_numpy(vals.reshape(-1)).cuda())
    inv_d = torch.from_numpy(inv).cuda().view(-1)
    for handle in (group._h, None):
        what = "specials dim %d %s %s" % (dim, "aligned" if aligned else "offset", "handle" if handle else "no handle")
        g, s = _run_gather_sum(handle, aligned, T, k, dim, vals_d, inv_d, what)
        _check_gather(g, vals, dst, what)
        _check_sum(s, refs, what)


AUTOGRAD_CASES = ["exact_bet_T1", "T1", "T3", "T97"]


@pytest.mark.parametrize("case", AUTOGRAD_CASES)
@pytest.mark.parametrize("dim", [1, 8, 12, 100])
def test_gather_rows_autograd_matches_float64_index_select_and_index_add(dim, case):
    """ops.GatherRows forward (bit exact against index_select) and backward (index_add in float64, bounded as above),
    on an exact-shape BET [U, dim] (T = 1, padded to k rows inside), padded BETs and 97 segments."""
    from elasticdl_b200 import ops

    T = {"exact_bet_T1": 1, "T1": 1, "T3": 3, "T97": 97}[case]
    k = 3000 if T < 97 else 500
    rng = np.random.RandomState(dim * 10 + T)
    pats = [PATTERNS[(dim + t) % 7] for t in range(T)]
    inv = np.stack([_inv_pattern(p, k, rng) for p in pats])
    if case == "exact_bet_T1":
        inv = (rng.zipf(1.3, size=(1, k)) - 1) % 1000
        inv[0, :1000] = rng.permutation(1000)  # U = 1000 rows, every one of them used
        inv = inv.astype(np.int32)
        rows = 1000
    else:
        rows = T * k
    dst = (np.arange(T)[:, None] * k + inv).reshape(-1)
    bet = torch.from_numpy(rng.standard_normal((rows, dim)).astype(F32)).cuda().requires_grad_(True)
    inv_d = torch.from_numpy(inv).cuda().view(-1)
    out = ops.GatherRows.apply(bet, inv_d, T, k, dim)
    assert out.shape == (T * k, dim)
    want = bet.detach().cpu().double().index_select(0, torch.from_numpy(dst)).float()
    assert torch.equal(out.detach().cpu().view(torch.int32), want.view(torch.int32))
    up = torch.from_numpy(rng.standard_normal((T * k, dim)).astype(F32))
    out.backward(up.cuda())
    assert bet.grad.shape == (rows, dim)
    _check_sum(bet.grad.cpu().numpy(), _sum_refs(up.numpy(), dst, rows), "GatherRows backward %s dim %d" % (case, dim))


def test_gather_and_segment_sum_refuse_65536_segments(group):
    lib = _lib()
    vals = torch.zeros(65536 * 4, device="cuda")
    inv = torch.zeros(65536, dtype=torch.int32, device="cuda")
    for h in (group._h, None):
        for fn, msg in ((lib.b200ps_gather_rows, "bad gather shape"), (lib.b200ps_segment_sum, "bad segment_sum shape")):
            buf, out = _float_buf(65536 * 4, 0)
            before = lib.b200ps_launch_count(h)
            assert fn(h, vals.data_ptr(), inv.data_ptr(), 65536, 1, 4, out.data_ptr(), _stream()) == -1
            assert msg in _err()
            torch.cuda.synchronize()
            assert lib.b200ps_launch_count(h) == before and bool(torch.isnan(buf).all())


@pytest.mark.parametrize("k,dim", [(1 << 31, 1), (1 << 28, 10), ((1 << 28) + 1, 8)])
def test_segment_sum_refuses_work_past_int32_max(group, k, dim):
    """The warp key row x chunks + chunk is 32 bits: more than INT32_MAX work items per segment (2^31 rows of dim 1,
    2^28 rows of dim 10 in 10 scalar chunks, 2^28 + 1 rows of dim 8 unaligned) are refused before anything is
    zeroed or launched.  `out` is NULL, so a call that got past the check would fail in the memset before touching
    memory; the dim-8 values sit one float off a 16 B boundary (the scalar class).  The accepted side of the limit
    needs over 8 GB per buffer and is not run."""
    lib = _lib()
    vals = torch.zeros(8, device="cuda")
    for h in (group._h, None):
        before = lib.b200ps_launch_count(h)
        rc = lib.b200ps_segment_sum(h, vals.data_ptr() + (4 if dim == 8 else 0), None, 1, k, dim, None, _stream())
        assert rc == -1 and "INT32_MAX (2147483647)" in _err(), (rc, _err())
        assert lib.b200ps_launch_count(h) == before


# ================================================================================================ trainer
def test_trainer_batched_lookups_equal_per_layer_lookups_at_100_groups():
    """A 2 x 100-layer DeepFM: the batched lookups dedup one group of 100 segments (past 96: the equal-runs layout,
    bounds dropped), gather and segment-sum 100 segments per family and pull 200 requests (split at 96).  Three Adam
    minibatches train like the per-layer lookups: the same losses and dense parameters, and tables within the noise
    the atomics' summation order leaves (below)."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer
    from elasticdl_b200.workloads.deepfm import DeepFMLayersModel

    rows = [7, 300, 5000, 40, 1200] * 20
    B = 256

    def run(batched):
        torch.manual_seed(3)
        model = DeepFMLayersModel(rows, lr=0.01, initializer="uniform").cuda()
        g = PSGroup(2, *ADAM, device=0, seed=11)
        client = PSClient(g)
        client.dense_output = "torch"
        trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
            get_model_steps=1, batched_embedding_lookups=batched))
        gen = torch.Generator().manual_seed(5)
        losses = []
        for step in range(3):
            ids = torch.stack([torch.randint(0, r, (B,), generator=gen) for r in rows]).cuda()
            dense = torch.randn(B, 13, generator=gen).cuda()
            labels = (torch.rand(B, generator=gen) < 0.3).float().cuda()
            accepted, version, loss = trainer.train_minibatch(DeepFMLayersModel.features_of(ids, dense), labels)
            assert accepted and version == step + 1
            losses.append(float(loss))
        g.check()
        tabs = {}
        for gi, r in enumerate(rows):
            for fam in ("deep", "wide"):
                name = "%s_%d/embeddings:0" % (fam, gi)
                tabs[name] = client.pull_embedding_vectors(name, torch.arange(r).cuda()).cpu()
        params, _ = client.pull_dense_parameters([0, 1], [-1, -1])
        params = {n: v.cpu() for n, v in params.items()}
        plan = trainer._lookup_plan
        g.close()
        return losses, tabs, params, plan

    l_b, t_b, p_b, plan = run(True)
    l_p, t_p, p_p, plan_p = run(False)
    assert plan and plan_p is False
    assert sorted((k, dim, len(m)) for k, dim, m in plan) == [(B, 1, 100), (B, 8, 100)]
    assert np.allclose(l_b, l_p, rtol=1e-6, atol=1e-7), (l_b, l_p)
    # hot ids' gradient sums carry the atomics' order in their last bits, and Adam's division by sqrt(v) + 1e-7
    # magnifies that where a sum is near zero: the batched path run twice differs by up to 4e-7 in 4 of its 1.2 M
    # table values.  A wrong row or a lost gradient moves a value by about lr = 1e-3.
    for name in t_p:
        assert torch.allclose(t_b[name], t_p[name], rtol=1e-5, atol=2e-6), name
    for name in p_p:
        assert torch.allclose(p_b[name], p_p[name], rtol=1e-5, atol=1e-7), name
