"""Edge tests of the feature-id kernels (csrc/feature_ids.cu, include/b200_features.h) against
oracle/feature_oracle.py.

Integer outputs are compared bit exact; the Normalizer's float32 output is compared with np.array_equal
against the float64 oracle cast once to float32 (the kernel computes in double and casts once too).
Batch sizes come from the device's SM count, the way the launch sizes its grid, so that the grid-stride
loops run one, two and four passes.  Every output is carved from a larger buffer filled with a sentinel
(-7 for ids, NaN for dense), so a skipped sample or a write past the end shows.

Fingerprint64's 4..64-byte branches are PARITY UNPINNED: the kernel and the oracle restate the same
published FarmHash algorithm, and nothing independent of both (TensorFlow, pyfarmhash) is available
offline.  These tests pin the kernel to the oracle on every length branch; only the 1..3-byte branch is
pinned by the reference's own vector (tests/test_oracle_features.py).
"""
import ctypes
import functools

import numpy as np
import pytest
import torch

from oracle import feature_oracle as FO

pytestmark = pytest.mark.gpu

IDS_SENTINEL = -7
GUARD = 1031  # sentinel elements after every output
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
I2_BINS = [-1.0, 0.0, 1.0, 1.0, 3.0, 8.0, 23.0, 56.0, 184.0]  # dac_ctr I2: a repeated boundary
SHAPES = ["1", "255", "257", "pass-1", "pass", "pass+1", "3pass+17", "32768"]


def _lib():
    from elasticdl_b200 import _lib as L

    return L.lib()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _err():
    return _lib().b200feat_last_error().decode()


def _max_blocks():
    # feature_ids.cu max_blocks(): 8 resident blocks of 256 threads per SM (cudaDevAttrMultiProcessorCount)
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count * 8


def _pass(rows):
    """Samples one grid-stride pass covers when `rows` = G + n_dense grid rows share the blocks (grid_x, per)."""
    per = -(-_max_blocks() // rows)
    return min(per, _max_blocks()) * 256


def _batch(shape, rows):
    p = _pass(rows)
    return {"1": 1, "255": 255, "257": 257, "pass-1": p - 1, "pass": p, "pass+1": p + 1, "3pass+17": 3 * p + 17,
            "32768": 32768}[shape]


def _poisoned(n, dtype):
    """(whole buffer, its first n elements) with the sentinel everywhere."""
    buf = torch.full((n + GUARD,), float("nan") if dtype.is_floating_point else IDS_SENTINEL, dtype=dtype, device="cuda")
    return buf, buf[:n]


def _untouched(t):
    t = t.cpu()
    return bool(torch.isnan(t).all()) if t.dtype.is_floating_point else bool((t == IDS_SENTINEL).all())


# ---------------------------------------------------------------------------------------------- value pools
def _int_edges():
    v = [0, 1, -1, I64_MIN, I64_MAX, I64_MIN + 1, I64_MAX - 1]
    for k in range(1, 19):  # decimal lengths 1..20 cross every FarmHash branch tf.as_string can reach
        v += [10 ** k - 1, 10 ** k, -10 ** k, -(10 ** k - 1)]
    v += [(1 << 24) + 1, (1 << 24) + 3, (1 << 53) + 1, (1 << 62) + 12345, -(1 << 62) - 1]
    return v


@functools.lru_cache(None)
def _int_pool():
    rng = np.random.RandomState(11)
    extra = np.concatenate([rng.randint(-10 ** 6, 10 ** 6, 1500), rng.randint(I64_MIN, I64_MAX, 1000, dtype=np.int64)])
    return np.unique(np.concatenate([np.array(_int_edges(), dtype=np.int64), extra.astype(np.int64)]))


def _f32_specials():
    f = np.float32
    tiny = np.finfo(f).tiny
    return np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, tiny / 2, tiny, -tiny, np.finfo(f).max,
                     -np.finfo(f).max, 1e30, -1e30, 16777216.0, 16777218.0], dtype=f)


def _float_values(bins, dtype):
    """Each boundary, its neighbours in `dtype` (and in float32), the specials and values beyond both ends."""
    b = np.asarray(bins, dtype=np.float32).astype(dtype)
    v = [b, np.nextafter(b, dtype(-np.inf)), np.nextafter(b, dtype(np.inf)), _f32_specials().astype(dtype)]
    if dtype == np.float64:
        b32 = np.asarray(bins, dtype=np.float32)
        v += [np.nextafter(b32, np.float32(-np.inf)).astype(dtype), np.nextafter(b32, np.float32(np.inf)).astype(dtype),
              np.array([0.99999999, 1.00000001, 5e-324, -5e-324, 1e300, -1e300, 0.1], dtype=dtype)]
    return np.concatenate(v).astype(dtype)


@functools.lru_cache(None)
def _string_pool(W, n=3000, seed=0):
    """n distinct byte strings of length 0..W (bytes 1..255, a quarter of them all >= 0x80), as a tuple."""
    rng = np.random.RandomState(seed * 100 + W)
    pool = {b""}
    for L in range(W + 1):
        pool.add(bytes([0xFF] * L))
        pool.add(bytes(rng.randint(0x80, 256, size=L).astype(np.uint8)))
    while len(pool) < n:
        L = rng.randint(0, W + 1)
        lo = 0x80 if rng.rand() < 0.25 else 1
        pool.add(bytes(rng.randint(lo, 256, size=L).astype(np.uint8)))
    return tuple(sorted(pool))


@functools.lru_cache(None)
def _pool_matrix(pool, W):
    from elasticdl_b200.preprocessing import encode_strings

    return encode_strings(list(pool), W, device="cuda")


# The oracle's Fingerprint64 is pure Python: each distinct value is fingerprinted once, and Hashing's
# `fingerprint % num_bins` (unsigned) is taken in numpy.  test_hash_int_values_and_bin_counts and
# test_hash_strings_every_length_up_to_width compare against FO.hashing itself.
@functools.lru_cache(None)
def _pool_fp(pool):
    return np.array([FO.fingerprint64(s) for s in pool], dtype=np.uint64)


def _pool_hash(pool, num_bins):
    return (_pool_fp(pool) % np.uint64(num_bins)).astype(np.int64)


_INT_FP = {}  # value -> Fingerprint64 of its tf.as_string decimal


def _hash_ints(vals, num_bins):
    u, inv = np.unique(vals, return_inverse=True)
    for v in u.tolist():
        if v not in _INT_FP:
            _INT_FP[v] = FO.fingerprint64(str(v).encode("ascii"))
    fp = np.array([_INT_FP[v] for v in u.tolist()], dtype=np.uint64)
    return (fp % np.uint64(num_bins)).astype(np.int64)[inv.reshape(-1)].reshape(vals.shape)


# ------------------------------------------------------------------------------------------- fused helpers
def _want(groups, dense, num, str_cols):
    """Layer-by-layer oracle of a FeatureTransform; str_cols[j] = (pool, idx) of string column j."""
    ids = []
    for g in groups:
        if g["kind"] == "discretize":
            v = FO.discretize(num[g["column"]], g["bins"])
        elif g["kind"] == "hash":
            pool, idx = str_cols[g["column"]]
            v = _pool_hash(pool, g["num_bins"])[idx]
        else:
            v = _hash_ints(num[g["column"]], g["num_bins"])
        ids.append(v + g.get("offset", 0))
    want_dense = None
    if dense:
        want_dense = np.stack([FO.normalize(num[c], s, d) for c, s, d in dense], 1).astype(np.float32)
    return np.stack(ids), want_dense


def _run(ft, numeric, strings, bufs=None):
    """ft(numeric, strings) into poisoned, guarded outputs (reused from `bufs`); returns numpy outputs and bufs."""
    B = numeric.shape[1]
    if bufs is None:
        bufs = (_poisoned(ft.G * B, ft.ids_dtype), _poisoned(B * ft.n_dense, torch.float32) if ft.n_dense else None)
    (ibuf, ids), dpair = bufs
    dense = dpair[1].view(B, ft.n_dense) if dpair else None
    got_ids, got_dense = ft(numeric, strings, ids_out=ids.view(ft.G, B), dense_out=dense)
    assert got_ids.data_ptr() == ibuf.data_ptr()
    torch.cuda.synchronize()
    assert _untouched(ibuf[ft.G * B:]), "ids written past row G-1's end"
    if dpair:
        assert _untouched(dpair[0][B * ft.n_dense:]), "dense written past its end"
    return (got_ids.cpu().numpy().astype(np.int64), got_dense.cpu().numpy() if dpair else None), bufs


def _check(ft, groups, dense, num_np, numeric, strings, str_cols, bufs=None):
    (ids, d), bufs = _run(ft, numeric, strings, bufs)
    want_ids, want_dense = _want(groups, dense, num_np, str_cols)
    assert ids.shape == want_ids.shape
    bad = np.argwhere(ids != want_ids)
    assert bad.size == 0, "first wrong id at (group, sample) %s: %d != %d" % (
        tuple(bad[0]), ids[tuple(bad[0])], want_ids[tuple(bad[0])])
    if dense:
        assert np.array_equal(d, want_dense)
    return bufs


# ---------------------------------------------------------------------------------- single-op entry points
def _bucketize_bins():
    return sorted(I2_BINS + [-3.5e9, 1e-40, 2.0 ** 24, 2.0 ** 40])


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("op", ["hash_strings", "fingerprint64", "hash_ints", "bucketize"])
def test_single_op_entry_points_write_every_sample(op, shape):
    lib = _lib()
    B = _batch(shape, 1)
    rng = np.random.RandomState(B)
    buf, out = _poisoned(B, torch.int64)
    launches = lib.b200feat_launch_count()
    if op in ("hash_strings", "fingerprint64"):
        pool = _string_pool(8)
        idx = rng.randint(len(pool), size=B)
        mat = _pool_matrix(pool, 8)[torch.from_numpy(idx).cuda()]
        if op == "hash_strings":
            assert lib.b200feat_hash_strings(mat.data_ptr(), 8, B, 1000003, out.data_ptr(), _stream()) == 0, _err()
            want = _pool_hash(pool, 1000003)[idx]
        else:
            assert lib.b200feat_fingerprint64(mat.data_ptr(), 8, B, out.data_ptr(), _stream()) == 0, _err()
            want = _pool_fp(pool)[idx].view(np.int64)
    elif op == "hash_ints":
        vals = _int_pool()[rng.randint(len(_int_pool()), size=B)]
        x = torch.from_numpy(vals).cuda()
        assert lib.b200feat_hash_ints(x.data_ptr(), B, 1 << 62, out.data_ptr(), _stream()) == 0, _err()
        want = _hash_ints(vals, 1 << 62)
    else:
        bins = _bucketize_bins()
        pool = _float_values(bins, np.float32)
        vals = np.concatenate([pool, (rng.standard_normal(B) * 200).astype(np.float32)])[rng.permutation(len(pool) + B)[:B]]
        x = torch.from_numpy(vals).cuda()
        bnd = (ctypes.c_float * len(bins))(*bins)
        assert lib.b200feat_bucketize(x.data_ptr(), B, bnd, len(bins), out.data_ptr(), _stream()) == 0, _err()
        want = FO.discretize(vals, bins)
    torch.cuda.synchronize()
    assert lib.b200feat_launch_count() == launches + 1
    assert _untouched(buf[B:])
    got = out.cpu().numpy()
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, "first wrong sample %d of %d: %d != %d" % (bad[0], B, got[bad[0]], want[bad[0]])


# ------------------------------------------------------------------------------------------ fused batches
def _dac_ctr_numeric_pool(f):
    from elasticdl_b200.workloads.dac_ctr_features import FEATURE_BOUNDARIES

    rng = np.random.RandomState(5)
    b = np.floor(np.asarray(FEATURE_BOUNDARIES[f])).astype(np.int64)
    return np.unique(np.concatenate([b - 1, b, b + 1, [-2, -1, 0, (1 << 24) + 1, 10 ** 12, -10 ** 12],
                                     np.floor(rng.lognormal(0.0, 2.0, 400) * 10).astype(np.int64)]))


@functools.lru_cache(maxsize=2)
def _dac_ctr_batch(B, seed):
    from elasticdl_b200.workloads.dac_ctr_features import FEATURE_DISTINCT_COUNT, STANDARDIZED_FEATURES

    rng = np.random.RandomState(seed * 7919 + B)
    num = np.stack([p[rng.randint(len(p), size=B)] for p in map(_dac_ctr_numeric_pool, STANDARDIZED_FEATURES)])
    pool = _string_pool(8, 2000, seed=1)
    idx = rng.randint(len(pool), size=(len(FEATURE_DISTINCT_COUNT), B))
    strings = _pool_matrix(pool, 8)[torch.from_numpy(idx).cuda()]
    return num, torch.from_numpy(num).cuda(), strings, [(pool, i) for i in idx]


def _dac_ctr_spec():
    from elasticdl_b200.workloads.dac_ctr_features import (BUCKET_GROUP_FEATURES, FEATURE_BOUNDARIES, FEATURES_AVGS,
                                                           FEATURES_STDDEVS, HASH_BINS, STANDARDIZED_FEATURES)

    groups = [{"kind": "discretize", "column": STANDARDIZED_FEATURES.index(f), "bins": FEATURE_BOUNDARIES[f]}
              for f in BUCKET_GROUP_FEATURES]
    groups += [{"kind": "hash", "column": j, "num_bins": b} for j, b in enumerate(HASH_BINS)]
    dense = [(i, FEATURES_AVGS[f], FEATURES_STDDEVS[f]) for i, f in enumerate(STANDARDIZED_FEATURES)]
    return groups, dense


@pytest.mark.parametrize("ids_dtype", [torch.int64, torch.int32], ids=["ids64", "ids32"])
@pytest.mark.parametrize("shape", SHAPES)
def test_fused_dac_ctr_transform_every_sample_every_pass(shape, ids_dtype):
    """dac_ctr's 38 id groups + 13 Normalizer columns (workloads/dac_ctr_features.dac_ctr_transform), twice into
    the same guarded buffers with different batches."""
    from elasticdl_b200.workloads.dac_ctr_features import dac_ctr_transform

    ft = dac_ctr_transform(ids_dtype)
    groups, dense = _dac_ctr_spec()
    assert (ft.G, ft.n_dense) == (38, 13)
    B = _batch(shape, ft.G + ft.n_dense)
    bufs = None
    for seed in (0, 1):
        num, numeric, strings, str_cols = _dac_ctr_batch(B, seed)
        bufs = _check(ft, groups, dense, num, numeric, strings, str_cols, bufs)


def _widest_spec(ids32):
    """64 id groups + 32 Normalizer columns (the most grid rows, so the fewest blocks per row): discretize groups
    whose boundaries sum to 256, hash groups sharing string columns, hash_int groups, nonzero offsets, Normalizer
    columns in non-identity order, several reading one column, the last column among them."""
    rng = np.random.RandomState(3)
    counts = [0, 1, 2, 9, 32, 60, 100, 52]
    bins = [[], [0.0], [1.0, 1.0], I2_BINS, sorted(np.round(rng.standard_normal(32) * 100).tolist())]
    bins.append(sorted(rng.randint(-(1 << 30), 1 << 30, 60).astype(float).tolist()))
    bins.append(sorted(np.floor(rng.lognormal(0, 3, 100)).tolist()))
    bins.append(sorted([-1e30, -2.0 ** 53, -16777217.0, 2.0 ** 24, 2.0 ** 24 + 2, 2.0 ** 53, 2.0 ** 62, 1e30]
                       + rng.randint(-1000, 1000, 44).astype(float).tolist()))
    assert [len(b) for b in bins] == counts and sum(counts) == 256
    n_num, n_str = 10, 6
    groups = [{"kind": "discretize", "column": (3 * i + 1) % n_num, "bins": b, "offset": 1000 * i}
              for i, b in enumerate(bins)]
    hash_bins = [1, 2, 97, 1000003, (1 << 30) - 3, (1 << 31) - 1]
    for i in range(24):
        nb = hash_bins[i % len(hash_bins)]
        groups.append({"kind": "hash", "column": (5 * i) % n_str, "num_bins": nb,
                       "offset": 1 if nb == (1 << 31) - 1 else 17 * i})  # offset 1: ids reach 2^31 - 1 exactly
    for i in range(32):
        nb = hash_bins[i % len(hash_bins)] if ids32 else [1, 2, 1 << 31, (1 << 32) + 1, 1 << 62][i % 5]
        groups.append({"kind": "hash_int", "column": n_num - 1 - (i % n_num), "num_bins": nb,
                       "offset": 0 if nb >= (1 << 31) - 1 else 5 * i})
    assert len(groups) == 64
    dense = [((7 * j + 2) % n_num, float(rng.standard_normal() * 100), [3.0, -2.5, 1e-3, -1e-300, 7e5][j % 5])
             for j in range(32)]
    dense[-1] = (n_num - 1, 0.5, 1.0)
    return groups, dense, n_num, n_str


@pytest.mark.parametrize("ids_dtype", [torch.int64, torch.int32], ids=["ids64", "ids32"])
@pytest.mark.parametrize("shape", SHAPES)
def test_fused_64_groups_32_dense_every_sample_every_pass(shape, ids_dtype):
    from elasticdl_b200.preprocessing import FeatureTransform

    groups, dense, n_num, n_str = _widest_spec(ids_dtype == torch.int32)
    ft = FeatureTransform(groups, dense, ids_dtype)
    B = _batch(shape, 64 + 32)
    rng = np.random.RandomState(B)
    bins = np.concatenate([np.asarray(g["bins"], dtype=np.float64) for g in groups if g["kind"] == "discretize"])
    bins = np.floor(bins).clip(-2.0 ** 62, 2.0 ** 62).astype(np.int64)
    ints = np.concatenate([_int_pool(), bins - 1, bins, bins + 1])
    bufs = None
    for _ in range(2):
        num = ints[rng.randint(len(ints), size=(n_num, B))]
        pool = _string_pool(16, 2500, seed=2)
        idx = rng.randint(len(pool), size=(n_str, B))
        strings = _pool_matrix(pool, 16)[torch.from_numpy(idx).cuda()]
        bufs = _check(ft, groups, dense, num, torch.from_numpy(num).cuda(), strings, [(pool, i) for i in idx], bufs)


# ---------------------------------------------------------------------------------------------- discretize
BIN_SETS = {
    "none": [],
    "one": [0.0],
    "i2_repeated": I2_BINS,
    "signed_zero": [-1.0, -0.0, 0.0, 1e-45, 1e-38],
    "256": sorted(np.concatenate([np.random.RandomState(9).standard_normal(200) * 1e3, [1.0] * 6, [0.5, 0.5],
                                  -np.logspace(-40, 38, 24), np.logspace(-40, 38, 24)]).astype(np.float32).tolist()),
}


@pytest.mark.parametrize("bins", list(BIN_SETS), ids=list(BIN_SETS))
@pytest.mark.parametrize("dtype", ["float32", "float64", "int64", "int32"])
def test_discretization_at_boundaries_and_specials(bins, dtype):
    """Each boundary, its neighbours, ±0, ±inf, NaN, subnormals and values beyond both ends, through the
    Discretization layer: every input compares in float (float64 inputs are cast to float32 first)."""
    from elasticdl_b200.preprocessing import Discretization

    b = BIN_SETS[bins]
    assert len(BIN_SETS["256"]) == 256
    if dtype in ("float32", "float64"):
        vals = _float_values(b, np.dtype(dtype).type)
    else:
        lim = np.iinfo(dtype)
        fb = np.floor(np.asarray(b, dtype=np.float64)).clip(lim.min // 2, lim.max // 2).astype(np.int64)
        vals = np.concatenate([fb - 1, fb, fb + 1, [0, 1, -1, lim.min, lim.max, (1 << 24) - 1, 1 << 24, (1 << 24) + 1,
                                                    (1 << 24) + 3, -(1 << 24) - 1]]).astype(dtype)
    out = Discretization(b)(torch.from_numpy(vals).cuda())
    assert out.dtype == torch.int64 and out.shape == vals.shape
    assert np.array_equal(out.cpu().numpy(), FO.discretize(vals, b))


def test_discretization_casts_float64_inputs_to_float32():
    """The reference layer is a Keras Layer of the float32 dtype policy: __call__ autocasts a float64 input to
    float32 before math_ops._bucketize, so values next to a boundary round onto it."""
    from elasticdl_b200.preprocessing import Discretization

    x = torch.tensor([0.99999999, np.nextafter(1.0, 0.0), 1.0, 1.00000001, 0.9999999], dtype=torch.float64, device="cuda")
    assert Discretization([1.0])(x).tolist() == [1, 1, 1, 1, 0]
    assert Discretization([1.0])(x.float()).tolist() == [1, 1, 1, 1, 0]
    # int64 inputs above 2^24 round to float before comparing: 16777217 -> 16777216.0f lands on the boundary
    i = torch.tensor([16777215, 16777216, 16777217, 16777219], device="cuda")
    assert Discretization([16777216.0])(i).tolist() == [0, 1, 1, 1]
    assert Discretization([16777217.0, 16777220.0])(i).tolist() == [0, 1, 1, 2]


# ------------------------------------------------------------------------------------------------ hash_int
@pytest.mark.parametrize("num_bins", [1, 2, (1 << 31) - 1, 1 << 31, (1 << 32) + 1, 1 << 62])
def test_hash_int_values_and_bin_counts(num_bins):
    """0, ±1, INT64_MIN/MAX and ±10^k, 10^k - 1 (decimal lengths 1..20) through b200feat_hash_ints and a fused
    hash_int group; num_bins above 2^31 with int64 ids only."""
    from elasticdl_b200.preprocessing import FeatureTransform

    vals = np.array(_int_edges(), dtype=np.int64)
    want = FO.hashing(vals, num_bins)
    x = torch.from_numpy(vals).cuda()
    buf, out = _poisoned(len(vals), torch.int64)
    assert _lib().b200feat_hash_ints(x.data_ptr(), len(vals), num_bins, out.data_ptr(), _stream()) == 0, _err()
    torch.cuda.synchronize()
    assert _untouched(buf[len(vals):]) and np.array_equal(out.cpu().numpy(), want)
    if num_bins == 1:
        assert not want.any()
    if num_bins == 1 << 62:
        assert want.max() >= 1 << 32  # the modulo is 64-bit
    for ids_dtype in ([torch.int64, torch.int32] if num_bins < 1 << 31 else [torch.int64]):
        groups = [{"kind": "hash_int", "column": 1, "num_bins": num_bins},
                  {"kind": "hash_int", "column": 0, "num_bins": num_bins, "offset": 3 if num_bins < 1 << 30 else 0}]
        num = np.stack([vals[::-1].copy(), vals])
        _check(FeatureTransform(groups, (), ids_dtype), groups, (), num, torch.from_numpy(num).cuda(), None, [])


# ---------------------------------------------------------------------------------------------- hash string
@pytest.mark.parametrize("W", [1, 3, 4, 7, 8, 9, 15, 16, 17, 31, 32, 33, 63, 64])
def test_hash_strings_every_length_up_to_width(W):
    """Lengths 0..W (W itself: no terminator), bytes >= 0x80, through b200feat_hash_strings,
    b200feat_fingerprint64 and a fused launch with several string columns."""
    from elasticdl_b200.preprocessing import FeatureTransform

    lib = _lib()
    pool = _string_pool(W, 200 if W == 1 else 400)  # W = 1 has 256 distinct strings
    assert {len(s) for s in pool} == set(range(W + 1))
    mat = _pool_matrix(pool, W)
    n = len(pool)
    for num_bins in (1000003, (1 << 32) + 1):
        buf, out = _poisoned(n, torch.int64)
        assert lib.b200feat_hash_strings(mat.data_ptr(), W, n, num_bins, out.data_ptr(), _stream()) == 0, _err()
        torch.cuda.synchronize()
        assert _untouched(buf[n:]) and np.array_equal(out.cpu().numpy(), FO.hashing(list(pool), num_bins))
    buf, out = _poisoned(n, torch.int64)
    assert lib.b200feat_fingerprint64(mat.data_ptr(), W, n, out.data_ptr(), _stream()) == 0, _err()
    torch.cuda.synchronize()
    assert _untouched(buf[n:]) and np.array_equal(out.cpu().numpy().view(np.uint64), _pool_fp(pool))

    rng = np.random.RandomState(W)
    idx = np.stack([rng.permutation(n), np.arange(n), rng.randint(n, size=n)])
    strings = mat[torch.from_numpy(idx).cuda()]
    for ids_dtype in (torch.int64, torch.int32):
        big = (1 << 62) if ids_dtype == torch.int64 else (1 << 31) - 1
        groups = [{"kind": "hash", "column": 2, "num_bins": 7, "offset": 100},
                  {"kind": "hash", "column": 0, "num_bins": big},
                  {"kind": "hash", "column": 1, "num_bins": 1000},
                  {"kind": "hash", "column": 2, "num_bins": 2}]
        num = np.zeros((1, n), dtype=np.int64)
        _check(FeatureTransform(groups, (), ids_dtype), groups, (), num, torch.from_numpy(num).cuda(), strings,
               [(pool, i) for i in idx])


# -------------------------------------------------------------------------------------------- composition
def test_fused_offsets_hash_int_column_order_and_normalizer_edges():
    """Offsets up to 2^40 with int64 ids; discretize / hash / hash_int groups reading int64 columns in
    non-identity order, several on one column, the last column; Normalizer with a negative divisor, a tiny
    divisor and values above 2^53."""
    from elasticdl_b200.preprocessing import FeatureTransform

    rng = np.random.RandomState(4)
    B = 3 * _pass(9 + 5) + 17
    n_num = 4
    groups = [{"kind": "discretize", "column": 3, "bins": I2_BINS, "offset": 1 << 40},
              {"kind": "hash_int", "column": 3, "num_bins": (1 << 32) + 1, "offset": 1 << 40},
              {"kind": "hash", "column": 1, "num_bins": 1 << 62, "offset": 12345},
              {"kind": "discretize", "column": 0, "bins": [2.0 ** 53, 2.0 ** 60]},
              {"kind": "hash_int", "column": 2, "num_bins": 1000003, "offset": 7},
              {"kind": "hash", "column": 0, "num_bins": 3},
              {"kind": "discretize", "column": 3, "bins": [], "offset": (1 << 40) + 1},
              {"kind": "hash_int", "column": 0, "num_bins": 1 << 62},
              {"kind": "discretize", "column": 2, "bins": [0.0]}]
    dense = [(3, 0.25, -3.0), (0, -1.5, 1e-300), (3, 0.0, 7.0), (2, 1e15, 2.5e-7), (1, 2.0 ** 53, -1.0)]
    ints = np.concatenate([_int_pool(), [(1 << 53) + 1, (1 << 53) + 3, (1 << 60) - 1, 1 << 60]]).astype(np.int64)
    num = ints[rng.randint(len(ints), size=(n_num, B))]
    pool = _string_pool(12, 1500, seed=3)
    idx = rng.randint(len(pool), size=(2, B))
    strings = _pool_matrix(pool, 12)[torch.from_numpy(idx).cuda()]
    ft = FeatureTransform(groups, dense, torch.int64)
    bufs = _check(ft, groups, dense, num, torch.from_numpy(num).cuda(), strings, [(pool, i) for i in idx])
    num2 = num[:, ::-1].copy()
    _check(ft, groups, dense, num2, torch.from_numpy(num2).cuda(), strings, [(pool, i) for i in idx], bufs)


@pytest.mark.parametrize("ids_dtype", [torch.int64, torch.int32], ids=["ids64", "ids32"])
def test_fused_float32_numeric_columns(ids_dtype):
    """Float32 numeric columns for Discretization (specials included: compared in float) and the Normalizer."""
    from elasticdl_b200.preprocessing import FeatureTransform

    rng = np.random.RandomState(6)
    B = _pass(6 + 4) + 1
    bins_a, bins_b = I2_BINS, BIN_SETS["256"][::2]
    spec = np.concatenate([_float_values(bins_a, np.float32), _float_values(bins_b, np.float32)])
    finite = np.concatenate([spec[np.isfinite(spec)], (rng.standard_normal(500) * 1e4).astype(np.float32)])
    num = np.stack([spec[rng.randint(len(spec), size=B)], finite[rng.randint(len(finite), size=B)],
                    spec[rng.randint(len(spec), size=B)]]).astype(np.float32)
    groups = [{"kind": "discretize", "column": 2, "bins": bins_a, "offset": 11},
              {"kind": "discretize", "column": 0, "bins": bins_b},
              {"kind": "discretize", "column": 1, "bins": bins_a, "offset": 3},
              {"kind": "discretize", "column": 2, "bins": [0.0]},
              {"kind": "hash", "column": 0, "num_bins": 1000},
              {"kind": "discretize", "column": 2, "bins": []}]
    dense = [(1, 3.0, -0.5), (1, 0.0, 1e-30), (1, -7.25, 3.0), (1, 1e6, 1e-3)]
    pool = _string_pool(4, 200, seed=4)
    idx = rng.randint(len(pool), size=(1, B))
    strings = _pool_matrix(pool, 4)[torch.from_numpy(idx).cuda()]
    ft = FeatureTransform(groups, dense, ids_dtype)
    _check(ft, groups, dense, num, torch.from_numpy(num).cuda(), strings, [(pool, idx[0])])


# ------------------------------------------------------------------------------------------------- layers
def test_layers_on_2d_3d_noncontiguous_and_int32_inputs():
    from elasticdl_b200.preprocessing import Discretization, Hashing

    rng = np.random.RandomState(8)
    ints = _int_pool()[rng.randint(len(_int_pool()), size=(6, 5, 4))]
    x = torch.from_numpy(ints).cuda()
    h = Hashing(1000003)
    for v in (x, x[0], x.transpose(0, 2), x[:, ::2, 1:], x[..., 0].t()):
        out = h(v)
        assert out.dtype == torch.int64 and out.shape == v.shape
        assert np.array_equal(out.cpu().numpy(), FO.hashing(v.cpu().numpy(), 1000003))
    i32 = torch.from_numpy(ints.clip(-2 ** 31, 2 ** 31 - 1).astype(np.int32)).cuda()[:, 1::2]
    out = h(i32)
    assert out.dtype == torch.int64 and out.shape == i32.shape
    assert np.array_equal(out.cpu().numpy(), FO.hashing(i32.cpu().numpy(), 1000003))

    pool = _string_pool(9, 300, seed=5)
    idx = rng.randint(len(pool), size=(4, 6))
    s = _pool_matrix(pool, 9)[torch.from_numpy(idx).cuda()]  # [4, 6, 9]
    for v, i in ((s, idx), (s[::2], idx[::2]), (s.transpose(0, 1), idx.T), (s[1], idx[1])):
        out = h(v)
        assert out.dtype == torch.int64 and out.shape == v.shape[:-1]
        assert np.array_equal(out.cpu().numpy(), _pool_hash(pool, 1000003)[i])

    d = Discretization(I2_BINS)
    f = torch.from_numpy(np.resize(_float_values(I2_BINS, np.float32), 60).reshape(3, 4, 5)).cuda()
    for v in (f, f.transpose(1, 2), f[:, ::3], f.double().permute(2, 0, 1), i32, x[:, 1]):
        out = d(v)
        assert out.dtype == torch.int64 and out.shape == v.shape
        assert np.array_equal(out.cpu().numpy(), FO.discretize(v.cpu().numpy(), I2_BINS))


def test_empty_batch_gives_empty_outputs_without_a_launch():
    from elasticdl_b200.preprocessing import Discretization, FeatureTransform, Hashing

    lib = _lib()
    n = lib.b200feat_launch_count()
    groups, dense = _dac_ctr_spec()
    ft = FeatureTransform(groups, dense)
    ids, d = ft(torch.zeros((13, 0), dtype=torch.int64, device="cuda"), torch.zeros((26, 0, 8), dtype=torch.uint8, device="cuda"))
    assert ids.shape == (38, 0) and ids.dtype == torch.int64 and d.shape == (0, 13) and d.dtype == torch.float32
    assert Hashing(5)(torch.zeros((0, 3), dtype=torch.int64, device="cuda")).shape == (0, 3)
    assert Discretization([1.0])(torch.zeros((2, 0), dtype=torch.float64, device="cuda")).shape == (2, 0)
    assert lib.b200feat_launch_count() == n


# ----------------------------------------------------------------------------------------------- refusals
def _raw(groups, boundaries=(), dense=(), n_numeric=2, numeric_is_float=0, n_string=1, W=8, B=300, ids32=0):
    """b200feat_transform straight through the C ABI into poisoned outputs; returns (rc, message, launches made,
    outputs untouched)."""
    from elasticdl_b200.preprocessing.layers import FeatureDense, FeatureGroup

    G, nd = len(groups), len(dense)
    ga = (FeatureGroup * max(G, 1))()
    for g, spec in enumerate(groups):
        ga[g].kind, ga[g].column = spec.get("kind", 1), spec.get("column", 0)
        ga[g].n_boundaries, ga[g].boundary_off = spec.get("n_boundaries", 0), spec.get("boundary_off", 0)
        ga[g].num_bins, ga[g].offset = spec.get("num_bins", 10), spec.get("offset", 0)
    da = (FeatureDense * max(nd, 1))()
    for j, (c, s, dv) in enumerate(dense):
        da[j].column, da[j].subtractor, da[j].divisor = c, s, dv
    bnd = (ctypes.c_float * max(len(boundaries), 1))(*boundaries)
    Bp = max(B, 1)
    numeric = torch.zeros((n_numeric, Bp), dtype=torch.float32 if numeric_is_float else torch.int64, device="cuda")
    strings = torch.full((max(n_string, 1), Bp, max(W, 1)), 65, dtype=torch.uint8, device="cuda")
    ibuf, ids = _poisoned(max(G, 1) * Bp, torch.int32 if ids32 else torch.int64)
    dbuf, dout = _poisoned(max(nd, 1) * Bp, torch.float32)
    lib = _lib()
    n = lib.b200feat_launch_count()
    rc = lib.b200feat_transform(ga, G, bnd, len(boundaries), da, nd, numeric.data_ptr(), n_numeric, numeric_is_float,
                                strings.data_ptr(), n_string, W, B, ids.data_ptr(), ids32, dout.data_ptr(), _stream())
    msg = _err()
    torch.cuda.synchronize()
    return rc, msg, lib.b200feat_launch_count() - n, _untouched(ibuf) and _untouched(dbuf)


HASH = {"kind": 1, "column": 0, "num_bins": 10}
DISC = {"kind": 0, "column": 0, "n_boundaries": 3, "boundary_off": 0}
REFUSALS = {
    "65_groups": (dict(groups=[HASH] * 65), "group count"),
    "33_dense": (dict(groups=[HASH], dense=[(0, 0.0, 1.0)] * 33), "dense column count"),
    "257_boundaries": (dict(groups=[dict(DISC, n_boundaries=257)], boundaries=list(range(257))), "too many boundaries"),
    "boundaries_out_of_range": (dict(groups=[dict(DISC, boundary_off=1)], boundaries=[0.0, 1.0, 2.0]), "out of range"),
    "W_65": (dict(groups=[HASH], W=65), "longer than 64"),
    "zero_batch": (dict(groups=[HASH], B=0), "batch size"),
    "num_bins_0": (dict(groups=[dict(HASH, num_bins=0)]), "num_bins"),
    "num_bins_negative": (dict(groups=[dict(HASH, kind=2, num_bins=-5)]), "num_bins"),
    "divisor_0": (dict(groups=[HASH], dense=[(0, 1.0, 0.0)]), "divisor"),
    "bad_string_column": (dict(groups=[HASH, dict(HASH, column=1)]), "bad string column"),
    "bad_numeric_column": (dict(groups=[dict(DISC, column=2)], boundaries=[0.0, 1.0, 2.0]), "bad numeric column"),
    "bad_hash_int_column": (dict(groups=[dict(HASH, kind=2, column=-1)]), "bad numeric column"),
    "bad_normalizer_column": (dict(groups=[HASH], dense=[(2, 0.0, 1.0)]), "bad numeric column"),
    "unknown_kind": (dict(groups=[HASH, dict(HASH, kind=3)]), "unknown group kind"),
    "unsorted_boundaries": (dict(groups=[DISC], boundaries=[0.0, 2.0, 1.0]), "not sorted"),
    "nan_boundary": (dict(groups=[DISC], boundaries=[0.0, float("nan"), 1.0]), "not sorted"),
    "unsorted_second_group": (dict(groups=[dict(DISC, n_boundaries=2), dict(DISC, n_boundaries=2, boundary_off=2)],
                                   boundaries=[0.0, 1.0, 5.0, 4.0]), "not sorted"),
    "hash_int_on_float32": (dict(groups=[dict(HASH, kind=2)], numeric_is_float=1), "hash_int"),
    "int32_num_bins_2^31_plus_offset": (dict(groups=[dict(HASH, num_bins=1 << 31, offset=1)], ids32=1), "int32"),
    "int32_num_bins_2^32": (dict(groups=[dict(HASH, kind=2, num_bins=1 << 32)], ids32=1), "int32"),
    "int32_discretize_offset": (dict(groups=[dict(DISC, offset=(1 << 31) - 3)], boundaries=[0.0, 1.0, 2.0], ids32=1),
                                "int32"),
    "int32_negative_offset": (dict(groups=[dict(HASH, offset=-(1 << 31) - 1)], ids32=1), "int32"),
}


@pytest.mark.parametrize("case", list(REFUSALS), ids=list(REFUSALS))
def test_transform_refusals_name_the_cause_and_launch_nothing(case):
    kw, cause = REFUSALS[case]
    rc, msg, launched, untouched = _raw(**kw)
    assert rc == -1 and cause in msg, (rc, msg)
    assert launched == 0 and untouched


def test_int32_limits_accept_the_largest_fitting_groups():
    for kw in (dict(groups=[dict(HASH, num_bins=1 << 31)]), dict(groups=[dict(HASH, num_bins=(1 << 31) - 1, offset=1)]),
               dict(groups=[dict(DISC, offset=(1 << 31) - 4)], boundaries=[0.0, 1.0, 2.0]),
               dict(groups=[dict(HASH, offset=-(1 << 31))])):
        rc, msg, launched, untouched = _raw(ids32=1, **kw)
        assert rc == 0 and launched == 1 and not untouched, msg


def test_single_op_refusals():
    lib = _lib()
    x = torch.zeros(64, dtype=torch.float32, device="cuda")
    buf, out = _poisoned(64, torch.int64)
    n = lib.b200feat_launch_count()
    bnd = (ctypes.c_float * 3)(0.0, 2.0, 1.0)
    assert lib.b200feat_bucketize(x.data_ptr(), 64, bnd, 3, out.data_ptr(), _stream()) == -1 and "not sorted" in _err()
    assert lib.b200feat_hash_ints(x.long().data_ptr(), 64, 0, out.data_ptr(), _stream()) == -1 and "num_bins" in _err()
    s = torch.ones((64, 65), dtype=torch.uint8, device="cuda")
    assert lib.b200feat_hash_strings(s.data_ptr(), 65, 64, 10, out.data_ptr(), _stream()) == -1
    assert "longer than 64" in _err()
    torch.cuda.synchronize()
    assert lib.b200feat_launch_count() == n and _untouched(buf)


def test_layer_refusals():
    from elasticdl_b200.preprocessing import Discretization, FeatureTransform, encode_strings

    with pytest.raises(ValueError, match="NUL"):
        encode_strings([b"ab", b"a\x00b"])
    with pytest.raises(ValueError, match="NUL"):
        encode_strings([[b"ab\x00"]], 8)
    with pytest.raises(ValueError, match="sorted"):
        Discretization([0.0, 2.0, 1.0])
    with pytest.raises(ValueError, match="sorted"):
        FeatureTransform([{"kind": "discretize", "column": 0, "bins": [3.0, 1.0]}])
    with pytest.raises(ValueError, match="unknown group kind"):
        FeatureTransform([{"kind": "hash_float", "column": 0, "num_bins": 3}])
    with pytest.raises(ValueError, match="num_bins"):
        FeatureTransform([{"kind": "hash_int", "column": 0, "num_bins": 0}])
    for spec in ({"kind": "hash", "column": 0, "num_bins": (1 << 31) + 1},
                 {"kind": "hash_int", "column": 0, "num_bins": 1 << 31, "offset": 1},
                 {"kind": "discretize", "column": 0, "bins": [0.0] * 10, "offset": (1 << 31) - 10},
                 {"kind": "hash", "column": 0, "num_bins": 5, "offset": -(1 << 31) - 1}):
        with pytest.raises(ValueError, match="int32"):
            FeatureTransform([spec], ids_dtype=torch.int32)
        FeatureTransform([spec], ids_dtype=torch.int64)
    FeatureTransform([{"kind": "discretize", "column": 0, "bins": [0.0] * 9, "offset": (1 << 31) - 10}], ids_dtype=torch.int32)

    lib = _lib()
    ft = FeatureTransform([{"kind": "discretize", "column": 0, "bins": [1.0]}, {"kind": "hash_int", "column": 0, "num_bins": 9}])
    buf, ids = _poisoned(2 * 16, torch.int64)
    n = lib.b200feat_launch_count()
    with pytest.raises(TypeError, match="hash_int"):
        ft(torch.zeros((1, 16), device="cuda"), ids_out=ids.view(2, 16))
    with pytest.raises(ValueError, match="ids_out"):
        ft(torch.zeros((1, 16), dtype=torch.int64, device="cuda"), ids_out=ids.view(2, 16)[:, :8])
    torch.cuda.synchronize()
    assert lib.b200feat_launch_count() == n and _untouched(buf)
