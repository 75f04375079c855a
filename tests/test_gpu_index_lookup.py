"""GPU tests of IndexLookup / LogRound / RoundIdentity (csrc/feature_ids.cu, include/b200_features.h) and of the
fused census transform, against oracle/lookup_oracle.py and oracle/feature_oracle.py.

Ids are compared bit exact.  The one allowance is LogRound's half-integer ties: CUDA's double log is within 1 ulp,
not correctly rounded, so where the oracle's quotient lies within 4 ulp of k + 0.5 both k and k + 1 are accepted.
Exact powers of the base are asserted strictly.  Outputs are carved from buffers poisoned past their end, and batch
sizes come from the device's SM count the way the launch sizes its grid, so the grid-stride loops run one, two and
four passes."""
import ctypes
import functools

import numpy as np
import pytest
import torch

from oracle import feature_oracle as FO
from oracle import lookup_oracle as LO

pytestmark = pytest.mark.gpu

IDS_SENTINEL = -7
GUARD = 1031
SHAPES = ["1", "255", "257", "pass-1", "pass", "pass+1", "3pass+17", "32768"]


def _lib():
    from elasticdl_b200 import _lib as L

    return L.lib()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _err():
    return _lib().b200feat_last_error().decode()


def _pass(rows):
    """Samples one grid-stride pass covers when `rows` grid rows share the launch's 8 blocks of 256 per SM."""
    mb = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count * 8
    return min(-(-mb // rows), mb) * 256


def _batch(shape, rows):
    p = _pass(rows)
    return {"1": 1, "255": 255, "257": 257, "pass-1": p - 1, "pass": p, "pass+1": p + 1, "3pass+17": 3 * p + 17,
            "32768": 32768}[shape]


def _poisoned(n, dtype=torch.int64):
    buf = torch.full((n + GUARD,), IDS_SENTINEL, dtype=dtype, device="cuda")
    return buf, buf[:n]


def _untouched(t):
    return bool((t.cpu() == IDS_SENTINEL).all())


def _rows(strings, W):
    """list of bytes (may hold NULs, each at most W bytes) -> uint8 CUDA tensor [n, W], zero padded."""
    buf = np.zeros((len(strings), W), dtype=np.uint8)
    for i, b in enumerate(strings):
        buf[i, :len(b)] = np.frombuffer(b, dtype=np.uint8)
    return torch.from_numpy(buf).cuda()


@functools.lru_cache(None)
def _vocab(V, seed=0):
    """V distinct terms of every width 1..64 (bytes 1..255), with "" at position min(3, V - 1) when V >= 4."""
    rng = np.random.RandomState(seed * 7 + V % 1000)
    if V > 5000:  # fast path: distinct by construction (a unique counter in the first 4 bytes, never NUL)
        lens = rng.randint(4, 65, V)
        body = rng.randint(1, 256, size=(V, 64)).astype(np.uint8)
        i = np.arange(V, dtype=np.int64)
        for k in range(4):
            body[:, k] = ((i >> (7 * k)) & 0x7F) + 1
        terms = [bytes(body[j, :lens[j]]) for j in range(V)]
    else:
        seen, terms = set(), []
        while len(terms) < V:
            L = 1 + len(terms) % 64 if len(terms) < 128 else rng.randint(1, 65)
            t = bytes(rng.randint(0x80 if rng.rand() < 0.25 else 1, 256, size=L).astype(np.uint8))
            if t not in seen:
                seen.add(t)
                terms.append(t)
    if V >= 4:
        terms[3] = b""
    return tuple(terms)


def _log_round_check(got, values, num_bins, default_value, base, strict=()):
    """Bit exact, except where the oracle's quotient lies within 4 ulp of a half integer (both neighbours accepted);
    positions in `strict` are always exact."""
    want = LO.log_round(values, num_bins, default_value, base)
    q = LO.log_round_q(values, base)
    with np.errstate(invalid="ignore"):
        tie = np.isfinite(q) & (np.abs(q - (np.floor(q) + 0.5)) <= 4 * np.spacing(np.abs(q)))
    tie[list(strict)] = False
    lo = LO._rounded_ids(np.floor(q), num_bins, default_value)
    hi = LO._rounded_ids(np.floor(q) + 1, num_bins, default_value)
    ok = (got == want) | (tie & ((got == lo) | (got == hi)))
    bad = np.flatnonzero(~ok)
    assert bad.size == 0, "first wrong value %r: %d != %d" % (values.reshape(-1)[bad[0]], got.reshape(-1)[bad[0]],
                                                              want.reshape(-1)[bad[0]])


# ------------------------------------------------------------------------------------- reference vectors
def test_reference_vectors_through_the_layers(tmp_path):
    from elasticdl_b200.preprocessing import IndexLookup, LogRound, RoundIdentity, encode_strings

    dense = encode_strings([["A"], ["B"], ["C"], ["D"], ["E"]])
    path = tmp_path / "vocab_test.txt"
    path.write_text("A\nB\nC\n")
    for vocab in (["A", "B", "C"], str(path)):
        layer = IndexLookup(vocabulary=vocab)
        assert layer(dense).tolist() == [[0], [1], [2], [3], [3]]  # index_lookup_test.py:55-59
        assert layer(encode_strings(["A", "B", "C", "D", "E"])).tolist() == [0, 1, 2, 3, 3]  # ragged / sparse values
        assert layer.vocab_size() == 4 and layer.get_config() == {"num_oov_tokens": 1, "vocabulary": None}
    assert IndexLookup(["A", "B", "C"])(encode_strings([["A"], ["C"], ["B"], ["D"], ["E"]])).tolist() == \
        [[0], [2], [1], [3], [3]]

    lr = LogRound(num_bins=20, base=2)  # log_round_test.py:27-61
    assert lr(torch.tensor([[0.0], [2.6], [0.2], [3.1], [1024]], device="cuda")).tolist() == [[0], [1], [0], [2], [10]]
    assert lr(torch.tensor([1.1, 3.4, 1025], device="cuda")).tolist() == [0, 2, 10]
    assert lr(torch.tensor([[1.2], [2.6], [0.2], [3.1], [1024]], device="cuda", dtype=torch.float64)).tolist() == \
        [[0], [1], [0], [2], [10]]
    assert LogRound(16, base=2)(torch.tensor([[1.2], [1.6], [0.2], [3.1], [100]], device="cuda")).tolist() == \
        [[0], [1], [0], [2], [7]]  # log_round.py:34-40
    ri = RoundIdentity(num_buckets=10)  # round_identity_test.py:27-47
    assert ri(torch.tensor([[1.2], [1.6], [0.2], [3.1], [4.9]], device="cuda")).tolist() == [[1], [2], [0], [3], [5]]
    assert ri(torch.tensor([1.1, 3.4, 0.5], device="cuda", dtype=torch.float16)).tolist() == [1, 3, 0]
    assert ri(torch.tensor([-1, 0, 9, 10], device="cuda", dtype=torch.int32)).tolist() == [0, 0, 9, 0]


# ------------------------------------------------------------------------------------------ IndexLookup
LOOKUP_CASES = [(1, 0), (1, 1), (1, 7), (8, 0), (8, 1), (8, 7), (1024, 1), (100000, 1), ((1 << 20) + 3, 1),
                (1 << 20, 7)]


@pytest.mark.parametrize("V,n_oov", LOOKUP_CASES, ids=["V%d-oov%d" % c for c in LOOKUP_CASES])
def test_index_lookup_bit_exact_against_the_oracle(V, n_oov):
    """Every term (all widths 1..64), strings outside the vocabulary, terms with bytes after a NUL, truncated and
    extended terms, "" inside (V >= 4) and outside (V < 4) the vocabulary; input widths below, at and above Wv.
    V a power of two fills the table to its maximum load (n_slots = 2V), so long probe chains are walked."""
    from elasticdl_b200.preprocessing import IndexLookup

    terms = _vocab(V)
    layer = IndexLookup(list(terms), num_oov_tokens=n_oov)
    assert layer.vocab_size() == V + n_oov
    assert layer.slots.shape[0] == _lib().b200feat_vocab_slots(V) and layer.terms.shape == (V, layer.Wv)
    if V & (V - 1) == 0 and V > 1:
        assert layer.slots.shape[0] == 2 * V
    rng = np.random.RandomState(V + n_oov)
    pick = rng.choice(V, min(V, 6000), replace=False)
    for W in sorted({layer.Wv, max(layer.Wv - 3, 1), 64}):
        inputs = [terms[i] for i in pick if len(terms[i]) <= W]
        inputs += [terms[i][:-1] for i in pick[:500] if len(terms[i]) <= W]  # prefixes: mostly out of vocabulary
        inputs += [terms[i] + b"\0" + b"\x01" * (W - len(terms[i]) - 1) for i in pick[:500] if len(terms[i]) < W]
        inputs += [terms[i] + b"x" for i in pick[:300] if len(terms[i]) < W]
        inputs += [bytes(rng.randint(1, 256, size=rng.randint(0, W + 1)).astype(np.uint8)) for _ in range(1500)]
        inputs += [b"", b"\0" * W, b"\xff" * W]
        x = _rows(inputs, W)
        buf, out = _poisoned(len(inputs))
        assert _lib().b200feat_index_lookup(x.data_ptr(), W, len(inputs), layer.slots.data_ptr(), layer.terms.data_ptr(),
                                            layer.slots.shape[0], V, layer.Wv, n_oov, out.data_ptr(), _stream()) == 0, _err()
        want = LO.index_lookup(inputs, terms, n_oov)
        torch.cuda.synchronize()
        assert _untouched(buf[len(inputs):])
        got = out.cpu().numpy()
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, "W=%d: first wrong input %r: %d != %d" % (W, inputs[bad[0]], got[bad[0]], want[bad[0]])
        k = min(len(inputs), 4000) // 40 * 40  # the layer on a [40, k / 40, W] view of the same rows
        assert np.array_equal(layer(x[:k].view(40, -1, W)).cpu().numpy().reshape(-1), want[:k])
    if V < 4:
        assert LO.index_lookup([b""], terms, n_oov)[0] == (V + FO.fingerprint64(b"") % n_oov if n_oov else -1)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("op", ["index_lookup", "log_round", "round_identity"])
def test_single_op_entry_points_write_every_sample(op, shape):
    lib = _lib()
    B = _batch(shape, 1)
    rng = np.random.RandomState(B)
    buf, out = _poisoned(B)
    launches = lib.b200feat_launch_count()
    if op == "index_lookup":
        from elasticdl_b200.preprocessing import IndexLookup

        terms = _vocab(1000)
        layer = IndexLookup(list(terms), num_oov_tokens=5)
        pool = list(terms[:400]) + [b"oov-%d" % i for i in range(200)]
        want_pool = LO.index_lookup(pool, terms, 5)
        idx = rng.randint(len(pool), size=B)
        x = _rows(pool, 64)[torch.from_numpy(idx).cuda()]
        assert lib.b200feat_index_lookup(x.data_ptr(), 64, B, layer.slots.data_ptr(), layer.terms.data_ptr(),
                                         layer.slots.shape[0], layer.V, layer.Wv, 5, out.data_ptr(), _stream()) == 0, _err()
        want = want_pool[idx]
    else:
        vals = (rng.standard_normal(B) * 30).astype(np.float32)
        if op == "log_round":
            vals = np.abs(vals) * 1000
            assert lib.b200feat_log_round(torch.from_numpy(vals).cuda().data_ptr(), 1, B, 9, -1, 1, 3.0,
                                          out.data_ptr(), _stream()) == 0, _err()
        else:
            assert lib.b200feat_round_identity(torch.from_numpy(vals).cuda().data_ptr(), 1, B, 17, 99,
                                               out.data_ptr(), _stream()) == 0, _err()
            want = LO.round_identity(vals, 17, 99)
    torch.cuda.synchronize()
    assert lib.b200feat_launch_count() == launches + 1
    assert _untouched(buf[B:])
    got = out.cpu().numpy()
    if op == "log_round":
        _log_round_check(got, vals, 9, -1, 3.0)
    else:
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, "first wrong sample %d of %d: %d != %d" % (bad[0], B, got[bad[0]], want[bad[0]])


# ----------------------------------------------------------------------------------- LogRound / RoundIdentity
def _float_specials():
    f = np.float32
    return np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, np.finfo(f).tiny, np.finfo(f).max,
                     -np.finfo(f).max, 0.5, 1.5, 2.5, -0.5, -1.5, 1.0, 2.0 ** 62, 2.0 ** 63, 2.0 ** 64, 1e30,
                     np.nextafter(f(0.5), f(0)), np.nextafter(f(0.5), f(1))], dtype=f)


@pytest.mark.parametrize("base", [None, 2, 10, 0.5, 3.7, 0, 1])
@pytest.mark.parametrize("dtype", ["float32", "float64", "int64", "int32"])
def test_log_round_against_the_oracle(base, dtype):
    from elasticdl_b200.preprocessing import LogRound

    rng = np.random.RandomState(17)
    if dtype.startswith("float"):
        vals = np.concatenate([_float_specials(), np.exp(rng.uniform(-30, 60, 20000)).astype(np.float32),
                               rng.uniform(-5, 5, 2000).astype(np.float32)]).astype(dtype)
        exact = [2.0 ** k for k in range(-20, 60)] if base in (2, 0.5) else [10.0 ** k for k in range(0, 11)] \
            if base == 10 else []
    else:
        lim = np.iinfo(dtype)
        vals = np.concatenate([[0, 1, -1, lim.min, lim.max], rng.randint(1, 1 << 20, 5000),
                               np.exp(rng.uniform(0, np.log(float(lim.max)) - 1, 5000))]).astype(dtype)
        exact = [2 ** k for k in range(0, 31)] if base in (2, 0.5) else [10 ** k for k in range(0, 10)] \
            if base == 10 else []
    vals = np.concatenate([np.asarray(exact, dtype=dtype), vals]) if exact else vals
    x = torch.from_numpy(vals).cuda()
    for num_bins, dflt in ((20, 0), (1 << 40, -5), (0, 3), (-4, 7)):
        got = LogRound(num_bins, dflt, base)(x).cpu().numpy()
        _log_round_check(got, vals, num_bins, dflt, base, strict=range(len(exact)))
    got = LogRound(64, -1, base)(x.view(2, -1) if len(vals) % 2 == 0 else x[None]).cpu().numpy().reshape(-1)
    _log_round_check(got, vals, 64, -1, base, strict=range(len(exact)))


@pytest.mark.parametrize("dtype", ["float32", "float64", "float16", "int64", "int32"])
def test_round_identity_against_the_oracle(dtype):
    from elasticdl_b200.preprocessing import RoundIdentity

    rng = np.random.RandomState(23)
    if dtype.startswith("float"):
        half = np.arange(-10, 40, dtype=np.float32) + np.float32(0.5)
        vals = np.concatenate([_float_specials(), half, (rng.standard_normal(20000) * 50).astype(np.float32),
                               np.array([0.49999997, 1e-8, 2.0 ** 24 + 2, 2.0 ** 53], dtype=np.float32)]).astype(dtype)
        if dtype == "float64":
            vals = np.concatenate([vals, [0.50000000001, 2.4999999999, 1e300, -1e300]])
    else:
        lim = np.iinfo(dtype)
        vals = np.concatenate([[0, 1, -1, lim.min, lim.max, 9, 10], rng.randint(-50, 50, 5000)]).astype(dtype)
    x = torch.from_numpy(vals).cuda()
    for nb, dflt in ((10, 0), (40, -3), (1 << 62, 5), (0, 1), (-1, -2)):
        got = RoundIdentity(nb, dflt)(x).cpu().numpy()
        want = LO.round_identity(vals.astype(np.float32) if dtype in ("float64", "float16") else vals, nb, dflt)
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, "nb=%d: first wrong value %r: %d != %d" % (nb, vals[bad[0]], got[bad[0]], want[bad[0]])


# ------------------------------------------------------------------------------------------------ census
def _census_want(raw_num, raw):
    """The layer-by-layer composition: lookup / hash / discretize plus get_id_boundaries offsets."""
    from elasticdl_b200.workloads import census_features as C

    rows = []
    for g in C.census_groups():
        if g["kind"] == "lookup":
            v = LO.index_lookup(raw[g["column"]], g["vocabulary"], 1)
        elif g["kind"] == "hash":
            v = FO.hashing(raw[g["column"]], g["num_bins"])
        else:
            v = FO.discretize(raw_num[g["column"]], g["bins"])
        rows.append(v + g["offset"])
    return np.stack(rows)


@functools.lru_cache(maxsize=4)
def _census_batch(B, seed):
    from elasticdl_b200.workloads import census_features as C

    num, strings, raw_num, raw = C.synthetic_raw_batch(B, seed, "cuda")
    return num, strings, _census_want(raw_num, raw)


@pytest.mark.parametrize("ids_dtype", [torch.int64, torch.int32], ids=["ids64", "ids32"])
@pytest.mark.parametrize("shape", SHAPES)
def test_census_transform_equals_the_layer_composition(shape, ids_dtype):
    from elasticdl_b200.workloads import census_features as C

    ft = C.census_transform(ids_dtype)
    assert ft.G == 12 and ft.max_ids == [9, 16, 22, 28, 30, 38, 45, 75, 6, 9, 15, 115]
    B = _batch(shape, 12)
    buf, ids = _poisoned(12 * B, ids_dtype)
    for seed in (0, 1):
        num, strings, want = _census_batch(B, seed)
        got, dense = ft(num, strings, ids_out=ids.view(12, B))
        torch.cuda.synchronize()
        assert dense is None and _untouched(buf[12 * B:])
        got = got.cpu().numpy().astype(np.int64)
        bad = np.argwhere(got != want)
        assert bad.size == 0, "first wrong id at (group, sample) %s: %d != %d" % (
            tuple(bad[0]), got[tuple(bad[0])], want[tuple(bad[0])])
        assert got.min() >= 0 and (got.max(1) < np.array(ft.max_ids)).all()


def test_census_transform_replays_from_a_cuda_graph():
    from elasticdl_b200.workloads import census_features as C

    B = 4096
    ft = C.census_transform(torch.int32)
    num0, strings0, _ = _census_batch(B, 5)
    num, strings = num0.clone(), strings0.clone()
    ids = torch.empty((12, B), dtype=torch.int32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ft(num, strings, ids_out=ids)  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ft(num, strings, ids_out=ids)
    for seed in (6, 7):
        n2, s2, want = _census_batch(B, seed)
        num.copy_(n2)
        strings.copy_(s2)
        ids.fill_(IDS_SENTINEL)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(ids.cpu().numpy().astype(np.int64), want)


# ---------------------------------------------------------------------------------------------- mixed
@pytest.mark.parametrize("numeric_dtype", [torch.int64, torch.float32], ids=["int64", "float32"])
@pytest.mark.parametrize("ids_dtype", [torch.int64, torch.int32], ids=["ids64", "ids32"])
def test_mixed_transform_new_and_old_kinds_with_normalizer(ids_dtype, numeric_dtype):
    """dac_ctr-style discretize / hash / hash_int groups and Normalizer columns in the same launch as lookup /
    log_round / round_identity groups, against each layer's oracle."""
    from elasticdl_b200.preprocessing import FeatureTransform

    rng = np.random.RandomState(31)
    B = 3 * _pass(14 + 3) + 17
    n_num = 3
    if numeric_dtype == torch.int64:
        num = np.stack([rng.randint(-100, 1 << 20, B), np.exp(rng.uniform(0, 40, B)).astype(np.int64),
                        rng.randint(-5, 70, B)]).astype(np.int64)
    else:
        num = np.stack([(rng.standard_normal(B) * 1e3), np.exp(rng.uniform(-10, 40, B)),
                        rng.uniform(-5, 70, B)]).astype(np.float32)
        num[2, :64] = np.arange(64) - 10.5  # ties
    v1, v2 = list(_vocab(300, 1)), [b"Male", b"Female", b""]
    pool = list(v1[:200]) + v2 + [b"x%d" % i for i in range(300)]
    idx = rng.randint(len(pool), size=(2, B))
    mat = _rows(pool, 64)
    strings = torch.stack([mat[torch.from_numpy(idx[0]).cuda()], mat[torch.from_numpy(idx[1]).cuda()]])
    groups = [{"kind": "discretize", "column": 0, "bins": [-10.0, 0.0, 5.5, 1000.0], "offset": 3},
              {"kind": "lookup", "column": 1, "vocabulary": v1, "num_oov_tokens": 7, "offset": 100},
              {"kind": "hash", "column": 0, "num_bins": 1000003},
              {"kind": "log_round", "column": 1, "num_bins": 30, "default_value": 0, "base": 2, "offset": 9},
              {"kind": "round_identity", "column": 2, "num_buckets": 50, "default_value": 51},
              {"kind": "lookup", "column": 0, "vocabulary": v2, "num_oov_tokens": 0, "offset": 1},
              {"kind": "log_round", "column": 1, "num_bins": 100, "default_value": -1},
              {"kind": "lookup", "column": 1, "vocabulary": v2, "num_oov_tokens": 1},
              {"kind": "round_identity", "column": 0, "num_buckets": 1 << 20, "default_value": 0, "offset": 5}]
    if numeric_dtype == torch.int64:
        groups.append({"kind": "hash_int", "column": 2, "num_bins": 97, "offset": 4})
    dense = [(2, 0.5, 3.0), (0, -1.0, 7.0), (1, 0.0, 1e3)]
    ft = FeatureTransform(groups, dense, ids_dtype)
    G = len(groups)
    buf, ids = _poisoned(G * B, ids_dtype)
    got, d = ft(torch.from_numpy(num).cuda(), strings, ids_out=ids.view(G, B))
    torch.cuda.synchronize()
    assert _untouched(buf[G * B:])
    got = got.cpu().numpy().astype(np.int64)
    sp = [[pool[i] for i in idx[0]], [pool[i] for i in idx[1]]]
    for g, spec in enumerate(groups):
        off = spec.get("offset", 0)
        k, c = spec["kind"], spec["column"]
        if k == "log_round":
            _log_round_check(got[g] - off, num[c], spec["num_bins"], spec["default_value"], spec.get("base"))
            continue
        if k == "discretize":
            want = FO.discretize(num[c], spec["bins"])
        elif k == "lookup":
            want = LO.index_lookup(sp[c], spec["vocabulary"], spec["num_oov_tokens"])
        elif k == "hash":
            want = FO.hashing(sp[c], spec["num_bins"])
        elif k == "hash_int":
            want = FO.hashing(num[c], spec["num_bins"])
        else:
            want = LO.round_identity(num[c], spec["num_buckets"], spec["default_value"])
        bad = np.flatnonzero(got[g] != want + off)
        assert bad.size == 0, "group %d (%s): first wrong sample %d: %d != %d" % (g, k, bad[0], got[g][bad[0]],
                                                                                  want[bad[0]] + off)
    want_dense = np.stack([FO.normalize(num[c], s, dv) for c, s, dv in dense], 1).astype(np.float32)
    assert np.array_equal(d.cpu().numpy(), want_dense)


# ------------------------------------------------------------------------------------------------ refusals
def _raw_ext(groups, exts, n_numeric=2, numeric_is_float=0, n_string=1, W=8, B=300, ids32=0, null_ext=False,
             strings=True):
    """b200feat_transform_ext into poisoned outputs: (rc, message, launches made, outputs untouched)."""
    from elasticdl_b200.preprocessing.layers import FeatureGroup, FeatureGroupExt

    G = len(groups)
    ga, ea = (FeatureGroup * G)(), (FeatureGroupExt * G)()
    for g, (spec, ext) in enumerate(zip(groups, exts)):
        ga[g].kind, ga[g].column = spec.get("kind", 3), spec.get("column", 0)
        ga[g].num_bins, ga[g].offset = spec.get("num_bins", 1), spec.get("offset", 0)
        for k, v in ext.items():
            setattr(ea[g], k, v)
    numeric = torch.zeros((n_numeric, B), dtype=torch.float32 if numeric_is_float else torch.int64, device="cuda")
    s = torch.full((max(n_string, 1), B, W), 65, dtype=torch.uint8, device="cuda")
    ibuf, ids = _poisoned(G * B, torch.int32 if ids32 else torch.int64)
    lib = _lib()
    n = lib.b200feat_launch_count()
    rc = lib.b200feat_transform_ext(ga, None if null_ext else ea, G, None, 0, None, 0, numeric.data_ptr(), n_numeric,
                                    numeric_is_float, s.data_ptr() if strings else None, n_string if strings else 0, W,
                                    B, ids.data_ptr(), ids32, None, _stream())
    msg = _err()
    torch.cuda.synchronize()
    return rc, msg, lib.b200feat_launch_count() - n, _untouched(ibuf)


@functools.lru_cache(None)
def _table():
    from elasticdl_b200.preprocessing import IndexLookup

    return IndexLookup(["a", "bb", "ccc"])


def _ext(**kw):
    t = _table()
    e = dict(slots_dev=t.slots.data_ptr(), terms_dev=t.terms.data_ptr(), n_slots=t.slots.shape[0], V=t.V, Wv=t.Wv)
    e.update(kw)
    return e


LOOKUP = {"kind": 3, "column": 0, "num_bins": 1}
EXT_REFUSALS = {
    "null_slots": (dict(groups=[LOOKUP], exts=[{"slots_dev": None}]), "null table"),
    "null_terms": (dict(groups=[LOOKUP], exts=[{"terms_dev": None}]), "null table"),
    "n_slots_not_pow2": (dict(groups=[LOOKUP], exts=[{"n_slots": 6}]), "power of two"),
    "n_slots_below_2V": (dict(groups=[LOOKUP], exts=[{"n_slots": 4}]), "power of two"),
    "V_0": (dict(groups=[LOOKUP], exts=[{"V": 0}]), "vocabulary size"),
    "Wv_0": (dict(groups=[LOOKUP], exts=[{"Wv": 0}]), "Wv"),
    "Wv_65": (dict(groups=[LOOKUP], exts=[{"Wv": 65}]), "Wv"),
    "num_oov_negative": (dict(groups=[dict(LOOKUP, num_bins=-1)], exts=[{}]), "num_oov_tokens"),
    "bad_string_column": (dict(groups=[dict(LOOKUP, column=1)], exts=[{}]), "bad string column"),
    "lookup_on_numeric_column": (dict(groups=[LOOKUP], exts=[{}], strings=False), "bad string column"),
    "log_round_bad_column": (dict(groups=[{"kind": 4, "column": 2, "num_bins": 5}], exts=[{}]), "bad numeric column"),
    "round_identity_bad_column": (dict(groups=[{"kind": 5, "column": -1, "num_bins": 5}], exts=[{}]),
                                  "bad numeric column"),
    "lookup_with_null_ext": (dict(groups=[LOOKUP], exts=[{}], null_ext=True), "unknown group kind"),
    "log_round_with_null_ext": (dict(groups=[{"kind": 4, "num_bins": 5}], exts=[{}], null_ext=True), "unknown group kind"),
    "round_identity_with_null_ext": (dict(groups=[{"kind": 5, "num_bins": 5}], exts=[{}], null_ext=True),
                                     "unknown group kind"),
    "kind_6": (dict(groups=[{"kind": 6}], exts=[{}]), "unknown group kind"),
    "int32_default_value": (dict(groups=[{"kind": 4, "num_bins": 5}], exts=[{"default_value": 1 << 31}], ids32=1),
                            "int32"),
    "int32_negative_default_value": (dict(groups=[{"kind": 5, "num_bins": 5}],
                                          exts=[{"default_value": -(1 << 31) - 1}], ids32=1), "int32"),
    "int32_no_oov_minus_one": (dict(groups=[dict(LOOKUP, num_bins=0, offset=-(1 << 31))], exts=[{}], ids32=1), "int32"),
    "int32_lookup_top": (dict(groups=[dict(LOOKUP, num_bins=(1 << 31) - 2)], exts=[{}], ids32=1), "int32"),
}


@pytest.mark.parametrize("case", list(EXT_REFUSALS), ids=list(EXT_REFUSALS))
def test_transform_ext_refusals_name_the_cause_and_launch_nothing(case):
    kw, cause = EXT_REFUSALS[case]
    kw = dict(kw, exts=[_ext(**e) for e in kw["exts"]])
    rc, msg, launched, untouched = _raw_ext(**kw)
    assert rc == -1 and cause in msg, (rc, msg)
    assert launched == 0 and untouched


def test_transform_ext_int32_limits_accept_the_largest_fitting_groups():
    for kw in (dict(groups=[dict(LOOKUP, num_bins=0, offset=-(1 << 31) + 1)], exts=[_ext()]),
               dict(groups=[dict(LOOKUP, num_bins=(1 << 31) - 3)], exts=[_ext()]),
               dict(groups=[{"kind": 4, "num_bins": 5}], exts=[_ext(default_value=(1 << 31) - 1)]),
               dict(groups=[{"kind": 5, "num_bins": 5, "offset": 3}], exts=[_ext(default_value=-(1 << 31) - 3)])):
        rc, msg, launched, untouched = _raw_ext(ids32=1, **kw)
        assert rc == 0 and launched == 1 and not untouched, msg


def test_layer_and_transform_refusals_on_inputs():
    from elasticdl_b200.preprocessing import FeatureTransform, IndexLookup, LogRound, RoundIdentity

    lib = _lib()
    layer = IndexLookup(["a", "b"])
    n = lib.b200feat_launch_count()
    with pytest.raises(TypeError, match="string"):
        layer(torch.zeros(4, dtype=torch.int64, device="cuda"))
    with pytest.raises(TypeError, match="string"):
        layer(torch.zeros((4, 3), dtype=torch.int32, device="cuda"))
    # empty batches: empty outputs, no launch
    assert layer(torch.zeros((0, 5), dtype=torch.uint8, device="cuda")).shape == (0,)
    assert layer(torch.zeros((3, 0, 5), dtype=torch.uint8, device="cuda")).shape == (3, 0)
    assert LogRound(4)(torch.zeros((2, 0), device="cuda")).shape == (2, 0)
    assert RoundIdentity(4)(torch.zeros((0,), dtype=torch.int64, device="cuda")).shape == (0,)
    ft = FeatureTransform([{"kind": "lookup", "column": 0, "vocabulary": ["a"]}, {"kind": "log_round", "column": 0,
                                                                                  "num_bins": 3}])
    ids, _ = ft(torch.zeros((1, 0), device="cuda"), torch.zeros((1, 0, 4), dtype=torch.uint8, device="cuda"))
    assert ids.shape == (2, 0)
    assert lib.b200feat_launch_count() == n
    # an input on another device from the table
    moved = IndexLookup(["a", "b"]).to("cpu")
    assert moved.slots.device.type == "cpu"
    with pytest.raises(ValueError, match="device|on cpu"):
        moved(torch.zeros((4, 3), dtype=torch.uint8, device="cuda"))
    ft_cpu = FeatureTransform([{"kind": "lookup", "column": 0, "vocabulary": ["a"]}], device="cpu")
    with pytest.raises(ValueError, match="vocabulary tables"):
        ft_cpu(torch.zeros((1, 4), device="cuda"), torch.zeros((1, 4, 4), dtype=torch.uint8, device="cuda"))
    if torch.cuda.device_count() > 1:
        other = IndexLookup(["a"]).to("cuda:1")
        with pytest.raises(ValueError):
            other(torch.zeros((4, 3), dtype=torch.uint8, device="cuda:0"))
    assert lib.b200feat_launch_count() == n
    # .to(device) moves the table correctly: the copy answers like the original
    back = moved.to("cuda")
    x = torch.tensor([[97, 0, 0], [98, 0, 0], [99, 0, 0]], dtype=torch.uint8, device="cuda")
    assert back(x).tolist() == [0, 1, 2]
    with pytest.raises(ValueError, match="int32"):
        FeatureTransform([{"kind": "lookup", "column": 0, "vocabulary": ["a"], "num_oov_tokens": 0,
                           "offset": -(1 << 31)}], ids_dtype=torch.int32)
    with pytest.raises(ValueError, match="int32"):
        FeatureTransform([{"kind": "round_identity", "column": 0, "num_buckets": 3, "default_value": 1 << 31}],
                         ids_dtype=torch.int32)
