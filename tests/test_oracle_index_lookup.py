"""CPU tests of IndexLookup / LogRound / RoundIdentity: the oracle (oracle/lookup_oracle.py) against the
reference's literal vectors and at its edges, the host vocabulary-table builder (b200feat_vocab_build) against
the layout include/b200_features.h documents, and the layer refusals that come before any device allocation."""
import collections
import ctypes
import os

import numpy as np
import pytest

from oracle import feature_oracle as FO
from oracle import lookup_oracle as LO

ABC = ["A", "B", "C"]


# ------------------------------------------------------------------------------------- reference vectors
def test_index_lookup_reference_vectors(tmp_path):
    # index_lookup_test.py:55-75: dense [[A],[B],[C],[D],[E]] -> [[0],[1],[2],[3],[3]]; ragged / sparse flat values
    assert LO.index_lookup([["A"], ["B"], ["C"], ["D"], ["E"]], ABC).tolist() == [[0], [1], [2], [3], [3]]
    assert LO.index_lookup(["A", "B", "C", "D", "E"], ABC).tolist() == [0, 1, 2, 3, 3]
    # test_model_with_lookup: A, C, B, D, E -> 0, 2, 1, 3, 3
    assert LO.index_lookup([["A"], ["C"], ["B"], ["D"], ["E"]], ABC).tolist() == [[0], [2], [1], [3], [3]]
    # the file form (index_lookup_test.py:34-42) reads the same vocabulary
    from elasticdl_b200.preprocessing.layers import read_vocabulary_file

    path = tmp_path / "vocab_test.txt"
    path.write_text("A\nB\nC\n")
    assert read_vocabulary_file(str(path)) == ABC
    assert LO.index_lookup(list("ABCDE"), read_vocabulary_file(str(path))).tolist() == [0, 1, 2, 3, 3]


def test_log_round_reference_vectors():
    # log_round_test.py:27-50 (num_bins=20, base=2)
    assert LO.log_round([[0.0], [2.6], [0.2], [3.1], [1024]], 20, base=2).tolist() == [[0], [1], [0], [2], [10]]
    assert LO.log_round([1.1, 3.4, 1025], 20, base=2).tolist() == [0, 2, 10]
    assert LO.log_round([1.2, 2.6, 0.2, 3.1, 1024], 20, base=2).tolist() == [0, 1, 0, 2, 10]
    # log_round.py:34-40 docstring (num_bins=16, base=2)
    assert LO.log_round([[1.2], [1.6], [0.2], [3.1], [100]], 16, base=2).tolist() == [[0], [1], [0], [2], [7]]


def test_round_identity_reference_vectors():
    # round_identity_test.py:27-40 (num_buckets=10): 0.5 rounds half to even -> 0
    assert LO.round_identity([[1.2], [1.6], [0.2], [3.1], [4.9]], 10).tolist() == [[1], [2], [0], [3], [5]]
    assert LO.round_identity([1.1, 3.4, 0.5], 10).tolist() == [1, 3, 0]


# ------------------------------------------------------------------------------------------- oracle edges
@pytest.mark.parametrize("n_oov", [0, 1, 3])
def test_index_lookup_oov_buckets(n_oov):
    vals = ["A", "C", "", "D", "E", "AB", "a", "A\x00zz", "B\x00"]
    got = LO.index_lookup(vals, ABC, n_oov)
    assert got[[0, 1, 7, 8]].tolist() == [0, 2, 0, 1]  # bytes after a NUL are ignored
    for i in (2, 3, 4, 5, 6):
        b = vals[i].encode()
        assert got[i] == (3 + FO.fingerprint64(b) % n_oov if n_oov else -1)
    assert LO.index_lookup([""], ["x", ""], n_oov).tolist() == [1]


def test_index_lookup_oracle_refusals():
    with pytest.raises(ValueError, match="repeated"):
        LO.index_lookup(["A"], ["A", "B", "A"])
    with pytest.raises(ValueError, match="non-empty"):
        LO.index_lookup(["A"], [])
    with pytest.raises(ValueError, match="num_oov_tokens"):
        LO.index_lookup(["A"], ABC, -1)


def test_log_round_specials():
    big = 2.0 ** 63
    x = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -1.0, 1.0, np.e, 1e300], dtype=np.float64)
    # natural log: NaN / inf / log(0) = -inf / negative -> default; 1e300 autocasts to float32 inf -> default
    got = LO.log_round(x, 1000, default_value=-9)
    assert got.tolist() == [-9, -9, -9, -9, -9, -9, 0, 1, -9]
    # ties round half to even: log2(2^0.5) = 0.5 -> 0, log2(2^2.5) = 2.5 -> 2 (both quotients exact in float64)
    assert np.rint(0.5) == 0 and LO.log_round(np.array([4, 16], dtype=np.int64), 9, base=4).tolist() == [1, 2]
    # float inputs are autocast to float32 first: 1e300 -> inf -> default
    assert LO.log_round([1e300], 1 << 40, default_value=7).tolist() == [7]
    # a rounded value >= 2^63 goes to the default, the float64 just below it does not; base 1 gives +-inf
    below = np.nextafter(big, 0.0)
    assert LO._rounded_ids([big, below], (1 << 63) - 1, 5).tolist() == [5, int(below)]
    assert LO.log_round([8.0, 0.5, 1.0], 1 << 62, 5, base=1).tolist() == [5, 5, 5]
    # integer inputs go straight to float64
    assert LO.log_round(np.array([1, 2, 4, 1024, 0, -4], dtype=np.int64), 20, 3, base=2).tolist() == [0, 1, 2, 10, 3, 3]
    # num_bins <= 0: every value is the default; base 0: -0.0 quotient -> 0
    assert LO.log_round([1.0, 8.0], 0, 4, base=2).tolist() == [4, 4]
    assert LO.log_round([8.0, 0.5], 5, 4, base=0).tolist() == [0, 0]
    # exactly num_bins - 1 is in range, num_bins is not
    assert LO.log_round([2.0 ** 19, 2.0 ** 20], 20, -1, base=2).tolist() == [19, -1]


def test_round_identity_specials():
    f = np.array([np.nan, np.inf, -np.inf, 0.0, -0.0, -0.5, -0.6, 0.5, 1.5, 2.5, 9.4999, 9.5, 2.0 ** 63, 2.0 ** 62],
                 dtype=np.float32)
    assert LO.round_identity(f, 10, -3).tolist() == [-3, -3, -3, 0, 0, 0, -3, 0, 2, 2, 9, -3, -3, -3]
    assert LO.round_identity(f[-1:], (1 << 63) - 1, -3).tolist() == [1 << 62]
    i = np.array([-1, 0, 9, 10, -(1 << 63), (1 << 63) - 1], dtype=np.int64)
    assert LO.round_identity(i, 10, 77).tolist() == [77, 0, 9, 77, 77, 77]
    assert LO.round_identity([2.4, 0.0], -1, 6).tolist() == [6, 6]


# ----------------------------------------------------------------------------------------- host builder
def _lib():
    from elasticdl_b200 import _lib as L

    return L.lib()


def _build(terms, Wv=None, n_slots=None):
    from elasticdl_b200.preprocessing.layers import VOCAB_SLOT_DTYPE

    lib = _lib()
    V = len(terms)
    wv = Wv or max(max(len(t) for t in terms), 1)
    mat = np.zeros((V, wv), dtype=np.uint8)
    for i, t in enumerate(terms):
        mat[i, :len(t)] = np.frombuffer(t, dtype=np.uint8)
    n = n_slots or lib.b200feat_vocab_slots(V)
    slots = np.zeros(max(n, 1), dtype=VOCAB_SLOT_DTYPE)
    dup = ctypes.c_int64(-1)
    rc = lib.b200feat_vocab_build(mat.ctypes.data, V, wv, n, slots.ctypes.data, ctypes.byref(dup))
    return rc, slots, mat, dup.value


def _walk(slots, mat, term):
    """The documented probe, in numpy: home slot fingerprint & (n_slots - 1), linear steps, stop at index -1."""
    fp = FO.fingerprint64(term)
    mask = len(slots) - 1
    h = fp & mask
    for _ in range(len(slots)):
        s = slots[h]
        if s["index"] < 0:
            return -1
        if int(s["fingerprint"]) == fp and s["length"] == len(term) and bytes(mat[s["index"], :len(term)]) == term:
            return int(s["index"])
        h = (h + 1) & mask
    return -1


@pytest.mark.parametrize("V", [1, 2, 3, 8, 1000, 4096])
def test_vocab_build_layout_finds_every_term(V):
    from elasticdl_b200.preprocessing.layers import VOCAB_SLOT_DTYPE, VocabSlot

    assert ctypes.sizeof(VocabSlot) == VOCAB_SLOT_DTYPE.itemsize == 16
    rng = np.random.RandomState(V)
    terms = list(collections.OrderedDict.fromkeys(
        [b""] + [bytes(rng.randint(1, 256, size=rng.randint(1, 65)).astype(np.uint8)) for _ in range(V + 8)]))[:V]
    assert len(terms) == V
    n = _lib().b200feat_vocab_slots(V)
    assert n >= 2 * V and n & (n - 1) == 0 and (n // 2 < 2 * V or n == 2)
    rc, slots, mat, _ = _build(terms)
    assert rc == 0
    assert (slots["index"] >= 0).sum() == V and sorted(slots["index"][slots["index"] >= 0]) == list(range(V))
    empty = slots[slots["index"] < 0]
    assert (empty["fingerprint"] == 0).all() and (empty["length"] == 0).all()
    for i, t in enumerate(terms):
        assert _walk(slots, mat, t) == i
    for t in (b"\x01" * 65, b"not-there", b"\xff" * 64):
        if t not in terms:
            assert _walk(slots, mat, t[:64]) == -1
    rc2, slots2, mat2, _ = _build(terms)
    assert rc2 == 0 and slots.tobytes() == slots2.tobytes() and mat.tobytes() == mat2.tobytes()


def test_vocab_build_at_maximum_load():
    """V a power of two: n_slots = 2V, the largest load the layout allows."""
    terms = [b"t%d" % i for i in range(1024)]
    rc, slots, mat, _ = _build(terms)
    assert rc == 0 and len(slots) == 2048
    assert all(_walk(slots, mat, t) == i for i, t in enumerate(terms))


def test_vocab_build_refuses_duplicates_at_the_second_occurrence():
    rc, _, _, dup = _build([b"a", b"b", b"c", b"b", b"a"])
    assert rc == -1 and dup == 3 and "term 3 repeats term 1" in _lib().b200feat_last_error().decode()
    rc, _, _, dup = _build([b"", b"x", b""])
    assert rc == -1 and dup == 2


def test_vocab_build_refuses_bad_arguments():
    from elasticdl_b200.preprocessing.layers import VOCAB_SLOT_DTYPE

    lib = _lib()
    assert lib.b200feat_vocab_slots(0) == -1 and lib.b200feat_vocab_slots(1 << 31) == -1
    assert lib.b200feat_vocab_slots(1) == 2 and lib.b200feat_vocab_slots((1 << 31) - 1) == 1 << 32
    mat = np.zeros((4, 65), dtype=np.uint8)
    slots = np.zeros(64, dtype=VOCAB_SLOT_DTYPE)

    def call(V, Wv, n, m=mat, s=slots):
        rc = lib.b200feat_vocab_build(m.ctypes.data if m is not None else None, V, Wv, n,
                                      s.ctypes.data if s is not None else None, None)
        return rc, lib.b200feat_last_error().decode()

    for kw, cause in [((0, 4, 8), "V must be"), ((1 << 31, 4, 1 << 33), "V must be"), ((4, 0, 8), "Wv"),
                      ((4, 65, 8), "Wv"), ((4, 4, 7), "power of two"), ((4, 4, 12), "power of two"),
                      ((4, 4, 4), "power of two"), ((4, 4, 0), "power of two")]:
        rc, msg = call(*kw)
        assert rc == -1 and cause in msg, (kw, msg)
    rc, msg = call(4, 4, 8, m=None)
    assert rc == -1 and "null" in msg
    rc, msg = call(4, 4, 8, s=None)
    assert rc == -1 and "null" in msg
    bad = np.array([[65, 0, 66, 0]], dtype=np.uint8)  # a byte after the terminating NUL
    rc, msg = call(1, 4, 2, m=bad)
    assert rc == -1 and "NUL" in msg


# ------------------------------------------------------------------------------------ layer refusals
@pytest.mark.parametrize("case", ["list_dup", "file_dup", "empty", "empty_file", "65_bytes", "nul", "neg_oov"])
def test_index_lookup_layer_refusals_without_a_device(case, tmp_path):
    """Validation comes before any device allocation, so these raise on a machine without a GPU too."""
    from elasticdl_b200.preprocessing import FeatureTransform, IndexLookup

    path = str(tmp_path / "v.txt")
    kw, match = {
        "list_dup": (dict(vocabulary=["A", "B", "A", "C", "B"]), r"repeated terms are \['A', 'B'\]"),
        "file_dup": (dict(vocabulary=path), r"repeated terms are \['x'\]"),
        "empty": (dict(vocabulary=[]), "non-empty"),
        "empty_file": (dict(vocabulary=str(tmp_path / "empty.txt")), "non-empty"),
        "65_bytes": (dict(vocabulary=["a", "b" * 65]), "65 bytes"),
        "nul": (dict(vocabulary=["a", "b\x00c"]), "NUL"),
        "neg_oov": (dict(vocabulary=ABC, num_oov_tokens=-1), "num_oov_tokens"),
    }[case]
    with open(path, "w") as f:
        f.write("x\ny\n  x \n")  # stripped: a repeated "x"
    open(str(tmp_path / "empty.txt"), "w").close()
    with pytest.raises(ValueError, match=match):
        IndexLookup(**kw)
    spec = {"kind": "lookup", "column": 0, "vocabulary": kw["vocabulary"], "num_oov_tokens": kw.get("num_oov_tokens", 1)}
    with pytest.raises(ValueError, match=match):
        FeatureTransform([spec])


def test_vocabulary_file_is_read_like_the_reference(tmp_path):
    from elasticdl_b200.preprocessing import read_vocabulary_file

    path = tmp_path / "v.txt"
    path.write_bytes(b"  alpha\t\n\nbeta\r\n\xffgam\xc3\xa9\n last")
    assert read_vocabulary_file(str(path)) == ["alpha", "", "beta", "gamé", "last"]


def test_census_feature_config():
    from elasticdl_b200.workloads import census_features as C

    assert C.ID_GROUP_DIMS == {"group1": 28, "group2": 75, "group3": 115}
    groups = C.census_groups()
    assert len(groups) == 12
    assert [g["offset"] for g in groups] == [0, 9, 16, 22, 0, 30, 38, 45, 0, 6, 9, 15]
    assert [g["kind"] for g in groups] == ["lookup", "discretize", "discretize", "discretize", "hash", "lookup", "lookup",
                                           "hash", "discretize", "lookup", "lookup", "hash"]
    num, strings, raw_num, raw = C.synthetic_raw_batch(300, 0, "cpu")
    assert num.shape == (4, 300) and strings.shape == (8, 300, 32) and len(raw) == 8
    for j, name in enumerate(C.NUMERIC_FEATURE_KEYS):
        assert set(C.FEATURES[name][1]) <= set(raw_num[j].tolist())
    assert "?" in raw[0] and set(C.WORK_CLASS_VOCABULARY) <= set(raw[0])
    assert os.path.basename(C.__file__) == "census_features.py"
