"""CPU tests of the feature-id oracle (oracle/feature_oracle.py) against every vector the reference holds
for the preprocessing layers of SURVEY.md section 8f-3.  Fingerprint64 is third-party arithmetic
(TensorFlow / FarmHash): the 1..3-byte branch is pinned by the reference's vector; the 4..64-byte
branches are PARITY UNPINNED offline (restated from the published algorithm)."""
import numpy as np
import pytest

from oracle import feature_oracle as FO


def test_hashing_py_35_39_example_vector():
    # elasticdl_preprocessing/layers/hashing.py:35-39, tests/hashing_test.py:27-31
    out = FO.hashing(np.asarray([["A"], ["B"], ["C"], ["D"], ["E"]]), 3)
    assert out.dtype == np.int64 and np.array_equal(out, [[1], [0], [1], [1], [2]])


def test_fingerprint64_known_answers():
    assert FO.fingerprint64(b"") == 0x9AE16A3B2F90404F  # k2: farmhashna::HashLen0to16 of the empty string
    # pyfarmhash README (farmhash.hash64('abc')), recalled -- a second anchor of the 1..3-byte branch
    assert FO.fingerprint64(b"abc") == 2640714258260161385
    with pytest.raises(ValueError):
        FO.fingerprint64(b"x" * 65)


def test_hashing_ints_go_through_decimal_strings():
    # hashing.py:63-72: integer inputs -> tf.as_string -> the same hash as the string
    vals = np.array([0, 7, -3, 1234567890123, 42], dtype=np.int64)
    want = FO.hashing([str(int(v)) for v in vals], 1000)
    assert np.array_equal(FO.hashing(vals, 1000), want)
    with pytest.raises(ValueError):
        FO.hashing(vals, 0)


def test_discretization_test_py_26_31():
    out = FO.discretize([[0.2], [1.6], [4.2], [6.1], [10.9]], [1, 5, 10])
    assert out.dtype == np.int64 and np.array_equal(out, [[0], [1], [1], [2], [3]])
    # bins include their left boundary (discretization.py:33-36)
    assert np.array_equal(FO.discretize([0.0, 1.0, 1.5, 2.0, -1.0], [0.0, 1.0, 2.0]), [1, 2, 2, 3, 0])
    # repeated boundaries (dac_ctr I2: [-1, 0, 1, 1, 3, ...]) are legal for upper_bound
    assert np.array_equal(FO.discretize([1, 2], [-1.0, 0.0, 1.0, 1.0, 3.0]), [4, 4])


def test_concatenate_with_offset_test_py_27_34():
    a1, a2 = np.array([[1], [1], [1]]), np.array([[2], [2], [2]])
    assert np.array_equal(FO.concatenate_with_offset([a1, a2], [0, 10], axis=1), [[1, 12], [1, 12], [1, 12]])
    with pytest.raises(ValueError):
        FO.concatenate_with_offset([a1, a2], [0], axis=1)


def test_normalizer_example():
    assert np.allclose(FO.normalize([[3.0], [5.0], [7.0]], 1.0, 2.0), [[1.0], [2.0], [3.0]])  # normalizer.py docstring
    with pytest.raises(ValueError):
        FO.normalize([1.0], 0.0, 0)


def test_discretize_compares_every_input_in_float32():
    # the reference layer's Keras __call__ autocasts floating inputs to its float32 compute dtype, so a float64
    # value next to a boundary rounds onto it before math_ops._bucketize sees it
    x64 = np.array([0.99999999, np.nextafter(1.0, 0.0), 1.0, np.nextafter(1.0, 2.0), 0.9999999], dtype=np.float64)
    assert np.array_equal(FO.discretize(x64, [1.0]), [1, 1, 1, 1, 0])
    assert np.array_equal(FO.discretize(x64.astype(np.float32), [1.0]), [1, 1, 1, 1, 0])
    assert np.array_equal(FO.discretize([0.99999999], [1.0]), [1])  # Python floats are float32 tensors too
    assert np.array_equal(FO.discretize(np.array([0.1]), [0.1]), [1])  # both round to float32(0.1)
    # int64 values round to float32 before the comparison: 16777217 -> 16777216.0f, 16777219 -> 16777220.0f
    ints = np.array([16777215, 16777216, 16777217, 16777218, 16777219], dtype=np.int64)
    assert np.array_equal(FO.discretize(ints, [16777216.0]), [0, 1, 1, 1, 1])
    assert np.array_equal(FO.discretize(ints, [16777217.0, 16777220.0]), [0, 1, 1, 1, 2])
    assert np.array_equal(FO.discretize(ints.astype(np.int32), [16777217.0]), [0, 1, 1, 1, 1])
    # NaN sorts past every boundary (upper_bound: NaN < b is false), -0.0 == 0.0 lands right of a 0 boundary
    for dt in (np.float32, np.float64):
        v = np.array([np.nan, -0.0, 0.0, -np.inf, np.inf], dtype=dt)
        assert np.array_equal(FO.discretize(v, [-1.0, 0.0, 1.0]), [3, 2, 2, 0, 3])
    assert np.array_equal(FO.discretize([1.5, -3.0], []), [0, 0])


def test_discretize_refuses_unsorted_boundaries():
    with pytest.raises(ValueError, match="sorted"):
        FO.discretize([1.0], [0.0, 2.0, 1.0])
    with pytest.raises(ValueError, match="sorted"):
        FO.discretize([1.0], [0.0, np.nan])
    # repeated boundaries and -0.0 next to 0.0 are sorted
    assert np.array_equal(FO.discretize([0.0, 1.0], [-0.0, 0.0, 1.0, 1.0]), [2, 4])
