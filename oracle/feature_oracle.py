"""CPU oracle of the feature-id generation layers -- TEST INFRASTRUCTURE (see ps_oracle.py's header:
only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import anything under oracle/).

Follows (paths relative to /root/reference/):
  * elasticdl_preprocessing/layers/hashing.py:61-92       Hashing: tf.as_string for ints, then
        tf.strings.to_hash_bucket_fast = FarmHash Fingerprint64(bytes) % num_bins (unsigned)
  * elasticdl_preprocessing/layers/discretization.py:60-78 Discretization: math_ops._bucketize =
        std::upper_bound over the float32 boundaries (bins include their left boundary), cast to int64
  * elasticdl_preprocessing/layers/concatenate_with_offset.py:50-87
  * elasticdl_preprocessing/layers/normalizer.py          (x - subtractor) / divisor in float64
  * model_zoo/dac_ctr/feature_transform.py:36-118         their composition

Third-party arithmetic: Fingerprint64 lives in TensorFlow (tensorflow==2.5.2, elasticdl/requirements.txt:6;
tensorflow/core/platform/fingerprint.h -> FarmHash 1.1 farmhashna::Hash64), not under /root/reference.
It is restated below from the published algorithm for lengths 0..64 bytes.
PINNING: the reference's only stored vector (hashing.py:35-39 / hashing_test.py:27-31: 'A'..'E' with
3 bins -> [1, 0, 1, 1, 2]) pins the 1..3-byte branch; the 4..64-byte branches are PARITY UNPINNED
offline (no TensorFlow here) -- tests/test_oracle_features.py says so too.
"""
import numpy as np

_M = (1 << 64) - 1
K0, K1, K2 = 0xC3A5C85C97CB3127, 0xB492B66FBE98F273, 0x9AE16A3B2F90404F


def _rot(v, s):
    return v if s == 0 else ((v >> s) | (v << (64 - s))) & _M


def _f64(s, i):
    return int.from_bytes(s[i:i + 8], "little")


def _f32(s, i):
    return int.from_bytes(s[i:i + 4], "little")


def _hash_len16(u, v, mul):
    a = ((u ^ v) * mul) & _M
    a ^= a >> 47
    b = ((v ^ a) * mul) & _M
    b ^= b >> 47
    return (b * mul) & _M


def fingerprint64(s):
    """FarmHash Fingerprint64 (farmhashna::Hash64) of a bytes object of at most 64 bytes."""
    s = bytes(s)
    n = len(s)
    if n > 64:
        raise ValueError("strings longer than 64 bytes are not supported")
    if n <= 16:
        if n >= 8:
            mul = (K2 + n * 2) & _M
            a = (_f64(s, 0) + K2) & _M
            b = _f64(s, n - 8)
            c = (_rot(b, 37) * mul + a) & _M
            d = ((_rot(a, 25) + b) * mul) & _M
            return _hash_len16(c, d, mul)
        if n >= 4:
            mul = (K2 + n * 2) & _M
            a = _f32(s, 0)
            return _hash_len16((n + (a << 3)) & _M, _f32(s, n - 4), mul)
        if n > 0:
            a, b, c = s[0], s[n >> 1], s[n - 1]
            y = (a + (b << 8)) & 0xFFFFFFFF
            z = (n + (c << 2)) & 0xFFFFFFFF
            v = ((y * K2) & _M) ^ ((z * K0) & _M)
            return ((v ^ (v >> 47)) * K2) & _M
        return K2
    mul = (K2 + n * 2) & _M
    if n <= 32:
        a = (_f64(s, 0) * K1) & _M
        b = _f64(s, 8)
        c = (_f64(s, n - 8) * mul) & _M
        d = (_f64(s, n - 16) * K2) & _M
        return _hash_len16((_rot((a + b) & _M, 43) + _rot(c, 30) + d) & _M, (a + _rot((b + K2) & _M, 18) + c) & _M, mul)
    a = (_f64(s, 0) * K2) & _M
    b = _f64(s, 8)
    c = (_f64(s, n - 8) * mul) & _M
    d = (_f64(s, n - 16) * K2) & _M
    y = (_rot((a + b) & _M, 43) + _rot(c, 30) + d) & _M
    z = _hash_len16(y, (a + _rot((b + K2) & _M, 18) + c) & _M, mul)
    e = (_f64(s, 16) * mul) & _M
    f = _f64(s, 24)
    g = ((y + _f64(s, n - 32)) * mul) & _M
    h = ((z + _f64(s, n - 24)) * mul) & _M
    return _hash_len16((_rot((e + f) & _M, 43) + _rot(g, 30) + h) & _M, (e + _rot((f + a) & _M, 18) + g) & _M, mul)


def _to_bytes(v):
    if isinstance(v, (bytes, bytearray, np.bytes_)):
        return bytes(v)
    if isinstance(v, str):
        return v.encode("utf-8")
    return str(int(v)).encode("ascii")  # tf.as_string(int): plain decimal, '-' for negatives


def hashing(values, num_bins):
    """Hashing(num_bins)(values): same shape, int64 (hashing.py:61-92)."""
    if num_bins is None or num_bins <= 0:
        raise ValueError("`num_bins` cannot be `None` or non-positive values.")
    arr = np.asarray(values, dtype=object)
    out = np.empty(arr.shape, dtype=np.int64)
    flat_in, flat_out = arr.reshape(-1), out.reshape(-1)
    for i, v in enumerate(flat_in):
        flat_out[i] = fingerprint64(_to_bytes(v)) % num_bins
    return out


def discretize(values, bins):
    """Discretization(bins)(values): id = number of boundaries <= x, compared in float32 for every input.
    The layer is a Keras Layer of the default float32 dtype policy: its __call__ autocasts floating inputs
    (float64 and Python floats too) to float32, and BucketizeOp<int64> compares `int64 < float boundary` in
    float (std::upper_bound with float boundaries).  Unsorted (or NaN) boundaries are refused, as Bucketize
    refuses them."""
    b = np.asarray(bins, dtype=np.float32).reshape(-1)
    if np.isnan(b).any() or np.any(b[1:] < b[:-1]):
        raise ValueError("boundaries must be sorted in ascending order")
    xf = np.asarray(values).astype(np.float32)
    return np.searchsorted(b, xf, side="right").astype(np.int64)


def concatenate_with_offset(inputs, offsets, axis=-1):
    """ConcatenateWithOffset(offsets, axis)(inputs) for dense tensors (concatenate_with_offset.py:50-87)."""
    if offsets is None:
        return np.concatenate([np.asarray(t) for t in inputs], axis=axis)
    if len(offsets) != len(inputs):
        raise ValueError("The offsets length is not equal to inputs length")
    return np.concatenate([np.asarray(t) + o for t, o in zip(inputs, offsets)], axis=axis)


def normalize(values, subtractor, divisor):
    """Normalizer(subtractor, divisor)(values): float64 (normalizer.py)."""
    if divisor == 0:
        raise ValueError("The divisor cannot be 0")
    return (np.asarray(values, dtype=np.float64) - subtractor) / divisor
