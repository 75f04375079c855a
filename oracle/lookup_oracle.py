"""CPU oracle of the id-mapping preprocessing layers IndexLookup, LogRound and RoundIdentity -- TEST
INFRASTRUCTURE (see ps_oracle.py's header: only tests/, __graft_entry__.smoke() and bench.py's CPU legs may import
anything under oracle/).  Fingerprint64 and the value-to-bytes rule are feature_oracle.py's.

Follows (paths relative to /root/reference/):
  * elasticdl_preprocessing/layers/index_lookup.py:57-128  IndexLookup: index_table_from_tensor with
        num_oov_buckets = IdTableWithHashBuckets over FastHashSpec: a vocabulary term -> its position i, any
        other string -> V + Fingerprint64 % num_oov_tokens, or the table's default_value -1 with no OOV bucket.
        PINNED by index_lookup_test.py:29-75 (["A","B","C"]: A,B,C,D,E -> 0,1,2,3,3; vocab_size() == 4).
        Matching is exact on the bytes before the first NUL; repeated terms and an empty vocabulary are refused.
        Also model_zoo/census_wide_deep_model/keras_process_layer.py:55-65 (CategoryLookup, one OOV bucket).
  * elasticdl_preprocessing/layers/log_round.py:53-98     LogRound: float inputs autocast to float32 (Keras),
        then float64 log(x) [/ log(base)], tf.math.round (half to even), out-of-range -> default_value.
        PINNED by log_round_test.py:27-61 and the log_round.py:34-40 docstring example.
  * elasticdl_preprocessing/layers/round_identity.py:44-86 RoundIdentity: float32 rint (integers pass
        through), out-of-range -> default_value.  PINNED by round_identity_test.py:27-47 (0.5 -> 0); the class
        docstring's num_buckets=5 example contradicts its own rule and is not used.
For LogRound and RoundIdentity, NaN, +-inf and values >= 2^63 go to default_value: TF on x86 casts them to int64
with cvttsd2si, which gives INT64_MIN (< 0).  NO reference vector pins this (x86 cast assumption).
"""
import numpy as np

from oracle.feature_oracle import _to_bytes, fingerprint64


def _vocab_terms(vocabulary):
    terms = [_to_bytes(v) for v in vocabulary]
    if not terms:
        raise ValueError("IndexLookup needs a non-empty vocabulary")
    seen = {}
    for i, t in enumerate(terms):
        if t in seen:
            raise ValueError("The passed vocabulary has at least one repeated term: %r at %d and %d" % (t, seen[t], i))
        seen[t] = i
    return seen


def index_lookup(values, vocabulary, num_oov_tokens=1):
    """IndexLookup(vocabulary, num_oov_tokens)(values): int64, the shape of `values` (str / bytes of any shape).
    A value is matched on its bytes before the first NUL."""
    if num_oov_tokens < 0:
        raise ValueError("num_oov_tokens must be >= 0")
    table = _vocab_terms(vocabulary)
    V = len(table)
    arr = np.asarray(values, dtype=object)
    out = np.empty(arr.shape, dtype=np.int64)
    flat_in, flat_out = arr.reshape(-1), out.reshape(-1)
    for i, v in enumerate(flat_in):
        b = _to_bytes(v).split(b"\0", 1)[0]
        if b in table:
            flat_out[i] = table[b]
        elif num_oov_tokens:
            flat_out[i] = V + fingerprint64(b) % num_oov_tokens
        else:
            flat_out[i] = -1
    return out


def _rounded_ids(r, num_bins, default_value):
    """tf.cast(r, int64) then `v < 0 || v >= num_bins -> default_value`, with NaN / +-inf / >= 2^63 -> default
    (x86's cast gives INT64_MIN for them)."""
    r = np.asarray(r, dtype=np.float64)
    bad = np.isnan(r) | (r < 0) | (r >= 2.0 ** 63)
    v = np.where(bad, 0.0, r).astype(np.int64)
    return np.where(bad | (v >= num_bins), np.int64(default_value), v).astype(np.int64)


def _autocast(values):
    x = np.asarray(values)
    with np.errstate(over="ignore"):
        return x.astype(np.float32) if x.dtype.kind == "f" else x


def log_round_q(values, base=None):
    """LogRound's unrounded quotient: float64 log(x) or log(x) / log(base), after the float32 autocast."""
    x = _autocast(values).astype(np.float64)
    with np.errstate(all="ignore"):
        q = np.log(x)
        if base is not None:
            q = q / np.log(np.float64(base))
    return q


def log_round(values, num_bins, default_value=0, base=None):
    """LogRound(num_bins, default_value, base)(values): int64, same shape (log_round.py:75-86)."""
    return _rounded_ids(np.rint(log_round_q(values, base)), num_bins, default_value)


def round_identity(values, num_buckets, default_value=0):
    """RoundIdentity(num_buckets, default_value)(values): int64, same shape (round_identity.py:70-81)."""
    x = _autocast(values)
    if x.dtype.kind in "iub":
        v = x.astype(np.int64)
        return np.where((v < 0) | (v >= num_buckets), np.int64(default_value), v).astype(np.int64)
    return _rounded_ids(np.rint(x.astype(np.float32)), num_buckets, default_value)
