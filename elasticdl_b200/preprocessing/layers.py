"""Feature-id generation layers on the GPU: mirrors of elasticdl_preprocessing/layers
(hashing.py:20-98, discretization.py:20-78, concatenate_with_offset.py:17-98, normalizer.py,
index_lookup.py:22-128, log_round.py:29-98, round_identity.py:17-86) with the same constructor
arguments, over CUDA tensors, calling the kernels of csrc/feature_ids.cu through the C ABI of
include/b200_features.h.  CUDA only -- there is no CPU path.

Strings travel as fixed-width zero-padded byte matrices (`encode_strings`): torch has no string
tensors, and a Criteo categorical value is at most 8 hex characters.  A string ends at its first NUL, so
strings holding a NUL byte are refused.

`FeatureTransform` is the fused form of model_zoo/dac_ctr/feature_transform.py:36-118
(transform_feature / transform_group): every group's Discretization / Hashing / IndexLookup / LogRound /
RoundIdentity, its ConcatenateWithOffset offset and the Normalizer of the dense columns in ONE launch that
writes the [G, B] id matrix (int64 or int32) b200ps_unique consumes.
"""
import collections
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib

MAX_STRING_BYTES = 64
INT32_IDS = 1 << 31


def _stream(device):
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _check(rc):
    if rc:
        raise ValueError("b200feat error %d: %s" % (rc, _lib.lib().b200feat_last_error().decode("utf-8", "replace")))


def _need_cuda(t, what):
    if not (isinstance(t, torch.Tensor) and t.is_cuda):
        raise RuntimeError("%s must be a CUDA tensor: elasticdl_b200 has no CPU path" % what)


def _check_bins(bins):
    """Discretization boundaries as the kernel keeps them (float32): the kernel binary-searches them, and TF's
    Bucketize refuses unsorted boundaries."""
    b = np.asarray(bins, dtype=np.float32).reshape(-1)
    if np.isnan(b).any() or np.any(b[1:] < b[:-1]):
        raise ValueError("Discretization bins must be sorted in ascending order (and hold no NaN): %r" % (list(bins),))
    return b


def encode_strings(values, width=None, device="cuda"):
    """list / array of str or bytes (any shape) -> uint8 tensor [*shape, width], zero padded."""
    arr = np.asarray(values, dtype=object)
    flat = [v if isinstance(v, (bytes, bytearray)) else str(v).encode("utf-8") for v in arr.reshape(-1)]
    if any(b"\0" in b for b in flat):
        raise ValueError("strings holding a NUL byte cannot be zero padded: the kernels end a string at its first NUL")
    w = max([len(b) for b in flat] + [1]) if width is None else int(width)
    if w > MAX_STRING_BYTES or any(len(b) > w for b in flat):
        raise ValueError("strings longer than %d bytes are not supported" % min(w, MAX_STRING_BYTES))
    buf = np.zeros((len(flat), w), dtype=np.uint8)
    for i, b in enumerate(flat):
        buf[i, :len(b)] = np.frombuffer(b, dtype=np.uint8)
    return torch.from_numpy(buf.reshape(arr.shape + (w,))).to(device)


class Hashing(torch.nn.Module):
    """output_id = FarmHash64(string) % num_bins; integer inputs are converted with tf.as_string
    first (hashing.py:20-98).  Input: an int64 CUDA tensor of any shape, or a uint8 CUDA tensor
    [..., W] of zero-padded strings; output: int64, the input's shape (without W)."""

    def __init__(self, num_bins):
        if num_bins is None or num_bins <= 0:
            raise ValueError("`num_bins` cannot be `None` or non-positive values.")
        super().__init__()
        self.num_bins = int(num_bins)

    def forward(self, inputs):
        _need_cuda(inputs, "inputs")
        lib = _lib.lib()
        with torch.cuda.device(inputs.device):
            if inputs.dtype == torch.uint8:
                x = inputs.contiguous()
                w = x.shape[-1]
                out = torch.empty(x.shape[:-1], dtype=torch.int64, device=x.device)
                if out.numel():
                    _check(lib.b200feat_hash_strings(x.data_ptr(), w, out.numel(), self.num_bins, out.data_ptr(),
                                                     _stream(x.device)))
                return out
            if inputs.dtype not in (torch.int32, torch.int64):
                raise TypeError("Hashing takes integer or string (uint8 [..., W]) inputs")
            x = inputs.to(torch.int64).contiguous()
            out = torch.empty_like(x)
            if out.numel():
                _check(lib.b200feat_hash_ints(x.data_ptr(), x.numel(), self.num_bins, out.data_ptr(), _stream(x.device)))
            return out

    def get_config(self):
        return {"num_bins": self.num_bins}


class Discretization(torch.nn.Module):
    """Buckets data into discrete ranges; bins include the left boundary (discretization.py:20-78)."""

    def __init__(self, bins):
        super().__init__()
        self.bins = list(bins)
        self._bnd = _check_bins(self.bins)

    def num_bins(self):
        return len(self.bins) + 1

    def forward(self, inputs):
        _need_cuda(inputs, "inputs")
        # float32 for every input: the reference layer is a Keras Layer of the default float32 dtype policy, whose
        # __call__ autocasts floating inputs (float64 too) to float32, and BucketizeOp compares integers in float
        x = inputs.to(torch.float32).contiguous()
        out = torch.empty(x.shape, dtype=torch.int64, device=x.device)
        bnd = (ctypes.c_float * max(len(self.bins), 1))(*self._bnd.tolist())
        if out.numel():
            with torch.cuda.device(x.device):
                _check(_lib.lib().b200feat_bucketize(x.data_ptr(), x.numel(), bnd, len(self.bins), out.data_ptr(),
                                                     _stream(x.device)))
        return out

    def get_config(self):
        return {"bins": self.bins}


class ConcatenateWithOffset(torch.nn.Module):
    """Adds offsets[i] to the i-th id tensor, then concatenates (concatenate_with_offset.py:17-98)."""

    def __init__(self, offsets, axis=-1):
        super().__init__()
        self.offsets = offsets
        self.axis = axis

    def forward(self, inputs):
        if self.offsets is None:
            return torch.cat(list(inputs), dim=self.axis)
        if not isinstance(inputs, list):
            return inputs
        if len(self.offsets) != len(inputs):
            raise ValueError("The offsets length is not equal to inputs length"
                             "the inputs are {}, offsets are {}".format(inputs, self.offsets))
        return torch.cat([t + o for t, o in zip(inputs, self.offsets)], dim=self.axis)


class Normalizer(torch.nn.Module):
    """(x - subtractor) / divisor in float64 (normalizer.py)."""

    def __init__(self, subtractor, divisor):
        super().__init__()
        if divisor == 0:
            raise ValueError("The divisor cannot be 0")
        self.subtractor, self.divisor = subtractor, divisor

    def forward(self, inputs):
        return (inputs.to(torch.float64) - self.subtractor) / self.divisor


class VocabSlot(ctypes.Structure):  # b200feat_vocab_slot_t
    _fields_ = [("fingerprint", ctypes.c_uint64), ("index", ctypes.c_int32), ("length", ctypes.c_int32)]


VOCAB_SLOT_DTYPE = np.dtype([("fingerprint", "<u8"), ("index", "<i4"), ("length", "<i4")])  # the same, in numpy


def read_vocabulary_file(path):
    """index_lookup.py:98-114 (_get_vocabulary_from_file): one token per line, UTF-8 with errors ignored, stripped;
    a blank line is the token ''."""
    with open(path, "rb") as f:
        return [line.decode("utf-8", "ignore").strip() for line in f]


def _term_bytes(vocabulary):
    """The vocabulary (list or file path) as a list of bytes; refuses what the table cannot hold."""
    if vocabulary is None:
        vocabulary = []
    elif isinstance(vocabulary, str):
        vocabulary = read_vocabulary_file(vocabulary)
    terms = [v if isinstance(v, (bytes, bytearray)) else str(v).encode("utf-8") for v in vocabulary]
    if not terms:
        raise ValueError("IndexLookup needs a non-empty vocabulary")
    for i, t in enumerate(terms):
        if b"\0" in t:
            raise ValueError("vocabulary term %d holds a NUL byte: the kernels end a string at its first NUL" % i)
        if len(t) > MAX_STRING_BYTES:
            raise ValueError("vocabulary term %d is %d bytes long; terms longer than %d bytes are not supported"
                             % (i, len(t), MAX_STRING_BYTES))
    return [bytes(t) for t in terms], list(vocabulary)


def build_vocab_table(terms):
    """Host build of the vocabulary table (b200feat_vocab_build): terms is a list of bytes (each at most 64 bytes,
    no NUL).  Returns (slots: numpy VOCAB_SLOT_DTYPE [n_slots], term matrix: uint8 [V, Wv]); a repeated term raises
    ValueError naming the repeated terms (index_lookup.py:61-76)."""
    V = len(terms)
    wv = max(max(len(t) for t in terms), 1)
    mat = np.frombuffer(b"".join(t.ljust(wv, b"\0") for t in terms), dtype=np.uint8).reshape(V, wv)
    lib = _lib.lib()
    n_slots = lib.b200feat_vocab_slots(V)
    if n_slots < 0:
        raise ValueError("vocabulary of %d terms: 1 .. 2^31 - 1 terms are supported" % V)
    slots = np.zeros(n_slots, dtype=VOCAB_SLOT_DTYPE)
    dup = ctypes.c_int64(-1)
    rc = lib.b200feat_vocab_build(mat.ctypes.data, V, wv, n_slots, slots.ctypes.data, ctypes.byref(dup))
    if rc and dup.value >= 0:
        repeated = [item for item, count in collections.Counter(terms).items() if count > 1]
        raise ValueError("The passed vocabulary has at least one repeated term. Please uniquify your dataset before "
                         "passing it to IndexLookup(). The repeated terms are %s"
                         % [t.decode("utf-8", "replace") for t in repeated])
    _check(rc)
    return slots, mat


class _VocabTable:
    """A vocabulary table built on the host (refusals first), then copied to `device`: slots (int64 [n_slots, 2],
    the 16-byte slots) and terms (uint8 [V, Wv])."""

    def __init__(self, terms, device):
        slots, mat = build_vocab_table(terms)
        self.V, self.Wv = mat.shape
        device = device() if callable(device) else device
        self.slots = torch.from_numpy(slots.view(np.int64).reshape(-1, 2)).to(device)
        self.terms = torch.from_numpy(mat.copy()).to(device)


def _current_cuda_device():
    return torch.device("cuda", torch.cuda.current_device())


class IndexLookup(torch.nn.Module):
    """Maps strings to their vocabulary position; any other string to V + Fingerprint64 % num_oov_tokens, or to -1
    with num_oov_tokens = 0 (index_lookup.py:22-128, index_table_from_tensor with num_oov_buckets).
    vocabulary: list of str / bytes, or the path of a one-token-per-line file.  A repeated term, an empty
    vocabulary, a term longer than 64 bytes or holding a NUL, and num_oov_tokens < 0 are refused.
    Input: a uint8 CUDA tensor [..., W] of zero-padded strings; output: int64, the input's shape without W.
    The table is built at construction and kept as buffers on the current CUDA device (it holds indices and
    fingerprints, not addresses, so .to(device) moves it)."""

    def __init__(self, vocabulary=None, num_oov_tokens=1, **kwargs):
        super().__init__()
        if num_oov_tokens is None or num_oov_tokens < 0:
            raise ValueError("num_oov_tokens must be >= 0")
        self.num_oov_tokens = int(num_oov_tokens)
        terms, self.vocabulary = _term_bytes(vocabulary)
        table = _VocabTable(terms, _current_cuda_device)
        self.V, self.Wv = table.V, table.Wv
        self.register_buffer("slots", table.slots)
        self.register_buffer("terms", table.terms)

    def vocab_size(self):
        return self.V + self.num_oov_tokens

    def forward(self, inputs):
        _need_cuda(inputs, "inputs")
        if inputs.dtype != torch.uint8:
            raise TypeError("IndexLookup takes string inputs (uint8 [..., W] zero-padded byte strings): "
                            "its vocabulary holds strings")
        if inputs.device != self.slots.device:
            raise ValueError("inputs are on %s, the vocabulary table on %s" % (inputs.device, self.slots.device))
        x = inputs.contiguous()
        out = torch.empty(x.shape[:-1], dtype=torch.int64, device=x.device)
        if out.numel():
            with torch.cuda.device(x.device):
                _check(_lib.lib().b200feat_index_lookup(
                    x.data_ptr(), x.shape[-1], out.numel(), self.slots.data_ptr(), self.terms.data_ptr(),
                    self.slots.shape[0], self.V, self.Wv, self.num_oov_tokens, out.data_ptr(), _stream(x.device)))
        return out

    def get_config(self):
        return {"num_oov_tokens": self.num_oov_tokens, "vocabulary": None}


def _numeric_input(inputs):
    """Floating inputs -> float32 (the Keras float32 autocast, as in Discretization), integers -> int64."""
    _need_cuda(inputs, "inputs")
    if inputs.dtype.is_floating_point:
        return inputs.to(torch.float32).contiguous(), 1
    if inputs.dtype in (torch.int8, torch.uint8, torch.int16, torch.int32, torch.int64):
        return inputs.to(torch.int64).contiguous(), 0
    raise TypeError("numeric inputs are integer or floating tensors")


class LogRound(torch.nn.Module):
    """id = rint(log(x) [/ log(base)]) in float64 if it lies in [0, num_bins), else default_value (NaN, +-inf and
    values >= 2^63 included); log_round.py:29-98.  Output: int64, the input's shape."""

    def __init__(self, num_bins, default_value=0, base=None):
        super().__init__()
        self.num_bins, self.default_value, self.base = int(num_bins), int(default_value), base

    def forward(self, inputs):
        x, is_float = _numeric_input(inputs)
        out = torch.empty(x.shape, dtype=torch.int64, device=x.device)
        if out.numel():
            with torch.cuda.device(x.device):
                _check(_lib.lib().b200feat_log_round(
                    x.data_ptr(), is_float, x.numel(), self.num_bins, self.default_value, self.base is not None,
                    0.0 if self.base is None else float(self.base), out.data_ptr(), _stream(x.device)))
        return out

    def get_config(self):
        return {"num_bins": self.num_bins, "base": self.base, "default_value": self.default_value}


class RoundIdentity(torch.nn.Module):
    """id = rint(x) (float32; integers pass through) if it lies in [0, num_buckets), else default_value;
    round_identity.py:17-86.  Output: int64, the input's shape."""

    def __init__(self, num_buckets, default_value=0):
        super().__init__()
        self.num_buckets, self.default_value = int(num_buckets), int(default_value)

    def forward(self, inputs):
        x, is_float = _numeric_input(inputs)
        out = torch.empty(x.shape, dtype=torch.int64, device=x.device)
        if out.numel():
            with torch.cuda.device(x.device):
                _check(_lib.lib().b200feat_round_identity(
                    x.data_ptr(), is_float, x.numel(), self.num_buckets, self.default_value, out.data_ptr(),
                    _stream(x.device)))
        return out

    def get_config(self):
        return {"num_buckets": self.num_buckets, "default_value": self.default_value}


def _check_out(t, shape, dtype, device, what):
    if t is not None and (t.device != device or t.dtype != dtype or tuple(t.shape) != shape or not t.is_contiguous()):
        raise ValueError("%s must be a contiguous %s tensor of shape %s on %s" % (what, dtype, shape, device))


class FeatureGroup(ctypes.Structure):  # b200feat_group_t
    _fields_ = [("kind", ctypes.c_int32), ("column", ctypes.c_int32), ("n_boundaries", ctypes.c_int32),
                ("boundary_off", ctypes.c_int32), ("num_bins", ctypes.c_int64), ("offset", ctypes.c_int64)]


class FeatureDense(ctypes.Structure):  # b200feat_dense_t
    _fields_ = [("column", ctypes.c_int32), ("pad", ctypes.c_int32), ("subtractor", ctypes.c_double),
                ("divisor", ctypes.c_double)]


class FeatureGroupExt(ctypes.Structure):  # b200feat_group_ext_t
    _fields_ = [("slots_dev", ctypes.c_void_p), ("terms_dev", ctypes.c_void_p), ("n_slots", ctypes.c_int64),
                ("V", ctypes.c_int32), ("Wv", ctypes.c_int32), ("default_value", ctypes.c_int64),
                ("has_base", ctypes.c_int32), ("absent", ctypes.c_int32), ("base", ctypes.c_double)]


DISCRETIZE, HASH_STRING, HASH_INT, LOOKUP, LOG_ROUND, ROUND_IDENTITY = 0, 1, 2, 3, 4, 5


class FeatureTransform:
    """Fused transform_feature (model_zoo/dac_ctr/feature_transform.py:36-78).

    groups: list of dicts, one per output id group, each
        {"kind": "discretize", "column": numeric column, "bins": [...]} or
        {"kind": "hash", "column": string column, "num_bins": n} or
        {"kind": "hash_int", "column": int64 numeric column, "num_bins": n} or
        {"kind": "lookup", "column": string column, "vocabulary": list | path, "num_oov_tokens": 1} or
        {"kind": "log_round", "column": numeric column, "num_bins": n, "default_value": 0, "base": None} or
        {"kind": "round_identity", "column": numeric column, "num_buckets": n, "default_value": 0},
    plus an optional "offset" and an optional "absent": True -- a cell ToSparse drops with its default
    ignore_value (an empty string, a float 0.0, an int64 -1) gets id -1, without the offset; bins are sorted; with ids_dtype=torch.int32 every group's ids (offset plus
    [0, max_id), and -1 / default_value where a group can give them) must fit int32.
    dense: list of (numeric column, subtractor, divisor) -- the Normalizer columns.
    device: where lookup groups keep their vocabulary tables (built at construction; default: the current device).
    __call__(numeric [n_numeric, B] int64 or float32, strings [n_string, B, W] uint8 or None)
      -> (ids [G, B] int64 / int32, dense [B, n_dense] float32 or None)."""

    def __init__(self, groups, dense=(), ids_dtype=torch.int64, device=None):
        self.G = len(groups)
        self.ids32 = 1 if ids_dtype == torch.int32 else 0
        self.ids_dtype = ids_dtype
        self._groups = (FeatureGroup * max(self.G, 1))()
        self._ext = (FeatureGroupExt * max(self.G, 1))()
        self._tables = []
        self.device = None
        bnd = []
        self.max_ids = []
        self._hash_int = False
        for g, spec in enumerate(groups):
            fg, ext = self._groups[g], self._ext[g]
            fg.column = int(spec["column"])
            fg.offset = int(spec.get("offset", 0))
            ext.absent = 1 if spec.get("absent", False) else 0
            lo, hi = 0, None  # smallest and (where it is not max_id - 1) largest id before the offset
            if spec["kind"] == "discretize":
                fg.kind, fg.n_boundaries, fg.boundary_off = DISCRETIZE, len(spec["bins"]), len(bnd)
                bnd.extend(_check_bins(spec["bins"]).tolist())
                self.max_ids.append(fg.offset + len(spec["bins"]) + 1)
            elif spec["kind"] in ("hash", "hash_int"):
                if spec["num_bins"] is None or spec["num_bins"] <= 0:
                    raise ValueError("`num_bins` cannot be `None` or non-positive values.")
                fg.kind = HASH_STRING if spec["kind"] == "hash" else HASH_INT
                fg.num_bins = int(spec["num_bins"])
                self.max_ids.append(fg.offset + fg.num_bins)
                self._hash_int |= fg.kind == HASH_INT
            elif spec["kind"] == "lookup":
                n_oov = spec.get("num_oov_tokens", 1)
                if n_oov is None or n_oov < 0:
                    raise ValueError("num_oov_tokens must be >= 0")
                terms, _ = _term_bytes(spec["vocabulary"])
                table = _VocabTable(terms, lambda: self.device or (_current_cuda_device() if device is None
                                                                   else torch.device(device)))
                self.device = table.slots.device
                self._tables.append(table)
                fg.kind, fg.num_bins = LOOKUP, int(n_oov)
                ext.slots_dev, ext.terms_dev = table.slots.data_ptr(), table.terms.data_ptr()
                ext.n_slots, ext.V, ext.Wv = table.slots.shape[0], table.V, table.Wv
                lo = 0 if n_oov else -1
                self.max_ids.append(fg.offset + table.V + fg.num_bins)  # census get_max_id: len(vocabulary) + 1
            elif spec["kind"] in ("log_round", "round_identity"):
                fg.kind = LOG_ROUND if spec["kind"] == "log_round" else ROUND_IDENTITY
                fg.num_bins = int(spec["num_bins"] if fg.kind == LOG_ROUND else spec["num_buckets"])
                ext.default_value = int(spec.get("default_value", 0))
                base = spec.get("base") if fg.kind == LOG_ROUND else None
                ext.has_base, ext.base = base is not None, 0.0 if base is None else float(base)
                lo = min(0, ext.default_value) if fg.num_bins > 0 else ext.default_value
                hi = max(fg.num_bins - 1, ext.default_value) if fg.num_bins > 0 else ext.default_value
                self.max_ids.append(fg.offset + fg.num_bins)
            else:
                raise ValueError("unknown group kind %r" % (spec["kind"],))
            top = self.max_ids[-1] - 1 if hi is None else fg.offset + hi
            if self.ids32 and (fg.offset + lo < -INT32_IDS or top >= INT32_IDS):
                raise ValueError("group %d: ids %d..%d do not fit int32 ids" % (g, fg.offset + lo, top))
        self._bnd = (ctypes.c_float * max(len(bnd), 1))(*bnd)
        self._n_bnd = len(bnd)
        self.n_dense = len(dense)
        self._dense = (FeatureDense * max(self.n_dense, 1))()
        for j, (col, sub, div) in enumerate(dense):
            if div == 0:
                raise ValueError("The divisor cannot be 0")
            self._dense[j].column, self._dense[j].subtractor, self._dense[j].divisor = int(col), float(sub), float(div)

    def __call__(self, numeric, strings=None, ids_out=None, dense_out=None):
        _need_cuda(numeric, "numeric")
        numeric = numeric.contiguous()
        if numeric.dtype not in (torch.int64, torch.float32):
            raise TypeError("numeric columns are int64 or float32")
        if numeric.dtype == torch.float32 and self._hash_int:
            raise TypeError("hash_int groups take int64 numeric columns: Hashing converts integer inputs only")
        n_num, B = numeric.shape
        n_str, W, sptr = 0, 0, None
        if strings is not None:
            _need_cuda(strings, "strings")
            if strings.dtype != torch.uint8 or strings.dim() != 3:
                raise TypeError("strings are uint8 [n_string, B, W]")
            strings = strings.contiguous()
            n_str, Bs, W = strings.shape
            if Bs != B:
                raise ValueError("numeric and string columns disagree on the batch size")
            sptr = strings.data_ptr()
        dev = numeric.device
        if self.device is not None and dev != self.device:
            raise ValueError("inputs are on %s, the vocabulary tables on %s" % (dev, self.device))
        if ids_out is None and self.G:
            ids_out = torch.empty((self.G, B), dtype=self.ids_dtype, device=dev)
        if dense_out is None and self.n_dense:
            dense_out = torch.empty((B, self.n_dense), dtype=torch.float32, device=dev)
        _check_out(ids_out, (self.G, B), self.ids_dtype, dev, "ids_out")
        _check_out(dense_out, (B, self.n_dense), torch.float32, dev, "dense_out")
        if B == 0:  # like the layers: an empty batch gives empty outputs, without a launch
            return ids_out, dense_out
        with torch.cuda.device(dev):
            _check(_lib.lib().b200feat_transform_ext(
                self._groups, self._ext, self.G, self._bnd, self._n_bnd, self._dense, self.n_dense, numeric.data_ptr(), n_num,
                1 if numeric.dtype == torch.float32 else 0, sptr, n_str, W, B,
                ids_out.data_ptr() if ids_out is not None else None, self.ids32,
                dense_out.data_ptr() if dense_out is not None else None, _stream(dev)))
        return ids_out, dense_out
