"""Feature-id generation layers on the GPU: mirrors of elasticdl_preprocessing/layers
(hashing.py:20-98, discretization.py:20-78, concatenate_with_offset.py:17-98, normalizer.py) with the
same constructor arguments, over CUDA tensors, calling the kernels of csrc/feature_ids.cu through
the C ABI of include/b200_features.h.  CUDA only -- there is no CPU path.

Strings travel as fixed-width zero-padded byte matrices (`encode_strings`): torch has no string
tensors, and a Criteo categorical value is at most 8 hex characters.  A string ends at its first NUL, so
strings holding a NUL byte are refused.

`FeatureTransform` is the fused form of model_zoo/dac_ctr/feature_transform.py:36-118
(transform_feature / transform_group): every group's Discretization / Hashing, its
ConcatenateWithOffset offset and the Normalizer of the dense columns in ONE launch that writes the
[G, B] id matrix (int64 or int32) b200ps_unique consumes.
"""
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


def _check_out(t, shape, dtype, device, what):
    if t is not None and (t.device != device or t.dtype != dtype or tuple(t.shape) != shape or not t.is_contiguous()):
        raise ValueError("%s must be a contiguous %s tensor of shape %s on %s" % (what, dtype, shape, device))


class FeatureGroup(ctypes.Structure):  # b200feat_group_t
    _fields_ = [("kind", ctypes.c_int32), ("column", ctypes.c_int32), ("n_boundaries", ctypes.c_int32),
                ("boundary_off", ctypes.c_int32), ("num_bins", ctypes.c_int64), ("offset", ctypes.c_int64)]


class FeatureDense(ctypes.Structure):  # b200feat_dense_t
    _fields_ = [("column", ctypes.c_int32), ("pad", ctypes.c_int32), ("subtractor", ctypes.c_double),
                ("divisor", ctypes.c_double)]


DISCRETIZE, HASH_STRING, HASH_INT = 0, 1, 2


class FeatureTransform:
    """Fused transform_feature (model_zoo/dac_ctr/feature_transform.py:36-78).

    groups: list of dicts, one per output id group, each
        {"kind": "discretize", "column": numeric column, "bins": [...]} or
        {"kind": "hash", "column": string column, "num_bins": n} or
        {"kind": "hash_int", "column": int64 numeric column, "num_bins": n}, plus an optional "offset";
    bins are sorted; with ids_dtype=torch.int32 every group's ids [offset, max_id) must fit int32.
    dense: list of (numeric column, subtractor, divisor) -- the Normalizer columns.
    __call__(numeric [n_numeric, B] int64 or float32, strings [n_string, B, W] uint8 or None)
      -> (ids [G, B] int64 / int32, dense [B, n_dense] float32 or None)."""

    def __init__(self, groups, dense=(), ids_dtype=torch.int64):
        self.G = len(groups)
        self.ids32 = 1 if ids_dtype == torch.int32 else 0
        self.ids_dtype = ids_dtype
        self._groups = (FeatureGroup * max(self.G, 1))()
        bnd = []
        self.max_ids = []
        self._hash_int = False
        for g, spec in enumerate(groups):
            fg = self._groups[g]
            fg.column = int(spec["column"])
            fg.offset = int(spec.get("offset", 0))
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
            else:
                raise ValueError("unknown group kind %r" % (spec["kind"],))
            if self.ids32 and (fg.offset < -INT32_IDS or self.max_ids[-1] > INT32_IDS):
                raise ValueError("group %d: ids %d..%d do not fit int32 ids" % (g, fg.offset, self.max_ids[-1] - 1))
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
        if ids_out is None and self.G:
            ids_out = torch.empty((self.G, B), dtype=self.ids_dtype, device=dev)
        if dense_out is None and self.n_dense:
            dense_out = torch.empty((B, self.n_dense), dtype=torch.float32, device=dev)
        _check_out(ids_out, (self.G, B), self.ids_dtype, dev, "ids_out")
        _check_out(dense_out, (B, self.n_dense), torch.float32, dev, "dense_out")
        if B == 0:  # like the layers: an empty batch gives empty outputs, without a launch
            return ids_out, dense_out
        with torch.cuda.device(dev):
            _check(_lib.lib().b200feat_transform(
                self._groups, self.G, self._bnd, self._n_bnd, self._dense, self.n_dense, numeric.data_ptr(), n_num,
                1 if numeric.dtype == torch.float32 else 0, sptr, n_str, W, B,
                ids_out.data_ptr() if ids_out is not None else None, self.ids32,
                dense_out.data_ptr() if dense_out is not None else None, _stream(dev)))
        return ids_out, dense_out
