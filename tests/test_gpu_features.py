"""GPU parity of the feature-id generation kernels (csrc/feature_ids.cu, include/b200_features.h) against
oracle/feature_oracle.py: bit-exact integer work."""
import numpy as np
import pytest
import torch

from oracle import feature_oracle as FO

pytestmark = pytest.mark.gpu


def test_hashing_reference_example_on_gpu():
    from elasticdl_b200.preprocessing import Hashing, encode_strings

    layer = Hashing(num_bins=3)
    out = layer(encode_strings([["A"], ["B"], ["C"], ["D"], ["E"]]))
    assert out.dtype == torch.int64 and out.shape == (5, 1)
    assert np.array_equal(out.cpu().numpy(), [[1], [0], [1], [1], [2]])  # hashing.py:35-39
    with pytest.raises(ValueError):
        Hashing(num_bins=0)


@pytest.mark.parametrize("width", [1, 3, 8, 16, 17, 33, 64])
def test_fingerprint64_all_length_branches(width):
    import ctypes

    from elasticdl_b200 import _lib
    from elasticdl_b200.preprocessing import encode_strings

    rng = np.random.RandomState(width)
    strs = [bytes(rng.randint(1, 256, size=rng.randint(0, width + 1)).astype(np.uint8)) for _ in range(3000)]
    strs[0] = b""
    strs[1] = bytes(rng.randint(1, 256, size=width).astype(np.uint8))
    x = encode_strings(strs, width)
    out = torch.empty(len(strs), dtype=torch.int64, device="cuda")
    lib = _lib.lib()
    assert lib.b200feat_fingerprint64(x.data_ptr(), width, len(strs), out.data_ptr(),
                                      ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)) == 0
    got = out.cpu().numpy().view(np.uint64)
    want = np.array([FO.fingerprint64(s) for s in strs], dtype=np.uint64)
    assert np.array_equal(got, want)


def test_hashing_ints_and_discretization_layers():
    from elasticdl_b200.preprocessing import ConcatenateWithOffset, Discretization, Hashing, Normalizer

    rng = np.random.RandomState(0)
    vals = np.concatenate([rng.randint(-10 ** 12, 10 ** 12, size=5000), [0, -1, 9223372036854775807, -9223372036854775807]]).astype(np.int64)
    out = Hashing(1000003)(torch.from_numpy(vals).cuda().view(-1, 1))
    assert np.array_equal(out.cpu().numpy().ravel(), FO.hashing(vals, 1000003))
    layer = Discretization(bins=[1, 5, 10])
    x = torch.tensor([[0.2], [1.6], [4.2], [6.1], [10.9]], device="cuda")
    assert np.array_equal(layer(x).cpu().numpy(), [[0], [1], [1], [2], [3]])  # discretization_test.py:26-31
    assert layer.num_bins() == 4
    xs = rng.randn(10000).astype(np.float32) * 50
    bins = [-1.0, 0.0, 1.0, 1.0, 3.0, 8.0, 23.0, 56.0, 184.0]
    assert np.array_equal(Discretization(bins)(torch.from_numpy(xs).cuda()).cpu().numpy(), FO.discretize(xs, bins))
    a1, a2 = torch.tensor([[1], [1], [1]], device="cuda"), torch.tensor([[2], [2], [2]], device="cuda")
    cat = ConcatenateWithOffset(offsets=[0, 10], axis=1)([a1, a2])
    assert np.array_equal(cat.cpu().numpy(), [[1, 12], [1, 12], [1, 12]])  # concatenate_with_offset_test.py:27-34
    n = Normalizer(1.0, 2.0)(torch.tensor([[3.0], [5.0], [7.0]], device="cuda"))
    assert n.dtype == torch.float64 and np.array_equal(n.cpu().numpy(), [[1.0], [2.0], [3.0]])


@pytest.mark.parametrize("ids_dtype", [torch.int64, torch.int32])
def test_fused_dac_ctr_transform_matches_layer_by_layer_oracle(ids_dtype):
    """transform_feature of model_zoo/dac_ctr/feature_transform.py:36-118 in one launch == the oracle's
    layer-by-layer composition, on synthetic Criteo-shaped raw features (13 int64 columns, 26 hex strings)."""
    from elasticdl_b200.preprocessing import encode_strings
    from elasticdl_b200.workloads.dac_ctr_features import (BUCKET_GROUP_FEATURES, FEATURE_BOUNDARIES, FEATURES_AVGS,
                                                           FEATURES_STDDEVS, HASH_BINS, STANDARDIZED_FEATURES,
                                                           dac_ctr_transform, synthetic_raw_batch)

    B = 4096
    numeric, strings, raw_strs = synthetic_raw_batch(B, seed=3, device="cuda")
    tf_ = dac_ctr_transform(ids_dtype)
    ids, dense = tf_(numeric, strings)
    assert ids.dtype == ids_dtype and ids.shape == (38, B) and dense.shape == (B, 13)
    num = numeric.cpu().numpy()
    want_ids = []
    for f in BUCKET_GROUP_FEATURES:
        col = STANDARDIZED_FEATURES.index(f)
        want_ids.append(FO.discretize(num[col], FEATURE_BOUNDARIES[f]))
    for j, bins in enumerate(HASH_BINS):
        want_ids.append(FO.hashing(raw_strs[j], bins))
    assert np.array_equal(ids.cpu().numpy().astype(np.int64), np.stack(want_ids))
    want_dense = np.stack([FO.normalize(num[i], FEATURES_AVGS[f], FEATURES_STDDEVS[f]) for i, f in enumerate(STANDARDIZED_FEATURES)], 1)
    assert np.array_equal(dense.cpu().numpy(), want_dense.astype(np.float32))  # double in the kernel, cast once
    assert tf_.max_ids[:3] == [5, 10, 9]  # len(boundaries) + 1, feature_transform.py:100-103
