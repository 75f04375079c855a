"""CPU-only tests: the C-ABI library loads and exports every symbol include/b200ps.h
declares, argument grammar errors surface without a device, host-side hashing matches
the reference's vectors, multi-rank host logic under gloo (world_size 2)."""
import ctypes
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_python_vectors.json")


def test_abi_v2_exports_every_declared_symbol():
    from elasticdl_b200 import _lib

    header = "".join(open(os.path.join(ROOT, "include", h)).read() for h in ("b200ps.h", "b200_deepfm.h", "b200_features.h"))
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(b200(?:ps|_deepfm|feat)_[a-z_0-9]+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.SYMBOLS), declared ^ set(_lib.SYMBOLS)
    lib = _lib.lib()
    for name in declared:
        assert getattr(lib, name) is not None
    assert lib.b200ps_abi_version() == _lib.ABI_VERSION == 2
    out = subprocess.check_output(["nm", "-D", "--defined-only", os.path.join(ROOT, "elasticdl_b200", "csrc", "libb200ps.so")], text=True)
    exported = set(re.findall(r"\b(b200(?:ps|_deepfm|feat)_[a-z_0-9]+)$", out, flags=re.M))
    assert declared <= exported


def test_build_digest_covers_every_header():
    """The library is rebuilt when a source in its digest changes: every csrc/*.cuh must be listed in HEADERS."""
    from elasticdl_b200 import build

    cuh = {f for f in os.listdir(build.CSRC) if f.endswith(".cuh")}
    assert cuh and cuh <= set(build.HEADERS), cuh - set(build.HEADERS)


def test_optimizer_grammar_errors_without_a_device():
    from elasticdl_b200 import _lib

    lib = _lib.lib()
    h = ctypes.c_void_p()
    bad = [
        (b"SGD", b"learning_rate=0.1;momentum=0.0;nesterov=true;redundant_arg=1;"),  # optimizer_test.go:233-237
        (b"SGD", b"momentum=0.0;nesterov=true;redundant_arg=1;"),                    # optimizer_test.go:239-243
        (b"Adam", b"learning_rate=0.2;beta_1=0.5;beta_2=0.3;epsilon=0.005;"),
        (b"RMSprop", b"learning_rate=0.1;"),
        (b"SGD", b"learning_rate=abc;momentum=0.0;nesterov=true;"),
        (b"SGD", b"learning_rate=0.1;momentum=0.0;nesterov=maybe;"),
    ]
    for t, a in bad:
        assert lib.b200ps_create(1, 0, t, a, 0, 0, ctypes.byref(h)) == _lib.EINVAL, (t, a)
        with pytest.raises(ValueError):
            _lib.check(_lib.EINVAL)
    if not torch.cuda.is_available():
        # a valid grammar gets past parsing and then fails LOUDLY for lack of a device
        rc = lib.b200ps_create(1, 0, b"SGD", b"learning_rate=0.1;momentum=0.0;nesterov=False;", 0, 0, ctypes.byref(h))
        assert rc == _lib.ECUDA
        with pytest.raises(_lib.PSError):
            _lib.check(rc)
    assert lib.b200ps_create(0, 0, b"SGD", b"learning_rate=0.1;momentum=0.0;nesterov=false;", 0, 0, ctypes.byref(h)) == _lib.EINVAL
    assert lib.b200ps_create(17, 0, b"SGD", b"learning_rate=0.1;momentum=0.0;nesterov=false;", 0, 0, ctypes.byref(h)) == _lib.EINVAL


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200 import ops

    with pytest.raises(RuntimeError, match="no CPU fallback"):
        PSGroup(1, "SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;")
    with pytest.raises(RuntimeError, match="no CPU path"):
        ops.unique(torch.arange(4))
    from elasticdl_b200.layers import Embedding

    with pytest.raises(RuntimeError):
        Embedding(4, input_dim=10)(torch.arange(4))


def test_product_does_not_import_the_oracle():
    pkg = os.path.join(ROOT, "elasticdl_b200")
    for d, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(d, f)).read()
                assert "ps_oracle" not in src and "from oracle" not in src and "import oracle" not in src, f


def test_hash_utils_match_reference_vectors():
    from elasticdl_b200.common.hash_utils import int_to_id, string_to_id

    gold = json.load(open(GOLD))
    for c in gold["string_to_id"]:
        assert string_to_id(c["name"], c["buckets"]) == c["id"]
    for c in gold["int_to_id"]:
        assert int_to_id(c["id"], c["buckets"]) == c["ps"]
    assert string_to_id("dense/kernel:0", 2) == 0 and string_to_id("dense/bias:0", 2) == 1  # pserver_servicer_test.py:509-541


def test_tensor_types():
    from elasticdl_b200.common.tensor_utils import EmbeddingTableInfo, Tensor, UniqueTensor

    t = Tensor("a", 1, None)
    assert t.name == "a" and t.indices is None and tuple(t) == ("a", 1, None)
    i = EmbeddingTableInfo("e", 8, "uniform", 1)
    assert i.capacity is None and i[:4] == ("e", 8, "uniform", 1)
    assert isinstance(UniqueTensor("a", 1, 2), Tensor)


def test_deepfm_workload_shapes_cpu():
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, DeepFMTower, synthetic_batch

    assert len(GROUP_ROWS) == 38 and sum(GROUP_ROWS) == 5549416
    for dist_kind in ("zipf", "uniform"):
        ids, dense, labels = synthetic_batch(1000, 3, "cpu", dist_kind)
        assert ids.shape == (38, 1000) and ids.dtype == torch.int64
        assert dense.shape == (1000, 13) and labels.shape == (1000,)
        rows = torch.tensor(GROUP_ROWS).unsqueeze(1)
        assert bool((ids >= 0).all()) and bool((ids < rows).all())
    ids2, _, _ = synthetic_batch(1000, 3, "cpu", "zipf")
    assert torch.equal(ids2, synthetic_batch(1000, 3, "cpu", "zipf")[0])  # seeded
    # tower == the written-out DeepFM formula (deepfm_model.py:61-109, deepfm_edl_embedding.py:50-56)
    torch.manual_seed(0)
    tw = DeepFMTower(5, 8)
    dense, wide, deep = torch.randn(7, 13), torch.randn(7, 5), torch.randn(7, 5, 8)
    x = torch.cat([dense, deep.reshape(7, -1)], 1)
    for layer in tw.dnn:
        x = torch.relu(layer(x))
    fm = 0.5 * ((deep.sum(1) ** 2) - (deep ** 2).sum(1)).sum(1)
    want = wide.sum(1) + tw.dense_linear(dense)[:, 0] + tw.dnn_logit(x)[:, 0] + fm
    assert torch.allclose(tw(dense, wide, deep), want, atol=1e-5)


def test_pack_batch_refuses_ids_that_do_not_fit_their_width():
    """pack_batch narrows ids with a plain cast, so an id that is negative or too wide for its group would wrap onto
    another, valid row (300 -> 44 in a 1-byte group, -1 -> 65535 in a 2-byte one, 2^32 + 5 -> 5).  Such an id is
    refused with ValueError naming the group and the value: narrow widths and the int32 default, int64 and int32
    ids, at every position of the batch."""
    from elasticdl_b200.workloads.deepfm import id_widths, pack_batch

    rows, B = [200, 5000, 1000000], 33
    narrow = id_widths(rows)
    assert narrow == [1, 2, 4]
    dense, labels = torch.randn(B, 13), torch.rand(B)
    cases = [(narrow, 0, 300), (narrow, 0, 256), (narrow, 0, -1), (narrow, 1, 70000), (narrow, 1, 65536),
             (narrow, 1, -1), (narrow, 2, 2 ** 32 + 5), (narrow, 2, 2 ** 31), (narrow, 2, -1),
             (None, 0, 2 ** 31), (None, 1, -1), (None, 2, 2 ** 32 + 5)]
    for widths, g, bad in cases:
        for pos in (0, B // 2, B - 1):
            ids = torch.zeros(3, B, dtype=torch.int64)
            ids[g, pos] = bad
            with pytest.raises(ValueError, match="id group %d: id %d " % (g, bad)):
                pack_batch(ids, dense, labels, widths=widths)
            if -2 ** 31 <= bad < 2 ** 31:
                with pytest.raises(ValueError, match="id group %d: id %d " % (g, bad)):
                    pack_batch(ids.to(torch.int32), dense, labels, widths=widths)


def test_pack_batch_round_trips_ids_at_every_width_boundary():
    """id_widths picks 1 / 2 / 4 bytes at <= 256 / <= 65536 / larger rows, and every id that fits its width --
    both sides of each byte and of the int16 / int32 sign bits -- reads back unsigned from the packed buffer as it
    went in (segments padded to 16 bytes), for int64 and int32 ids; dense and labels follow the ids."""
    from elasticdl_b200.workloads.deepfm import N_DENSE, id_widths, pack_batch, packed_views

    assert id_widths([1, 2, 255, 256, 257, 65535, 65536, 65537, 2 ** 31]) == [1, 1, 1, 1, 2, 2, 2, 4, 4]
    edges = {1: [0, 1, 127, 128, 254, 255], 2: [0, 255, 256, 32767, 32768, 65534, 65535],
             4: [0, 65535, 65536, 2 ** 31 - 2, 2 ** 31 - 1]}
    # B = 9: every segment padded to 16 bytes, the int32 layout too (its ids come back as the uint8 region);
    # B = 8: no padding, the int32 layout is an int32 [G, B] view
    for widths, B in (([1, 2, 4, 2, 1], 9), ([4, 4, 4], 9), ([4, 4, 4], 8), ([1, 2, 4], 8)):
        ids = torch.zeros(len(widths), B, dtype=torch.int64)
        for g, w in enumerate(widths):
            ids[g, :len(edges[w])] = torch.tensor(edges[w])
        dense, labels = torch.randn(B, N_DENSE), torch.rand(B)
        for dtype in (torch.int64, torch.int32):
            buf = pack_batch(ids.to(dtype), dense, labels, widths=widths)
            region, d, lab = packed_views(buf, len(widths), B, widths)
            assert torch.equal(d, dense) and torch.equal(lab, labels)
            if all(w == 4 for w in widths) and B % 4 == 0:
                assert region.dtype == torch.int32 and torch.equal(region.to(torch.int64), ids)
                continue
            raw, off = region.numpy(), 0
            for g, w in enumerate(widths):
                got = raw[off:off + B * w].view({1: np.uint8, 2: np.uint16, 4: np.uint32}[w]).astype(np.int64)
                assert np.array_equal(got, ids[g].numpy()), (widths, B, g, got)
                off += (B * w + 15) // 16 * 16
            assert off == raw.size


_GLOO_WORKER = r"""
import os, sys
sys.path.insert(0, sys.argv[1])
import torch.distributed as dist
from elasticdl_b200.ps.group import exchange_blobs
rank = int(os.environ["RANK"])
dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%s" % sys.argv[2], rank=rank, world_size=2)
merged = exchange_blobs({rank: b"blob-of-%d" % rank}, 2)
assert merged == {0: b"blob-of-0", 1: b"blob-of-1"}, merged
try:
    exchange_blobs({0: b"x"}, 2)          # both ranks claim shard 0 -> error on every rank
    raise SystemExit("duplicate owner not detected")
except RuntimeError as e:
    assert "two ranks" in str(e)
try:
    exchange_blobs({rank: b"y"}, 3)       # nobody owns shard 2
    raise SystemExit("missing owner not detected")
except RuntimeError as e:
    assert "no rank owns" in str(e)
dist.barrier()
print("rank", rank, "ok")
"""


def test_blob_exchange_gloo_world2(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_GLOO_WORKER)
    port = str(29500 + os.getpid() % 2000)
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=port)
        procs.append(subprocess.Popen([sys.executable, str(script), ROOT, port], env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=120)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), outs
    assert all("ok" in o for o in outs)


def test_exchange_blobs_single_process():
    from elasticdl_b200.ps.group import exchange_blobs

    assert exchange_blobs({0: b"a", 1: b"b"}, 2) == {0: b"a", 1: b"b"}
    with pytest.raises(RuntimeError):
        exchange_blobs({0: b"a"}, 2)


def test_trainer_graph_input_staging_helpers():
    """Host logic of the trainer's CUDA-graph mode (worker/ps_trainer.py): static input buffers keep the features of
    one dtype consecutive in ONE buffer (so rows-of-one-array features stay one zero-copy id array), the per-step
    copy is a single copy when the sources are consecutive pieces of one array and a multi-tensor copy otherwise,
    and the capture signature changes with shapes / dtypes / learning rate."""
    import types

    import torch

    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer as T

    ids = torch.arange(5 * 16, dtype=torch.int64).reshape(5, 16)
    dense = torch.randn(16, 13)
    labels = torch.rand(16)
    feats = {"dense": dense}
    feats.update({"ids_%d" % g: ids[g] for g in range(5)})
    srcs = [v for _, v in T._feature_items(feats)] + [labels]
    statics, groups = T._static_like(srcs)
    assert [tuple(s.shape) for s in statics] == [tuple(s.shape) for s in srcs]
    assert sorted(str(b.dtype) for b, _ in groups) == ["torch.float32", "torch.int64"]
    id_statics = statics[1:6]
    one = T._as_one(id_statics)
    assert one is not None and one.numel() == 5 * 16 and one.data_ptr() == id_statics[0].data_ptr()
    assert all(s.reshape(-1)._base is id_statics[0].reshape(-1)._base for s in id_statics)
    assert T._as_one([ids[0], ids[2]]) is None and T._as_one([ids[0].clone(), ids[1].clone()]) is None
    assert T._as_one([ids[g] for g in range(5)]) is not None
    st = {"statics": statics, "groups": groups}
    T._copy_inputs(st, srcs)
    assert all(torch.equal(a, b) for a, b in zip(statics, srcs))
    scattered = [s.clone() + 1 for s in srcs]  # separately allocated sources: the multi-tensor copy
    T._copy_inputs(st, scattered)
    assert all(torch.equal(a, b) for a, b in zip(statics, scattered))
    rebuilt = T._rebuild_features(feats, statics[:-1])
    assert list(rebuilt) == list(feats) and rebuilt["ids_3"] is statics[4]
    assert T._rebuild_features(dense, [statics[0]]) is statics[0]
    assert isinstance(T._rebuild_features((dense, ids[0]), statics[:2]), tuple)
    # the signature needs device tensors: host features never qualify for the graph
    fake = types.SimpleNamespace(_feature_items=T._feature_items,
                                 _optimizer=types.SimpleNamespace(param_groups=[{"lr": 0.1}]))
    assert T._graph_signature(fake, feats, labels) is None


def test_optimizer_strings_of_the_reference_parse_here():
    """tests/golden `optimizer_info`: the (opt_type, opt_args) strings written by the reference's own
    get_optimizer_info (common/model_utils.py:227-254, executed by tests/golden/gen_from_reference.py) for SGD /
    Nesterov / a callable learning rate / Adam / AMSGrad / Adagrad -- Python's str(float) and str(bool) spellings.
    The C-ABI parser takes every one of them past the grammar (without a device: up to the CUDA error, loudly), and
    the oracle's parser reads the same values."""
    import json

    from elasticdl_b200 import _lib
    from oracle import ps_oracle as O

    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_python_vectors.json")) as f:
        vec = json.load(f)["optimizer_info"]
    assert {v["opt_type"] for v in vec} == {"SGD", "Adam", "Adagrad"}
    lib = _lib.lib()
    for v in vec:
        h = ctypes.c_void_p()
        rc = lib.b200ps_create(1, 0, v["opt_type"].encode(), v["opt_args"].encode(), 0, 0, ctypes.byref(h))
        assert rc in (_lib.OK, _lib.ECUDA), (v, rc)  # never EINVAL: the grammar is accepted
        if rc == _lib.OK:
            lib.b200ps_destroy(h)
        args = O.parse_opt_args(v["opt_type"], v["opt_args"])
        assert float(args["learning_rate"]) > 0
        for k in ("nesterov", "amsgrad"):
            if k in args:
                assert O.parse_bool(args[k]) in (True, False)
    want = {"learning_rate": "0.001", "beta_1": "0.9", "beta_2": "0.999", "epsilon": "1e-07", "amsgrad": "False"}
    assert O.parse_opt_args("Adam", vec[3]["opt_args"]) == want
