"""The tile tower reading its embedding rows straight from the table records (b200_deepfm_rows_t, the engine's
row_source="table") instead of from rows pulled into bet_wide / bet_deep first.

Kernel level: one PS state per case, set with set_rows, holds each group's live rows at distinct random ids
(row 0 and the last row of every table among them) and NaN in every other record, so a row read from the
wrong place shows.  The forward logits must equal those of the same tower on the pulled rows bit for bit (same
fp32 words in, no atomics in the forward pass), and forward + backward must pass the float64 reference bound
of oracle/tower_oracle.py.  Adam and SGD tables are both used: their records are 24 / 4 and 8 / 4 floats.

Engine level: training with the row source "table" and with "pull" from the same seed gives the same created
rows and, up to the order of fp32 atomic adds, the same losses, rows and dense parameters."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import tower_oracle as T
from tests.test_gpu_tower_reference import NAN, SHAPES_B, Buffers, _batch, _call, _group_rows, _n_sm, make_inputs

gpu = pytest.mark.gpu
ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")
SGD = ("SGD", "learning_rate=0.01;momentum=0.0;nesterov=false;")
STRIDES = {"Adam": (24, 4), "SGD": (8, 4)}  # deep / wide record, floats


def _table_state(opt, inputs, seed):
    """A one-shard PS holding the live rows of `inputs` (module docstring); returns (group, uniq [G, B])."""
    from elasticdl_b200.ps import PSGroup

    inv, n_unique, bet_wide, bet_deep = inputs[:4]
    G, B = inv.shape
    dev = inv.device
    gen = torch.Generator(device=dev).manual_seed(seed)
    nu = n_unique.tolist()
    rows = [max(r, u) for r, u in zip(_group_rows(G), nu)]
    group = PSGroup(1, *opt, device=0)
    for g in range(G):
        group.register_table("deep_%d" % g, T.D, "zero", rows[g])
        group.register_table("wide_%d" % g, 1, "zero", rows[g])
    group.commit()
    uniq = torch.zeros((G, B), dtype=torch.int64, device=dev)
    for g in range(G):
        r, u = rows[g], nu[g]
        ends = torch.tensor(sorted({0, r - 1}), device=dev)
        perm = torch.randperm(r, generator=gen, device=dev)
        ids = torch.cat([ends, perm[(perm != 0) & (perm != r - 1)]])[:u]
        ids = ids[torch.randperm(u, generator=gen, device=dev)]  # row 0 / the last row at random ranks
        everything = torch.arange(r, device=dev)
        group.set_rows([("deep_%d" % g, everything, torch.full((r, T.D), NAN, device=dev)),
                        ("wide_%d" % g, everything, torch.full((r, 1), NAN, device=dev))])
        group.set_rows([("deep_%d" % g, ids, bet_deep[g, :u]), ("wide_%d" % g, ids, bet_wide[g, :u].unsqueeze(1))])
        uniq[g, :u] = ids
    torch.cuda.synchronize()
    return group, uniq


def _rows_struct(group, G, uniq):
    from elasticdl_b200._lib import DeepFMRows

    r = DeepFMRows()
    r.uniq = uniq.data_ptr()
    for fam, bases in (("deep", r.deep_base), ("wide", r.wide_base)):
        for g in range(G):
            tid = group.lookup("%s_%d" % (fam, g))[0]
            base, stride, off, n = ctypes.POINTER(ctypes.c_float)(), ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
            assert group.lib.b200ps_table_rows_ptr(group._h, tid, 0, ctypes.byref(base), ctypes.byref(stride),
                                                   ctypes.byref(off), ctypes.byref(n)) == 0
            bases[g] = ctypes.cast(base, ctypes.c_void_p).value
            assert n.value >= int(uniq[g].max()) + 1
            setattr(r, fam + "_stride", stride.value)
            setattr(r, fam + "_param_off", off.value)
    return r


def run_table_rows(G, B, pattern="zipf", opt=ADAM, seed=0):
    inputs, ref = make_inputs(G, B, pattern, seed=seed)
    group, uniq = _table_state(opt, inputs, seed)
    rows = _rows_struct(group, G, uniq)
    assert (rows.deep_stride, rows.wide_stride) == STRIDES[opt[0]]
    buf = Buffers(G, B)
    buf.load(inputs)
    assert _call("tile", buf.args()) == 0
    torch.cuda.synchronize()
    logits_pull = buf.logits.clone()

    buf.load(inputs)
    buf.bet_wide.fill_(NAN)
    buf.bet_deep.fill_(NAN)
    a = buf.args()
    a.bet_wide = a.bet_deep = None  # not needed with a row source
    a.rows = ctypes.pointer(rows)
    assert _call("tile", a) == 0
    torch.cuda.synchronize()
    label = "table rows %s G=%d B=%d %s:" % (opt[0], G, B, pattern)
    assert torch.equal(buf.logits, logits_pull), label
    got = {"logits": buf.logits, "loss": buf.loss, "grads": buf.grads, "gsum_wide": buf.gsum_wide,
           "gsum_deep": buf.gsum_deep}
    T.check(got, ref, label=label, n_sm=_n_sm())
    dead = torch.arange(B, device=buf.inv.device).unsqueeze(0) >= inputs[1].unsqueeze(1).long()
    assert torch.isnan(buf.gsum_wide[dead]).all(), label
    assert torch.isnan(buf.gsum_deep[dead]).all(), label
    group.close()


@gpu
@pytest.mark.parametrize("B", SHAPES_B + ["262144"])
@pytest.mark.parametrize("G", [1, 5, 33, 38])
def test_table_rows_shapes(G, B):
    run_table_rows(G, _batch(B), seed=G)


@gpu
@pytest.mark.parametrize("B", ["33", "tile_wave2", "32768"])
@pytest.mark.parametrize("pattern", ["equal", "distinct", "zipf", "lanes", "straddle"])
def test_table_rows_id_patterns(pattern, B):
    run_table_rows(38, _batch(B), pattern=pattern, seed=11)


@gpu
@pytest.mark.parametrize("B", ["33", "tile_wave2", "32768"])
@pytest.mark.parametrize("G", [1, 38])
def test_table_rows_sgd_records(G, B):
    run_table_rows(G, _batch(B), opt=SGD, seed=17)


@gpu
def test_row_source_refused_where_it_does_not_apply():
    """Forward-only, fused and mma towers refuse a row source; a hashed table, a dense parameter and a raw buffer
    have no record slab to hand out."""
    from elasticdl_b200 import _lib
    from elasticdl_b200.ps import PSGroup

    G, B = 5, 64
    inputs, _ = make_inputs(G, B, seed=5)
    group, uniq = _table_state(ADAM, inputs, 5)
    rows = _rows_struct(group, G, uniq)
    buf = Buffers(G, B)
    buf.load(inputs)
    L = _lib.lib()
    for tower, name in (("forward_tile", b"forward-only tile tower"), ("fused", b"fused tower"), ("mma", b"mma tower")):
        a = buf.args(not tower.startswith("forward"))
        a.rows = ctypes.pointer(rows)
        assert _call(tower, a) == -1, tower
        assert name + b" reads pulled rows only" in L.b200_deepfm_last_error(), (tower, L.b200_deepfm_last_error())
    torch.cuda.synchronize()
    assert torch.isnan(buf.logits).all()
    group.close()

    group = PSGroup(1, *ADAM, device=0)
    ids = [group.register_table("hashed", 8, "zero", expected_rows=100),
           group.register_dense("dense", (4, 4), 0),
           _lib.check(group.lib.b200ps_raw_register(group._h, b"raw", 1024))]
    group.commit()
    base, n = ctypes.POINTER(ctypes.c_float)(), ctypes.c_int64()
    for tid in ids:
        assert group.lib.b200ps_table_rows_ptr(group._h, tid, 0, ctypes.byref(base), ctypes.byref(n), ctypes.byref(n),
                                               ctypes.byref(n)) == _lib.EINVAL
    group.close()


def _train(row_source, mode, rows, B, steps):
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, HostFeeder, synthetic_batch

    batches = [synthetic_batch(B, 60 + i, torch.device("cuda", 0), "zipf", group_rows=rows) for i in range(steps)]
    group = PSGroup(1, *ADAM, device=0)
    # no initial set_rows: the created-row bitmaps then record exactly the rows the steps touched
    eng = DeepFMPSEngine(group, B, group_rows=rows, init_rows=False, row_source=row_source)
    assert eng.row_source == row_source
    losses = []
    if mode == "eager":
        for ids, dense, labels in batches:
            losses.append(float(eng.step(ids, dense, labels)))
    else:
        feeder = HostFeeder(eng, 3, lookahead=True)
        host = [tuple(t.cpu().pin_memory() for t in b) for b in batches]
        feeder.submit(*host[0])
        feeder.submit(*host[1])
        for i in range(steps):
            if i + 2 < steps:
                feeder.submit(*host[i + 2])
            losses.append(float(feeder.run_next()))
    torch.cuda.synchronize()
    group.check()
    sizes = [group.table_size(n) for n in eng.wide_names + eng.deep_names]
    state = []
    for names in (eng.wide_names, eng.deep_names):
        for n, r in zip(names, rows):
            state += [group.slot_rows(n, torch.arange(r), k).cpu().numpy() for k in range(3)]
    d = group.pull_dense([n for n, _ in eng.params])
    state += [d[n].cpu().numpy() for n, _ in eng.params]
    group.close()
    return losses, sizes, state


@gpu
@pytest.mark.parametrize("mode", ["eager", "lookahead_graph"])
def test_engine_table_rows_match_pulled_rows(mode):
    rows, B, steps = [11, 700, 5000, 9, 64, 100000], 4096, 5
    l0, n0, s0 = _train("pull", mode, rows, B, steps)
    l1, n1, s1 = _train("table", mode, rows, B, steps)
    assert n0 == n1, (n0, n1)
    assert 0 < sum(n1) < 2 * sum(rows)
    assert np.allclose(l0, l1, rtol=1e-5, atol=0), (l0, l1)
    for a, b in zip(s0, s1):
        assert np.allclose(a, b, rtol=0, atol=2e-4), float(np.abs(a - b).max())


@gpu
def test_engine_row_source_auto():
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    rows = [11, 700, 5000]
    for n_shards, kw, want in ((1, {}, "table"), (1, {"paired": True}, "pull"), (2, {}, "pull"),
                               (1, {"tower": "torch"}, "pull"), (1, {"tower": "fused"}, "pull"),
                               (1, {"group_rows": [7] * 39}, "pull")):
        group = PSGroup(n_shards, *ADAM, device=0)
        eng = DeepFMPSEngine(group, 64, **dict({"group_rows": rows}, **kw))
        assert eng.row_source == want, (n_shards, kw)
        group.close()
    group = PSGroup(2, *ADAM, device=0)
    with pytest.raises(ValueError):
        DeepFMPSEngine(group, 64, group_rows=rows, row_source="table")
    group.close()


def test_resolve_row_source():
    from elasticdl_b200.workloads.deepfm import resolve_row_source

    assert resolve_row_source("auto", "tile", 1, "direct", False) == "table"
    for args in (("fused", 1, "direct", False), ("torch", 1, "direct", False), ("tile", 2, "direct", False),
                 ("tile", 2, "owner", False), ("tile", 1, "direct", True)):
        assert resolve_row_source("auto", *args) == "pull", args
        assert resolve_row_source("pull", *args) == "pull", args
        with pytest.raises(ValueError):
            resolve_row_source("table", *args)
