"""GPU parity of the parameter-server update kernels that the small-size optimizer tests do not reach, against
the CPU oracle, bit for bit:

* paired records (k_pair_pull / k_pair_push<OPT>, DeepFMPSEngine(paired=True)) for every optimizer: the
  per-slot-count lane layouts, the pair's initial record contents, pads that no push may touch;
* the fused dense reduce (k_push_dense_reduce<OPT, VEC, TWICE>) over 1..16 replica gradients, both vector widths,
  the AMSGrad quirk-Q1 instance, multiply (allreduce postscale) and divide (sync-SGD average) semantics;
* sync-SGD through PSClient: dense gradients averaged as fl(fl(sum) / grads_to_wait) (python/ps/servicer.py:207)."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ps_oracle as O
from tests.test_gpu_parity import OPTS, make_pair, oinfo

pytestmark = pytest.mark.gpu
F = np.float32


class _DevFloats:
    """A float32 device array at a raw address, for torch.as_tensor (no copy)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "<f4", "data": (int(ptr), False),
                                         "version": 3}


def _record_slab(group, tid, shard):
    """The record slab of a direct-indexed table on `shard` as a [rows, row_stride] host copy (does not mark rows)."""
    base, stride, off, rows = ctypes.POINTER(ctypes.c_float)(), ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
    assert group.lib.b200ps_table_rows_ptr(group._h, tid, shard, ctypes.byref(base), ctypes.byref(stride),
                                           ctypes.byref(off), ctypes.byref(rows)) == 0
    ptr = ctypes.cast(base, ctypes.c_void_p).value
    dev = torch.as_tensor(_DevFloats(ptr, rows.value * stride.value), device=group.device)
    torch.cuda.synchronize()
    return dev.cpu().numpy().reshape(rows.value, stride.value).copy()


def _oracle_rows(oc, name, ids, slot=None):
    """Rows (slot None) or optimizer-slot rows of `ids` from the oracle shards (id % N routing)."""
    out = np.empty((len(ids), oc.servers[0].tables[name].dim), dtype=F)
    n = len(oc.servers)
    for s in oc.servers:
        m = ids % n == s.id
        t = s.tables[name] if slot is None else s.opt.table_slots[s.opt.slot_names[slot]][name]
        out[m] = t.get(ids[m])
    return out


# ------------------------------------------------------------------ paired records
PAIR_CAPS = (7, 3000, 200_003)  # the big pair's segment makes the grid loop


def _check_pairs_against_oracle(group, oc, names, seen, n_slots):
    for (a, b), ids in zip(names, seen):
        assert np.array_equal(group.pull_rows([(a, ids)])[0].cpu().numpy(), _oracle_rows(oc, a, ids)), a
        assert np.array_equal(group.pull_rows([(b, ids)])[0].cpu().numpy(), _oracle_rows(oc, b, ids)), b
        for k in range(n_slots):
            for name in (a, b):
                got = group.slot_rows(name, ids, k + 1).cpu().numpy()
                assert np.array_equal(got, _oracle_rows(oc, name, ids, k)), (name, k)


@pytest.mark.parametrize("opt", list(OPTS))
@pytest.mark.parametrize("n_shards", [1, 3])
def test_paired_records_every_optimizer_match_oracle(opt, n_shards):
    """Three pairs (dim-8 A + dim-1 B in one record per id) in one b200ps_push_rows_pair launch per round, device-side
    live counts that are not multiples of the rows per warp, an explicit and the optimizer's own lr: params and every
    slot of both halves equal the oracle (each pair = two ordinary tables) bit for bit after every round."""
    group, client, oc = make_pair(n_shards, opt)
    lib = group.lib
    names = [("pa%d" % i, "pb%d" % i) for i in range(len(PAIR_CAPS))]
    tids = [group.register_pair(a, b, c) for (a, b), c in zip(names, PAIR_CAPS)]
    group.commit()
    oc.push_embedding_table_infos([oinfo(n, d) for a, b in names for n, d in ((a, 8), (b, 1))])
    n_slots = len(oc.servers[0].opt.slot_names)
    sec = 12  # record section: [A(8) | B(1) | pad(3)]
    init = [0.0] * (n_slots + 1)
    if opt.startswith("ftrl"):
        init[1] = float(oc.servers[0].opt.init_accum)

    # 1. the fresh records, every float of every section: A's and B's columns at the slot's initial value, pads 0
    slabs = {}
    for (ta, _), (a, _) in zip(tids, names):
        for s in range(n_shards):
            slab = _record_slab(group, ta, s)
            assert slab.shape[1] == sec * (n_slots + 1)
            for k in range(n_slots + 1):
                part = slab[:, k * sec:(k + 1) * sec]
                assert (part[:, :9] == F(init[k])).all(), (a, s, k)
                assert (part[:, 9:] == 0).all(), (a, s, k)
            slabs[(a, s)] = slab
    # ... and through the pull paths: every row of the small pairs, the lower half (and the last row) of the big one,
    # so that the pushes below create rows of their own
    seen = [np.arange(c, dtype=np.int64) for c in PAIR_CAPS[:-1]]
    seen.append(np.append(np.arange(PAIR_CAPS[-1] // 2), PAIR_CAPS[-1] - 1).astype(np.int64))
    _check_pairs_against_oracle(group, oc, names, seen, n_slots)

    rng = np.random.RandomState(len(opt) * 10 + n_shards)
    seg_n = [7, 2000, 150_000]
    live_n = [5, 1997, 149_995]  # odd: not a multiple of 8 / 4 / 2 rows per warp
    rows_cap = [(c + n_shards - 1) // n_shards for c in PAIR_CAPS]
    for rnd, lr in enumerate((0.0, 0.05, 0.0, 0.0)):
        segs = []
        for cap, n, live in zip(PAIR_CAPS, seg_n, live_n):
            ids = rng.permutation(cap)[:n].astype(np.int64)
            ids = np.concatenate([[0, cap - 1], ids[(ids != 0) & (ids != cap - 1)]])[:n]
            live_ids = ids[:live].copy()
            rng.shuffle(live_ids)
            ids[:live] = live_ids  # 0 and cap - 1 at random live positions
            segs.append((ids, live))
        bad = None
        if rnd == 3:  # one id past the table in the middle segment: reported, every other row still updated
            bad = (1, 17)
            segs[1][0][17] = rows_cap[1] * n_shards + 5
        items, rows_b, keep, ograds = [], [], [], []
        for (ta, _), (ids, live), (a, b) in zip(tids, segs, names):
            ga = (rng.randn(len(ids), 8) * 0.1).astype(F)
            gb = (rng.randn(len(ids)) * 0.1).astype(F)
            t_ids = torch.from_numpy(ids).cuda()
            n_dev = torch.tensor([live], dtype=torch.int32, device="cuda")
            t_ga, t_gb = torch.from_numpy(ga).cuda(), torch.from_numpy(gb).cuda()
            keep.append((t_ids, n_dev, t_ga, t_gb))
            items.append((ta, len(ids), t_ids, n_dev, t_ga))
            rows_b.append(t_gb)
            ok = np.ones(live, dtype=bool)
            if bad is not None and a == names[bad[0]][0]:
                ok[bad[1]] = False
            ograds += [O.Tensor(a, ga[:live][ok].copy(), ids[:live][ok].copy()),
                       O.Tensor(b, gb[:live][ok].reshape(-1, 1).copy(), ids[:live][ok].copy())]
        group.push_begin(lr, [0] * n_shards)
        group.pair_call(lib.b200ps_push_rows_pair, items, rows_b)
        group.push_end()
        if bad is None:
            group.check()
        else:
            with pytest.raises(ValueError):
                group.check()
        oc.push_gradients([], ograds, lr, [0] * n_shards)
        # created rows: the pushes mark theirs in both halves' bitmaps, rows past the live counts stay unmarked
        for a, b in names:
            for name in (a, b):
                assert group.table_size(name) == sum(len(s.tables[name]) for s in oc.servers), (rnd, name)
        for i, (ids, live) in enumerate(segs):
            valid = ids[ids < PAIR_CAPS[i]]
            seen[i] = np.union1d(seen[i], valid)
        _check_pairs_against_oracle(group, oc, names, seen, n_slots)
        # the pads of every record section are untouched
        for (ta, _), (a, _) in zip(tids, names):
            for s in range(n_shards):
                slab = _record_slab(group, ta, s)
                for k in range(n_slots + 1):
                    assert np.array_equal(slab[:, k * sec + 9:(k + 1) * sec], slabs[(a, s)][:, k * sec + 9:(k + 1) * sec])

    # 2. the pair pull (rows past the live count untouched) == the flat pulls of A and of B == the oracle
    items, rows_b, keep = [], [], []
    for (ta, _), cap, n, live in zip(tids, PAIR_CAPS, seg_n, live_n):
        ids = rng.permutation(cap)[:n].astype(np.int64)
        t_ids = torch.from_numpy(ids).cuda()
        n_dev = torch.tensor([live], dtype=torch.int32, device="cuda")
        ra = torch.full((n, 8), -7.0, device="cuda")
        rb = torch.full((n,), -7.0, device="cuda")
        keep.append((ids, live, t_ids, n_dev, ra, rb))
        items.append((ta, n, t_ids, n_dev, ra))
        rows_b.append(rb)
    group.pair_call(lib.b200ps_pull_rows_pair, items, rows_b)
    group.check()
    for (a, b), (ids, live, t_ids, _, ra, rb) in zip(names, keep):
        ga, gb = ra.cpu().numpy(), rb.cpu().numpy()
        fa, fb = group.pull_rows([(a, t_ids[:live]), (b, t_ids[:live])])
        assert np.array_equal(ga[:live], fa.cpu().numpy()) and np.array_equal(ga[:live], _oracle_rows(oc, a, ids[:live]))
        assert np.array_equal(gb[:live], fb.cpu().numpy()[:, 0]) and np.array_equal(gb[:live], _oracle_rows(oc, b, ids[:live])[:, 0])
        assert (ga[live:] == -7.0).all() and (gb[live:] == -7.0).all(), a
    group.close()


# ------------------------------------------------------------------ dense reduce
DENSE_SHAPES = {"v4": (2304, 1000), "v1": (37, 7), "v4_offset": (16, 20)}  # v4: the grid loops; v4_offset -> VEC 1


@pytest.mark.parametrize("divide", [False, True], ids=["mul", "div"])
@pytest.mark.parametrize("R", [1, 2, 3, 16])
@pytest.mark.parametrize("opt", list(OPTS) + ["amsgrad_q1"])
def test_dense_reduce_replicas_match_oracle(opt, R, divide):
    """b200ps_push_dense_reduce over R local replica gradients: the fp32 left-to-right sum, times fp32(1/R) or divided
    by R, then the optimizer update -- params and every slot bit for bit after two reduces.  Sizes with numel % 4 == 0
    (128-bit path), numel % 4 != 0, and a multiple of 4 whose last replica is 4 bytes off 16 B alignment (scalar)."""
    q1 = opt == "amsgrad_q1"
    group, _, oc = make_pair(1, "amsgrad" if q1 else opt, reproduce_q1=q1)
    srv = oc.servers[0]
    gen = torch.Generator(device="cuda").manual_seed(R * 31 + len(opt) + int(divide))
    for name, shape in DENSE_SHAPES.items():
        group.register_dense(name, shape, 0)
    group.commit()
    for name, shape in DENSE_SHAPES.items():
        p0 = torch.randn(shape, device="cuda", generator=gen)
        group.set_dense([(name, p0)])
        srv.dense[name] = p0.cpu().numpy().copy()
        srv.opt.init_dense(name, shape)
    scale = F(R) if divide else F(1.0 / R)
    for rnd, lr in enumerate((0.05, 0.0)):
        dense_g = {}
        group.push_begin(lr, [0])
        for name, shape in DENSE_SHAPES.items():
            numel = int(np.prod(shape))
            grads = []
            for r in range(R):
                if name == "v4_offset" and r == R - 1:
                    buf = torch.randn(numel + 4, device="cuda", generator=gen)
                    grads.append(buf[1:1 + numel])
                    assert grads[-1].data_ptr() % 16 == 4
                else:
                    grads.append(torch.randn(numel, device="cuda", generator=gen))
            host = [g.cpu().numpy() for g in grads]
            s = host[0].copy()
            for h in host[1:]:
                s = s + h  # fp32, replica order
            dense_g[name] = (s / scale if divide else s * scale).astype(F).reshape(shape)
            group.push_dense_reduce(name, grads, scale=float(scale), divide=divide)
        group.push_end()
        group.check()
        srv.push_gradients(dense_g, {}, lr, 0)
        for name in DENSE_SHAPES:
            assert np.array_equal(group.pull_dense([name])[name].cpu().numpy(), srv.dense[name]), (rnd, name)
            for k, sn in enumerate(srv.opt.slot_names):
                got = group.slot_dense(name, k + 1).cpu().numpy()
                assert np.array_equal(got, srv.opt.dense_slots[sn][name]), (rnd, name, sn)
    group.close()


def test_dense_reduce_rejects_a_zero_divisor():
    group, _, _ = make_pair(1, "sgd")
    group.register_dense("w", (8,), 0)
    group.commit()
    g = torch.ones(8, device="cuda")
    with pytest.raises(ValueError):
        group.push_dense_reduce("w", [g], scale=0.0, divide=True)
    group.close()


# ------------------------------------------------------------------ sync-SGD through PSClient
@pytest.mark.parametrize("w", [2, 3, 5])
@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_sync_sgd_dense_average_divides_like_the_python_ps(opt, w):
    """grads_to_wait = w pushes are summed in push order and divided by w in fp32 (python/ps/servicer.py:178-211:
    grad / self._grads_to_wait), then applied once; two such rounds.  x * fl(1/w) differs from x / w in the last bit
    for a third of the values at w = 3, so only the division reproduces the Python PS."""
    from elasticdl_b200.common.tensor_utils import Tensor
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient

    ot, oa = OPTS[opt]
    group = PSGroup(1, ot, oa, device=0, use_async=False, grads_to_wait=w)
    client = PSClient(group)
    srv = O.OracleServer(0, ot, oa)
    rng = np.random.RandomState(w * 7 + len(opt))
    shapes = {"k": (64, 33), "b": (37,)}
    client.partition_dense_parameters(shapes.keys())
    params = {n: rng.randn(*s).astype(F) for n, s in shapes.items()}
    client.push_dense_parameters([Tensor(n, v, None) for n, v in params.items()], 0, 0)
    srv.push_model(dense={n: v.copy() for n, v in params.items()})
    version = 0
    for rnd, lr in enumerate((0.1, 0.0)):
        sums = {}
        for i in range(w):
            g = {n: (rng.randn(*s) * 3).astype(F) for n, s in shapes.items()}
            for n in shapes:
                sums[n] = g[n].copy() if i == 0 else sums[n] + g[n]
            acc, ver = client.push_gradients([Tensor(n, v, None) for n, v in g.items()], [], lr, [version])
            assert acc and ver == (version if i < w - 1 else version + 1)
        version += 1
        srv.push_gradients({n: sums[n] / F(w) for n in shapes}, {}, lr, version - 1)
        for n in shapes:
            assert np.array_equal(group.pull_dense([n])[n].cpu().numpy(), srv.dense[n]), (rnd, n)
            for k, sn in enumerate(srv.opt.slot_names):
                assert np.array_equal(group.slot_dense(n, k + 1).cpu().numpy(), srv.opt.dense_slots[sn][n]), (rnd, n, sn)
    group.close()
