"""Hashed embedding tables (unbounded ids: an Embedding without input_dim, FrappeDeepFMEngine(input_dim=None), every
table a checkpoint restore registers) at the places open addressing goes wrong: ids that share a home slot, probe
chains that wrap past the last slot, many colliding new ids claimed in one launch, one new id at thousands of
positions of one pull, ids equal in their low 32 bits, 0 and 2^63 - 1, a table filled to its last slot, and a
default-sized table's id walk.  oracle/hashed_oracle.py crafts the ids on the host and reads back the slot each id
landed in: a "uniform" hashed table draws a row's initial values by slot.  Then every optimizer kind at every row
width updates such ids bit for bit like the oracle, the Keras kinds also on the unrolled flat push, and a
checkpoint of such a table restores at another shard count."""
import functools
import zlib

import numpy as np
import pytest
import torch

from oracle import hashed_oracle as H
from oracle import ps_oracle as O
from tests import test_gpu_keras_optimizers as KO
from tests import test_gpu_parity as P

pytestmark = pytest.mark.gpu
F = np.float32
SGD = ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;")
SEED = 0  # PSGroup's default seed
DIMS = (1, 4, 8, 10, 64)  # k_push_rows / k_rows_copy at VPT 0 (1, 10: ten chunks), 1 (4) and 2 (8, 64: eight chunks)
PER_SHARD = 300  # expected rows per shard of the small tables: 1024 slots per shard
I64_MAX = 2 ** 63 - 1


def new_group(n_shards, opt=SGD):
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient

    group = PSGroup(n_shards, *opt, device=0, seed=SEED)
    return group, PSClient(group)


def register(group, specs, expected_rows):
    for name, dim, init in specs:
        group.register_table(name, dim, init, None, expected_rows=expected_rows)
    group.commit()


@functools.lru_cache(maxsize=None)
def crafted(n_shards, slots):
    """Per shard: a run of 5 ids with one home slot in the middle, a run of 5 whose home is the last slot (their
    chain wraps to slots 0..3), and 3 ids equal in their low 32 bits with one home slot; then 0 and 2^63 - 1.
    Cached: callers do not modify the arrays."""
    out = {}
    for s in range(n_shards):
        h = 300 + 97 * s
        out[s] = {"run": (h, H.craft(5, slots, n_shards, s, h)),
                  "wrap": (slots - 1, H.craft(5, slots, n_shards, s, slots - 1)),
                  "twins": (700 - 13 * s, H.craft(3, slots, n_shards, s, 700 - 13 * s, start=1 + s,
                                                  low32=(0x2468ACE1 * n_shards + s) & 0xFFFFFFFF))}
    special = np.array([0, I64_MAX], dtype=np.int64)
    return out, special


def pool_of(runs, special):
    ids = np.concatenate([ids for per in runs.values() for _, ids in per.values()] + [special])
    assert len(np.unique(ids)) == len(ids)
    return ids


def init_rows(name, shard, slots, dim, which):
    return H.uniform_init(H.shard_seed(SEED, name, shard), np.asarray(which, dtype=np.int64)[:, None],
                          np.arange(dim, dtype=np.int64)[None, :])


def _q(rng, *shape):
    return (rng.randint(-256, 257, shape) / 64.0).astype(F)


def _grid(rng, *shape):  # exact under p - 0.5 * g with g on the 1/64 grid
    return (rng.randint(-64, 65, shape) / 8.0).astype(F)


def all_table_ids(group, name):
    return np.sort(np.concatenate([group.table_ids(name, s).cpu().numpy() for s in range(group.n_shards)]))


# ------------------------------------------------------------------ placement and dict semantics
@pytest.mark.parametrize("n_shards", [1, 2, 3, 4])
def test_sequential_colliding_inserts_take_consecutive_slots_and_keep_their_own_rows(n_shards):
    """One new id per launch: the j-th id of a run with home slot h lands at (h + j) mod slots, across the last slot
    too, in every table of the launch (k_rows_copy reads at VPT 0, 1, 2), created by pull_rows or by slot_rows alike.
    Then set_rows, pulls with repeats and pushes each address that id's own row; ids equal in their low 32 bits are
    distinct rows; a negative id (INT64_MIN is the empty-slot key) raises and creates nothing."""
    from elasticdl_b200.common.tensor_utils import Tensor

    group, client = new_group(n_shards)
    names = ["u%d" % d for d in DIMS]
    register(group, [(n, d, "uniform") for n, d in zip(names, DIMS)], PER_SHARD * n_shards)
    slots = H.hashed_slots(PER_SHARD * n_shards, n_shards)
    assert slots == 1024
    runs, special = crafted(n_shards, slots)
    model = H.GroupModel(slots, n_shards)
    order, want_slot = [], {}
    for s in range(n_shards):
        for kind in ("run", "wrap"):
            h, ids = runs[s][kind]
            for j, i in enumerate(ids.tolist()):
                order.append(i)
                want_slot[i] = (h + j) & (slots - 1)
    order += runs_ids(runs, "twins") + special.tolist()
    for j, i in enumerate(order):
        s = int(H.shard_of(np.array([i]), n_shards)[0])
        slot = int(model.place([i])[0])
        assert want_slot.get(i, slot) == slot, "crafted run does not collide on the host"
        before = [group.table_size(n) for n in names]
        if j % 2 == 0:
            rows = [r.cpu().numpy() for r in group.pull_rows([(n, [i]) for n in names])]
        else:
            rows = [group.slot_rows(n, [i], 0).cpu().numpy() for n in names]
        for n, d, r in zip(names, DIMS, rows):
            assert np.array_equal(r, init_rows(n, s, slots, d, [slot])), (n, i, s, slot)
        assert [group.table_size(n) for n in names] == [b + 1 for b in before], (i, j)
    for s in range(n_shards):  # the twins of a shard hold three different slots
        tw = runs[s]["twins"][1]
        assert len({model.shards[s].slot[int(i)] for i in tw}) == 3
    created = model.ids()
    for n in names:
        assert np.array_equal(all_table_ids(group, n), created), n
        for s in range(n_shards):
            assert (H.shard_of(group.table_ids(n, s).cpu().numpy(), n_shards) == s).all()

    rng = np.random.RandomState(n_shards)
    perm = rng.permutation(created)
    vals = {n: _grid(rng, len(perm), d) for n, d in zip(names, DIMS)}
    group.set_rows([(n, perm, vals[n]) for n in names])  # k_rows_copy writes, one launch per class
    group.check()
    pos = {int(i): k for k, i in enumerate(perm.tolist())}
    q = rng.choice(created, 3000)
    got = group.pull_rows([(n, q) for n in names])
    for n, r in zip(names, got):
        assert np.array_equal(r.cpu().numpy(), vals[n][[pos[int(i)] for i in q.tolist()]]), n
    g = {n: _q(rng, len(perm), d) for n, d in zip(names, DIMS)}
    acc, _ = client.push_gradients([], [Tensor(n, g[n], perm) for n in names], 0.5, [0] * n_shards)
    assert acc
    for n in names:
        want = vals[n] - F(0.5) * g[n]
        assert np.array_equal(client.pull_embedding_vectors(n, perm), want), n
        assert group.table_size(n) == len(created), n

    for bad in ([-1], [-2 ** 63], [-(2 ** 40) - 5, -2 ** 63 + 1]):
        group.pull_rows([(names[2], bad)])
        with pytest.raises(ValueError, match="negative"):
            group.check()
        group.set_rows([(names[3], bad, np.zeros((len(bad), DIMS[3]), F))])
        with pytest.raises(ValueError, match="negative"):
            group.check()
    group.check()
    for n in names:
        assert group.table_size(n) == len(created) and np.array_equal(all_table_ids(group, n), created), n
    group.close()


def runs_ids(runs, kind):
    return [i for s in sorted(runs) for i in runs[s][kind][1].tolist()]


@pytest.mark.parametrize("n_shards", [1, 2, 3, 4])
def test_one_launch_of_colliding_new_ids_claims_one_contiguous_run(n_shards):
    """300 new ids per shard with one home slot in ONE pull_rows launch (shard 0's run wraps past the last slot): they
    occupy exactly the 300 slots from the home slot on, one each, in some order; a second pull returns the same rows.
    Then one new id of the same home at 10^4 positions of one pull (PSGroup.pull_rows does not deduplicate): it is
    created once, past the end of the run, and every position reads its row."""
    group, _ = new_group(n_shards)
    register(group, [("u", 8, "uniform")], PER_SHARD * n_shards)
    slots = H.hashed_slots(PER_SHARD * n_shards, n_shards)
    homes = [slots - 100] + [200 + 150 * s for s in range(1, n_shards)]
    runs = [H.craft(300, slots, n_shards, s, homes[s]) for s in range(n_shards)]
    rng = np.random.RandomState(10 + n_shards)
    ids = rng.permutation(np.concatenate(runs))
    (rows,) = group.pull_rows([("u", ids)])
    group.check()
    rows = rows.cpu().numpy()
    sh = H.shard_of(ids, n_shards)
    for s in range(n_shards):
        got = np.sort(H.slots_of(SEED, "u", s, rows[sh == s], slots))
        want = np.sort((homes[s] + np.arange(300)) & (slots - 1))
        assert np.array_equal(got, want), s
        assert group.table_size("u", s) == 300
        assert np.array_equal(np.sort(group.table_ids("u", s).cpu().numpy()), np.sort(runs[s]))
    assert group.table_size("u") == 300 * n_shards
    (again,) = group.pull_rows([("u", ids)])
    assert np.array_equal(again.cpu().numpy(), rows)

    new = H.craft(1, slots, n_shards, 0, homes[0], start=int(runs[0].max()) + 1)
    q = np.empty(12_000, dtype=np.int64)
    at = rng.permutation(len(q))[:10_000]
    q[:] = rng.choice(ids, len(q))
    q[at] = new[0]
    (rows2,) = group.pull_rows([("u", q)])
    group.check()
    rows2 = rows2.cpu().numpy()
    assert group.table_size("u") == 300 * n_shards + 1
    assert np.array_equal(rows2[at], np.repeat(init_rows("u", 0, slots, 8, [(homes[0] + 300) & (slots - 1)]), 10_000, 0))
    rest = np.setdiff1d(np.arange(len(q)), at)
    pos = {int(i): k for k, i in enumerate(ids.tolist())}
    assert np.array_equal(rows2[rest], rows[[pos[int(i)] for i in q[rest].tolist()]])
    group.close()


def test_exactly_full_table():
    """One shard at the 1024-slot minimum: 1000 ids (colliding runs, a wrapped run, twins) created over four launches,
    then one launch with 50 of them, 24 new ids and one more.  Exactly one new id finds no slot: check() raises
    "full" once and is clear afterwards; the other ids of that launch read their rows; all 1024 slots are held by
    distinct ids; later pulls and pushes of those 1024 ids are exact."""
    from elasticdl_b200.common.tensor_utils import Tensor

    group, client = new_group(1)
    register(group, [("u", 8, "uniform")], 512)
    slots = H.hashed_slots(512, 1)
    assert slots == 1024
    rng = np.random.RandomState(1024)
    special = [H.craft(40, slots, 1, 0, 1000), H.craft(30, slots, 1, 0, 500), H.craft(3, slots, 1, 0, 9, low32=0x0BADF00D),
               np.array([0, I64_MAX], dtype=np.int64)]
    fill = np.unique(rng.randint(1, 2 ** 62, 1200).astype(np.int64))
    fill = rng.permutation(np.setdiff1d(fill, np.concatenate(special)))
    ids = np.concatenate(special + [fill])[:1025]
    assert len(np.unique(ids)) == 1025
    first, new = ids[:1000], ids[1000:]
    slot_of = {}
    for chunk in np.array_split(rng.permutation(first), 4):
        (rows,) = group.pull_rows([("u", chunk)])
        got = H.slots_of(SEED, "u", 0, rows.cpu().numpy(), slots)
        assert (got >= 0).all()
        slot_of.update(zip(chunk.tolist(), got.tolist()))
    group.check()
    assert group.table_size("u") == 1000 and len(set(slot_of.values())) == 1000

    old = rng.choice(first, 50, replace=False)
    q = rng.permutation(np.concatenate([old, new]))
    out = torch.full((len(q), 8), -7.0, dtype=torch.float32, device="cuda")
    t_q = torch.from_numpy(q).cuda()
    group._run_segs(group.lib.b200ps_pull_rows, [(group.lookup("u")[0], len(q), t_q, None, out)])
    with pytest.raises(ValueError, match="full"):
        group.check()
    group.check()
    out = out.cpu().numpy()
    is_new = np.isin(q, new)
    missed = (out == -7.0).all(1)
    assert missed.sum() == 1 and is_new[missed].all()
    got = H.slots_of(SEED, "u", 0, out[~missed], slots)
    assert (got >= 0).all()
    for i, s in zip(q[~missed].tolist(), got.tolist()):
        assert slot_of.setdefault(i, s) == s, i
    assert sorted(slot_of.values()) == list(range(slots))
    placed = np.array(sorted(slot_of), dtype=np.int64)
    assert group.table_size("u") == slots
    assert np.array_equal(np.sort(group.table_ids("u", 0).cpu().numpy()), placed)

    (rows,) = group.pull_rows([("u", placed)])
    group.check()
    want = init_rows("u", 0, slots, 8, [slot_of[int(i)] for i in placed.tolist()])
    assert np.array_equal(rows.cpu().numpy(), want)
    g = _q(rng, len(placed), 8)
    acc, _ = client.push_gradients([], [Tensor("u", g, placed)], 0.5, [0])
    assert acc
    assert np.array_equal(client.pull_embedding_vectors("u", placed), want - F(0.5) * g)
    group.pull_rows([("u", q[missed])])  # still no room
    with pytest.raises(ValueError, match="full"):
        group.check()
    group.check()
    assert group.table_size("u") == slots
    group.close()


def test_table_ids_on_a_default_sized_table():
    """A hashed table of the default size (2^21 slots at one shard: the id walk runs four grid passes) with ids at
    slot 0, in the middle and at the last slot, plus 200 000 random ids: table_ids / table_size are exactly the
    created set."""
    from elasticdl_b200.ps.group import DEFAULT_CAPACITY

    group, _ = new_group(1)
    group.register_table("big", 4, "uniform", None)
    group.commit()
    slots = H.hashed_slots(DEFAULT_CAPACITY, 1)
    assert slots == 1 << 21
    at = [0, slots // 2, slots - 1]
    edge = np.concatenate([H.craft(1, slots, 1, 0, h) for h in at])
    (rows,) = group.pull_rows([("big", edge)])
    group.check()
    assert np.array_equal(rows.cpu().numpy(), init_rows("big", 0, slots, 4, at))
    rng = np.random.RandomState(21)
    bulk = np.setdiff1d(np.unique(rng.randint(0, 2 ** 62, 200_000).astype(np.int64)), edge)
    group.pull_rows([("big", rng.permutation(bulk))])
    group.check()
    created = np.union1d(edge, bulk)
    got = group.table_ids("big", 0).cpu().numpy()
    assert len(got) == len(created) and np.array_equal(np.sort(got), created)
    assert group.table_size("big") == len(created)
    group.close()


# ------------------------------------------------------------------ every optimizer kind at every row width
KINDS = {**{k: (P.make_pair, P.OPTS[k]) for k in P.OPTS}, **{k: (KO.make_pair, KO.KERAS_OPTS[k]) for k in KO.KERAS_OPTS}}


def _init_slot_value(opt_args, k):
    return 0.1 if "initial_accumulator_value=0.1" in opt_args and k == 0 else 0.0


@pytest.mark.parametrize("opt", list(KINDS))
@pytest.mark.parametrize("n_shards", [1, 3])
def test_every_optimizer_every_row_width_on_colliding_ids(opt, n_shards):
    """k_push_rows<OPT, VPT> at VPT 0, 1 and 2 and rows of one to ten chunks, for all 13 kinds: four pushes of unique
    ids (colliding runs, wrapped runs, twins, 0 and 2^63 - 1; some created by a pull first, the others by their first
    push) into five "zero" hashed tables give the oracle's params and slots bit for bit; ids no push named keep their
    rows and their slots' initial values (FTRL's accumulator starts at 0.1 in every slot)."""
    from elasticdl_b200.common.tensor_utils import Tensor

    make, (ot, oa) = KINDS[opt]
    group, client, oc = make(n_shards, opt)
    names = ["h%d" % d for d in DIMS]
    register(group, [(n, d, "zero") for n, d in zip(names, DIMS)], PER_SHARD * n_shards)
    oc.push_embedding_table_infos([P.oinfo(n, d) for n, d in zip(names, DIMS)])
    slots = H.hashed_slots(PER_SHARD * n_shards, n_shards)
    runs, special = crafted(n_shards, slots)
    pool = pool_of(runs, special)
    rng = np.random.RandomState(zlib.crc32(repr(("hashed", opt, n_shards)).encode()))
    pool = rng.permutation(pool)
    by_pull, never = pool[: len(pool) // 3], pool[: len(pool) // 8]
    for n in names:
        assert np.array_equal(client.pull_embedding_vectors(n, by_pull), oc.pull_embedding_vectors(n, by_pull))
    pushable = np.setdiff1d(pool, never)
    lr_own = float(oa.split("learning_rate=")[1].split(";")[0])
    versions = [0] * n_shards
    for step in range(4):
        ids = rng.permutation(pushable)[: len(pushable) if step == 0 else int(len(pushable) * 0.7)]
        grads = {n: _q(rng, len(ids), d) for n, d in zip(names, DIMS)}
        lr = 0.5 * lr_own if step == 2 else 0.0
        a1 = client.push_gradients([], [Tensor(n, grads[n].copy(), ids.copy()) for n in names], lr, versions)
        a2 = oc.push_gradients([], [O.Tensor(n, grads[n].copy(), ids.copy()) for n in names], lr, list(versions))
        assert a1 == a2 == (True, step + 1)
        versions = [a1[1]] * n_shards
    slot_names = oc.servers[0].opt.slot_names
    for n, d in zip(names, DIMS):
        created = np.sort(np.concatenate([s.tables[n].keys() for s in oc.servers]))
        assert np.array_equal(created, np.sort(pool)), n
        assert group.table_size(n) == len(pool), n
        assert np.array_equal(all_table_ids(group, n), created), n
        assert np.array_equal(client.pull_embedding_vectors(n, pool), oc.pull_embedding_vectors(n, pool)), n
        sh = H.shard_of(pool, n_shards)
        for k, sn in enumerate(slot_names):
            got = group.slot_rows(n, pool, k + 1).cpu().numpy()
            want = np.empty_like(got)
            for s in oc.servers:
                want[sh == s.id] = s.opt.table_slots[sn][n].get(pool[sh == s.id])
            assert np.array_equal(got, want), (n, sn)
            untouched = np.isin(pool, never)
            assert (got[untouched] == F(_init_slot_value(oa, k))).all(), (n, sn)
        assert not client.pull_embedding_vectors(n, never).any(), n
    group.close()


@pytest.mark.parametrize("opt", list(KO.KERAS_OPTS))
@pytest.mark.parametrize("n_shards", [1, 3])
def test_keras_kinds_on_the_unrolled_flat_push(opt, n_shards):
    """k_push_flat<OPT, 2, NS> for RMSprop (four variants), Adadelta, Adamax and Nadam: the push every DeepFM
    benchmark step runs, millions of lane-items, two rows in flight per thread."""
    P._flat_launch_case(opt, n_shards, large=True, make_pair=KO.make_pair)


# ------------------------------------------------------------------ checkpoint
def test_checkpoint_of_colliding_ids_restores_at_another_shard_count(tmp_path):
    """A hashed table holding colliding runs, wrapped runs, twins, 0 and 2^63 - 1 saved at two shards and restored at
    three: load registers it hashed again for max(2 x saved, 65536) rows, every row comes back, each shard holds its
    own ids, and a new id lands at its home slot of the restored 65536-slot shard."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.ps import checkpoint as ck
    from elasticdl_b200.worker.ps_client import PSClient

    group, client = new_group(2, P.OPTS["adam"])
    register(group, [("hashed", 8, "uniform")], PER_SHARD * 2)
    runs, special = crafted(2, H.hashed_slots(PER_SHARD * 2, 2))
    pool = pool_of(runs, special)
    rng = np.random.RandomState(23)
    vals = rng.randn(len(pool), 8).astype(F)
    group.set_rows([("hashed", pool, vals)])
    group.check()
    assert group.table_size("hashed") == len(pool)
    vdir = ck.save(group, str(tmp_path))
    group.close()

    g3 = PSGroup(3, *P.OPTS["adam"], device=0, seed=SEED)
    c3 = PSClient(g3)
    ck.load(g3, c3, vdir)
    assert np.array_equal(c3.pull_embedding_vectors("hashed", pool), vals)
    for s in range(3):
        assert np.array_equal(np.sort(g3.table_ids("hashed", s).cpu().numpy()), np.sort(pool[pool % 3 == s])), s
    slots = H.hashed_slots(max(2 * len(pool), 1 << 16), 3)
    assert slots == 1 << 16
    model = H.GroupModel(slots, 3)
    model.place(pool)
    new = H.craft(1, slots, 3, 1, 12345)
    (row,) = g3.pull_rows([("hashed", new)])
    g3.check()
    assert np.array_equal(row.cpu().numpy(), init_rows("hashed", 1, slots, 8, model.place(new)))
    assert g3.table_size("hashed") == len(pool) + 1
    g3.close()
