"""oracle/hashed_oracle.py, the host restatement the hashed-table GPU tests craft their ids with and read slots
back through, checked on the CPU: its mix64 / uniform_init against ps_oracle.c's oracle_uniform_init, its seeds
against PSGroup's, and the crafted ids against what they claim (one shard, one home slot, equal low 32 bits)."""
import numpy as np

from oracle import hashed_oracle as H
from oracle import ps_oracle as O

EDGE_IDS = [0, 1, 2, 2 ** 31 - 1, 2 ** 31, 2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, 2 ** 40 + 12345, 2 ** 62, 2 ** 63 - 1,
            -1, -2 ** 63, 5 << 32, 7 << 32]
EDGE_SEEDS = [0, 1, 0x9E3779B97F4A7C15, 2 ** 64 - 1, 2 ** 63, 0x0123456789ABCDEF]


def test_uniform_init_matches_the_c_generator_bitwise():
    rng = np.random.RandomState(3)
    ids = EDGE_IDS + rng.randint(-2 ** 63, 2 ** 63 - 1, size=40, dtype=np.int64).tolist()
    seeds = EDGE_SEEDS + [int(s) for s in rng.randint(0, 2 ** 63 - 1, size=6, dtype=np.int64)]
    cols = np.array([0, 1, 7, 63, 1 << 20], dtype=np.int64)
    for seed in seeds:
        got = H.uniform_init(seed, np.array(ids, dtype=np.int64)[:, None], cols[None, :])
        want = np.array([[O.lib.oracle_uniform_init(seed, i, int(c)) for c in cols] for i in ids], dtype=np.float32)
        assert got.dtype == np.float32
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), seed
        assert got.min() >= -0.05 and got.max() < 0.05


def test_mix64_is_the_finaliser_the_generator_uses():
    # uniform_init(seed, id, col) = f(mix64(seed ^ mix64(id * GOLDEN + col))): with id = 0 and col = c the inner
    # argument is c, so two seeds that differ by mix64(c) ^ mix64(c') swap the draws of columns c and c'
    for c0, c1 in ((0, 1), (3, 1000), (2 ** 40, 5)):
        m0, m1 = (int(H.mix64(np.array([c], dtype=np.int64))[0]) for c in (c0, c1))
        seed = 0x5555AAAA5555AAAA
        a = O.lib.oracle_uniform_init(seed, 0, c0)
        b = O.lib.oracle_uniform_init(seed ^ m0 ^ m1, 0, c1)
        assert a == b
    # a fixed point and a known value of the finaliser
    assert int(H.mix64(np.array([0], dtype=np.uint64))[0]) == 0
    x = np.array([1], dtype=np.uint64)
    want = 1
    want ^= want >> 33
    want = want * 0xFF51AFD7ED558CCD & H.MASK64
    want ^= want >> 33
    want = want * 0xC4CEB9FE1A85EC53 & H.MASK64
    want ^= want >> 33
    assert int(H.mix64(x)[0]) == want


def test_seeds_match_the_group():
    from elasticdl_b200.ps.group import table_seed

    for seed in (0, 11, 2 ** 63 + 5):
        for name in ("h", "emb_table_with_a_long_name", "u"):
            assert H.table_seed(seed, name) == table_seed(seed, name)
            for s in range(4):
                assert H.shard_seed(seed, name, s) == table_seed(seed, name) ^ (0x9E3779B97F4A7C15 * (s + 1)) % 2 ** 64


def test_slot_count_and_routing():
    assert H.hashed_slots(1, 1) == 1024
    assert H.hashed_slots(512, 1) == 1024
    assert H.hashed_slots(513, 1) == 2048
    assert H.hashed_slots(1000, 3) == 1024  # ceil(1000 / 3) = 334 -> 668
    assert H.hashed_slots(1 << 20, 1) == 1 << 21
    assert H.hashed_slots(1 << 16, 3) == 1 << 16  # ceil(65536 / 3) = 21846 -> 43692
    assert H.hashed_slots(3073, 3) == 4096  # ceil(3073 / 3) = 1025 -> 2050
    ids = np.array([0, 1, 2, 3, 4, 5, 2 ** 32, 2 ** 63 - 1, 2 ** 33 + 7], dtype=np.int64)
    for n in (1, 2, 3, 4, 8):
        want = np.array([int(i) % n for i in ids.tolist()])
        assert np.array_equal(H.shard_of(ids, n), want), n


def test_crafted_ids_share_shard_and_home_slot():
    for n in (1, 2, 3, 4):
        for s in range(n):
            for slots, home in ((1024, 17), (1024, 1023), (1 << 21, 0)):
                ids = H.craft(4 if slots == 1024 else 1, slots, n, s, home, start=1 + 1000 * s)
                assert (ids > 0).all() and len(np.unique(ids)) == len(ids)
                assert (H.shard_of(ids, n) == s).all() and (H.home_slot(ids, slots) == home).all()
            low = (0x1234567 * n + s) & 0xFFFFFFFF
            tw = H.craft(3, 1024, n, s, 500, start=1, low32=low)
            assert ((tw & 0xFFFFFFFF) == low).all() and len(np.unique(tw >> 32)) == 3
            assert (H.shard_of(tw, n) == s).all() and (H.home_slot(tw, 1024) == 500).all()


def test_probe_model_wraps_and_keeps_order_independent_occupancy():
    run = H.craft(5, 1024, 1, 0, 1022)
    m = H.ShardModel(1024)
    assert m.place(run).tolist() == [1022, 1023, 0, 1, 2]
    assert m.place(run[::-1]).tolist() == [2, 1, 0, 1023, 1022]  # placed ids stay put
    rng = np.random.RandomState(0)
    ids = rng.randint(0, 2 ** 62, 700).astype(np.int64)
    a, b = H.ShardModel(1024), H.ShardModel(1024)
    a.place(ids)
    b.place(rng.permutation(ids))
    assert np.array_equal(a.occupied(), b.occupied())


def test_slots_of_reads_back_the_slot():
    seed, name, slots = 7, "u", 1024
    for shard in (0, 2):
        rows = H.slot_rows(seed, name, shard, slots, 8)
        which = np.array([0, 1, 511, 1023, 5])
        assert H.slots_of(seed, name, shard, rows[which], slots).tolist() == which.tolist()
        assert H.slot_of(seed, name, shard, rows[1023], slots) == 1023
        assert H.slot_of(seed, name, shard, np.zeros(8, np.float32), slots) == -1
        want = np.array([[O.lib.oracle_uniform_init(H.shard_seed(seed, name, shard), int(s), c) for c in range(8)]
                         for s in which], dtype=np.float32)
        assert np.array_equal(rows[which], want)
    # another shard's draws are not this shard's
    assert H.slot_of(seed, name, 1, H.slot_rows(seed, name, 0, slots, 8)[3], slots) == -1
