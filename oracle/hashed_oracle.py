"""Host restatement of where a hashed embedding table puts an id -- TEST INFRASTRUCTURE.

Only tests import this module; nothing under elasticdl_b200/ does.

A hashed table (b200ps_table_register_hashed, csrc/b200ps.cu) has, on every shard, a power-of-two array of
slots: the smallest power of two >= max(1024, 2 * ceil(expected_rows / N)).  An id goes to shard `id & (N-1)`
when N is a power of two and `id % N` otherwise, starts at its home slot `mix64(id) & (slots - 1)` and takes the
first slot of the linear probe chain that is free or already holds it (probe_slot, csrc/ps_kernels.cuh).  Slots
are never freed, so the set of slots a group of ids occupies does not depend on the order they arrived in; only
which id of a colliding group holds which of those slots does.

A "uniform" hashed table draws a row's initial values by SLOT, not by id (alloc_table_on_shard: the generator
of oracle_uniform_init at row index = slot, seed table_seed ^ 0x9E3779B97F4A7C15 * (shard + 1)), so a freshly
created row tells which slot its id landed in: `slot_of` / `slots_of` read it back.
"""
import functools

import numpy as np

F = np.float32
U = np.uint64
GOLDEN = 0x9E3779B97F4A7C15
MIN_SLOTS = 1024
MASK64 = (1 << 64) - 1


def _u64(x):
    """int64 / uint64 / Python ints (any sign) -> uint64 array, two's complement."""
    a = np.asarray(x)
    if a.dtype == np.uint64:
        return a
    if a.dtype == np.int64:
        return a.view(np.uint64)
    return np.array([int(v) & MASK64 for v in np.ravel(a)], dtype=np.uint64).reshape(a.shape)


def mix64(x):
    """The 64-bit finaliser of ps_kernels.cuh / ps_oracle.c, elementwise over uint64 (wrapping multiply)."""
    x = _u64(x).copy()
    with np.errstate(over="ignore"):
        x ^= x >> U(33)
        x *= U(0xFF51AFD7ED558CCD)
        x ^= x >> U(33)
        x *= U(0xC4CEB9FE1A85EC53)
        x ^= x >> U(33)
    return x


def uniform_init(seed, ids, cols):
    """oracle_uniform_init(seed, id, col) broadcast over ids and cols, float32: u * 0.1f - 0.05f, u in [0, 1)."""
    ids, cols = np.broadcast_arrays(_u64(ids), _u64(cols))
    with np.errstate(over="ignore"):
        h = mix64(_u64(seed) ^ mix64(ids * U(GOLDEN) + cols))
    u = (h >> U(40)).astype(F) * F(1.0 / 16777216.0)
    return u * F(0.1) + F(-0.05)


def table_seed(group_seed, name):
    """PSGroup's per-table seed: the group seed xor the table name's first 8 bytes, little endian."""
    return (int(group_seed) ^ int.from_bytes(name.encode()[:8].ljust(8, b"\0"), "little")) & MASK64


def shard_seed(group_seed, name, shard):
    """Seed of the slot-keyed initial values of `name` on `shard`."""
    return (table_seed(group_seed, name) ^ (GOLDEN * (shard + 1))) & MASK64


def hashed_slots(expected_rows, n_shards):
    """Slots per shard of a hashed table registered for `expected_rows` distinct ids over `n_shards` shards."""
    per_shard = -(-int(expected_rows) // int(n_shards))
    slots = MIN_SLOTS
    while slots < 2 * per_shard:
        slots <<= 1
    return slots


def shard_of(ids, n_shards):
    """Owning shard of non-negative ids."""
    u = _u64(ids)
    n = U(n_shards)
    return ((u & (n - U(1))) if n_shards & (n_shards - 1) == 0 else (u % n)).astype(np.int64)


def home_slot(ids, slots):
    """First slot of each id's probe chain on its shard."""
    return (mix64(ids) & U(slots - 1)).astype(np.int64)


def craft(k, slots, n_shards, shard, home, start=1, low32=None):
    """The first k ids, scanning upward from `start`, that go to `shard` and whose home slot is `home`.  With
    `low32`, the candidates are (hi << 32) | low32 for hi = start, start + 1, ...: ids equal in their low 32 bits.
    Returns int64 ids, all positive and below 2^63."""
    if low32 is not None and n_shards & (n_shards - 1) == 0 and (low32 & (n_shards - 1)) != shard:
        raise ValueError("low32 routes every candidate to shard %d" % (low32 & (n_shards - 1)))
    out, pos = [], int(start)
    limit = 1 << 31 if low32 is not None else 1 << 63
    chunk = min(1 << 22, max(1 << 12, 2 * k * slots * n_shards))  # about twice the expected scan
    while len(out) < k:
        if pos >= limit:
            raise ValueError("no more candidates")
        c = np.arange(pos, min(pos + chunk, limit), dtype=np.uint64)
        ids = (c << U(32)) | U(low32) if low32 is not None else c
        m = (home_slot(ids, slots) == home) & (shard_of(ids, n_shards) == shard)
        out.extend(ids[m][: k - len(out)].view(np.int64).tolist())
        pos += len(c)
    return np.array(out, dtype=np.int64)


class ShardModel:
    """One shard's key array under linear probing, ids placed one at a time."""

    def __init__(self, slots):
        self.slots = int(slots)
        self.key_at = {}  # slot -> id
        self.slot = {}  # id -> slot

    def place(self, ids):
        """Place ids in this order (an id already present stays where it is); returns their slots."""
        out = []
        for i in np.asarray(ids, dtype=np.int64).reshape(-1).tolist():
            if i not in self.slot:
                if len(self.key_at) == self.slots:
                    raise ValueError("full")
                h = int(home_slot(np.array([i], dtype=np.int64), self.slots)[0])
                while h in self.key_at:
                    h = (h + 1) & (self.slots - 1)
                self.key_at[h] = i
                self.slot[i] = h
            out.append(self.slot[i])
        return np.array(out, dtype=np.int64)

    def occupied(self):
        return np.array(sorted(self.key_at), dtype=np.int64)


class GroupModel:
    """ShardModel per shard of an N-shard group: place() routes ids by shard_of."""

    def __init__(self, slots, n_shards):
        self.n_shards = int(n_shards)
        self.shards = [ShardModel(slots) for _ in range(self.n_shards)]

    def place(self, ids):
        ids = np.asarray(ids, dtype=np.int64).reshape(-1)
        sh = shard_of(ids, self.n_shards)
        return np.array([self.shards[s].place([i])[0] for i, s in zip(ids.tolist(), sh.tolist())], dtype=np.int64)

    def ids(self):
        return np.sort(np.array([i for m in self.shards for i in m.slot], dtype=np.int64))


@functools.lru_cache(maxsize=64)
def _slot_table(seed, slots, dim):
    rows = uniform_init(seed, np.arange(slots, dtype=np.int64)[:, None], np.arange(dim, dtype=np.int64)[None, :])
    index = {}
    for s, key in enumerate(map(bytes, rows)):
        index.setdefault(key, []).append(s)
    return rows, index


def slot_rows(group_seed, name, shard, slots, dim, which=None):
    """Initial rows of the given slots (all slots when `which` is None) of a "uniform" hashed table's shard."""
    rows, _ = _slot_table(shard_seed(group_seed, name, shard), int(slots), int(dim))
    return rows if which is None else rows[np.asarray(which, dtype=np.int64)]


def slots_of(group_seed, name, shard, rows, slots):
    """The slot whose initial values each freshly created row of a "uniform" hashed table's shard carries; -1 for a
    row that matches no slot or more than one."""
    rows = np.ascontiguousarray(rows, dtype=F)
    rows = rows.reshape(rows.shape[0], -1)
    _, index = _slot_table(shard_seed(group_seed, name, shard), int(slots), rows.shape[1])
    out = np.full(rows.shape[0], -1, dtype=np.int64)
    for r, key in enumerate(map(bytes, rows)):
        hit = index.get(key, ())
        if len(hit) == 1:
            out[r] = hit[0]
    return out


def slot_of(group_seed, name, shard, row, slots):
    """slots_of for one row."""
    return int(slots_of(group_seed, name, shard, np.asarray(row, dtype=F).reshape(1, -1), slots)[0])
