"""PSGroup: the N HBM-resident shards of one parameter-server group, seen from one
client process, as torch-tensor level calls into libb200ps.so.

This is plumbing (pointers, streams, rendezvous); every byte of table data is
moved or updated by the CUDA kernels behind include/b200ps.h.  Reference
counterpart: the set of `elasticdl_ps` processes a job starts
(go/cmd/elasticdl_ps/main.go:48-74) plus the channel list PSClient is built
from (python/worker/ps_client.py:37-84).
"""
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib
from elasticdl_b200._lib import Seg, check

DEFAULT_CAPACITY = 1 << 20


def table_seed(seed, name):
    """Seed of a table's counter-based uniform initialiser (shared with the oracle in tests)."""
    return (int(seed) ^ int.from_bytes(name.encode()[:8].ljust(8, b"\0"), "little")) & (2 ** 64 - 1)


def exchange_blobs(local_blobs, n_shards, group=None):
    """All-gather {shard_id: bytes} over torch.distributed (host logic, backend agnostic).

    Returns the merged dict for every shard in the group.  Raises if a shard is
    exported by no rank or by more than one.
    """
    import torch.distributed as dist

    if not dist.is_available() or not dist.is_initialized():
        merged = dict(local_blobs)
    else:
        gathered = [None] * dist.get_world_size(group)
        dist.all_gather_object(gathered, dict(local_blobs), group=group)
        merged = {}
        for d in gathered:
            for k, v in d.items():
                if k in merged:
                    raise RuntimeError("shard %d exported by two ranks" % k)
                merged[k] = v
    missing = [s for s in range(n_shards) if s not in merged]
    if missing:
        raise RuntimeError("no rank owns shards %s" % missing)
    return merged


class PSGroup:
    """A parameter-server group of ``n_shards`` shards.

    opt_type / opt_args: exactly what the reference hands the Go PS
    (``-opt_type=Adam -opt_args="learning_rate=0.001;beta_1=0.9;..."``,
    python/common/model_utils.py:227-254, go/pkg/ps/optimizer.go:304-390).
    Accepted types and keys (every key required, no other key allowed):
      SGD       learning_rate, momentum, nesterov
      Adam      learning_rate, beta_1, beta_2, epsilon, amsgrad
      Adagrad   learning_rate, epsilon
      Ftrl      learning_rate, initial_accumulator_value, l1_regularization_strength,
                l2_regularization_strength, l2_shrinkage_regularization_strength, beta
      RMSprop   learning_rate, rho, momentum, epsilon, centered
      Adadelta  learning_rate, rho, epsilon
      Adamax    learning_rate, beta_1, beta_2, epsilon
      Nadam     learning_rate, beta_1, beta_2, epsilon
    The last four are the Python PS's Keras optimizers with get_config() key names, applied
    to the pushed rows only (DESIGN.md section 4).

    local_shards: shard ids whose memory this process owns (default: all, the
    single-process layout the reference's own tests use,
    python/tests/test_utils.py:301-327).  shard_devices: device index per local
    shard (default: the client device).
    """

    def __init__(self, n_shards, opt_type, opt_args, device=None, lr_staleness_modulation=False,
                 local_shards=None, shard_devices=None, reproduce_q1=False, track_rows=True,
                 process_group=None, seed=0, use_async=True, grads_to_wait=1, sync_version_tolerance=0):
        self._h = None
        self.lib = _lib.lib()
        if not torch.cuda.is_available():
            raise RuntimeError("elasticdl_b200 needs a CUDA device: the PS shards live in HBM "
                               "and there is no CPU fallback")
        if device is None:
            device = torch.cuda.current_device()
        self.device = torch.device("cuda", device if isinstance(device, int) else torch.device(device).index)
        self.n_shards = int(n_shards)
        self.opt_type, self.opt_args = opt_type, opt_args
        self.process_group = process_group
        self.seed = int(seed)
        self.lr_staleness_modulation = bool(lr_staleness_modulation)
        # PS-side mode flags (python/ps/parameter_server.py / go/cmd/elasticdl_ps/main.go:32-35).
        # The Go PS is async only (server.go:177); sync-SGD follows python/ps/servicer.py:168-238.
        self.use_async = bool(use_async)
        self.grads_to_wait = int(grads_to_wait)
        self.sync_version_tolerance = int(sync_version_tolerance)
        import threading

        self._sync_lock = threading.Lock()
        self._sync_buffer = {"n": 0, "dense": {}, "sparse": {}}
        flags = (1 if reproduce_q1 else 0) | (0 if track_rows else 2)
        h = ctypes.c_void_p()
        check(self.lib.b200ps_create(self.n_shards, self.device.index, opt_type.encode(), opt_args.encode(),
                                     1 if lr_staleness_modulation else 0, flags, ctypes.byref(h)))
        self._h = h
        self.local_shards = list(range(self.n_shards)) if local_shards is None else list(local_shards)
        devs = shard_devices or {}
        for s in self.local_shards:
            check(self.lib.b200ps_shard_create_local(self._h, s, int(devs.get(s, self.device.index))))
        self.tables = {}  # name -> (id, dim, is_dense, shape)
        self.table_initializers = {}  # name -> initializer string (EmbeddingTableInfo.initializer)
        self.dense_owner = {}  # dense parameter name -> shard
        self._pinned_state = torch.empty(3 * _lib.MAX_SHARDS, dtype=torch.int64).pin_memory()
        self._pinned_versions = torch.empty(_lib.MAX_SHARDS, dtype=torch.int32).pin_memory()
        self._ws = None
        if len(self.local_shards) == self.n_shards:
            check(self.lib.b200ps_commit(self._h))

    # ------------------------------------------------------------------ lifecycle
    def close(self):
        if self._h is not None:
            self.lib.b200ps_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def clone_view(self, device=None):
        """A second client view of the same shards for another worker thread / stream of this
        process (b200ps_clone_view).  Register every table on the owning group first."""
        view = object.__new__(PSGroup)
        view.__dict__.update({k: v for k, v in self.__dict__.items() if k not in ("_h", "_ws", "_ws_bounded")})
        view._h = None
        dev = self.device if device is None else torch.device("cuda", device)
        h = ctypes.c_void_p()
        check(self.lib.b200ps_clone_view(self._h, dev.index, ctypes.byref(h)))
        view._h = h
        view.device = dev
        view.local_shards = []  # owns no memory
        view.tables = dict(self.tables)
        view._owner = self  # keep the owner alive
        view._pinned_state = torch.empty(3 * _lib.MAX_SHARDS, dtype=torch.int64).pin_memory()
        view._pinned_versions = torch.empty(_lib.MAX_SHARDS, dtype=torch.int32).pin_memory()
        view._ws = None
        check(self.lib.b200ps_commit(view._h))
        return view

    def sync_peers(self):
        """Export local shards, all-gather the CUDA-IPC blobs, import the peers' shards."""
        blobs = {}
        for s in self.local_shards:
            size = ctypes.c_size_t()
            check(self.lib.b200ps_shard_export(self._h, s, None, 0, ctypes.byref(size)))
            buf = ctypes.create_string_buffer(size.value)
            check(self.lib.b200ps_shard_export(self._h, s, buf, size.value, ctypes.byref(size)))
            blobs[s] = buf.raw[: size.value]
        if len(self.local_shards) < self.n_shards:
            merged = exchange_blobs(blobs, self.n_shards, self.process_group)
            for s, blob in merged.items():
                if s in self.local_shards:
                    continue
                check(self.lib.b200ps_shard_import(self._h, s, blob, len(blob)))
        check(self.lib.b200ps_commit(self._h))

    # ------------------------------------------------------------------ definition
    def register_table(self, name, dim, initializer="uniform", capacity=None, expected_rows=None):
        """≙ push_embedding_table_infos for one table (idempotent).  capacity (= the layer's
        input_dim) gives a direct-indexed table; without it ids are unbounded and the table is
        hashed, sized for `expected_rows` distinct ids (default DEFAULT_CAPACITY)."""
        if name in self.tables:
            return self.tables[name][0]
        seed = table_seed(self.seed, name)
        self.table_initializers[name] = str(initializer)
        if not capacity:
            cap = int(expected_rows or DEFAULT_CAPACITY)
            tid = check(self.lib.b200ps_table_register_hashed(self._h, name.encode(), int(dim),
                                                              str(initializer).encode(), cap, seed))
            self.tables[name] = (tid, int(dim), False, (None, int(dim)))
            return tid
        cap = int(capacity)
        tid = check(self.lib.b200ps_table_register(self._h, name.encode(), int(dim), str(initializer).encode(),
                                                   cap, seed))
        self.tables[name] = (tid, int(dim), False, (cap, int(dim)))
        return tid

    def register_pair(self, name_a, name_b, capacity, initializer="zero"):
        """A dim-8 table `name_a` and a dim-1 table `name_b` addressed with the same ids, stored as
        one record per id (b200ps_table_register_pair); both stay addressable by name."""
        if name_a in self.tables and name_b in self.tables:
            return self.tables[name_a][0], self.tables[name_b][0]
        seed = table_seed(self.seed, name_a)
        ta = check(self.lib.b200ps_table_register_pair(self._h, name_a.encode(), name_b.encode(),
                                                       str(initializer).encode(), int(capacity), seed))
        tb = check(self.lib.b200ps_lookup(self._h, name_b.encode()))
        self.tables[name_a] = (ta, 8, False, (int(capacity), 8))
        self.tables[name_b] = (tb, 1, False, (int(capacity), 1))
        self.table_initializers[name_a] = self.table_initializers[name_b] = str(initializer)
        return ta, tb

    def pair_call(self, fn, seg_items, rows_b):
        """fn = b200ps_pull_rows_pair / b200ps_push_rows_pair over [(tid_a, n, ids, n_dev, rows_a)] + B rows."""
        half = _lib.MAX_SEGS // 2
        for i in range(0, len(seg_items), half):
            arr, n = self.make_segs(seg_items[i:i + half])
            ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in rows_b[i:i + half]])
            check(fn(self._h, arr, ptrs, n, self._stream()))

    def xchg_create(self, G, B, deep_table_ids, wide_table_ids):
        """Collective: allocate this rank's owner-computes exchange buffer (csrc/ps_exchange.cuh) for G
        (dim-8, dim-1) table pairs and batches of B ids per group, then map the peers' buffers."""
        d = (ctypes.c_int32 * G)(*[int(t) for t in deep_table_ids])
        w = (ctypes.c_int32 * G)(*[int(t) for t in wide_table_ids])
        check(self.lib.b200ps_xchg_create(self._h, int(G), int(B), d, w))
        self.commit()

    def register_dense(self, name, shape, shard):
        if name in self.tables:
            return self.tables[name][0]
        shape = tuple(int(x) for x in shape)
        numel = int(np.prod(shape)) if len(shape) else 1
        rows = shape[0] if len(shape) >= 2 else numel
        dim = numel // rows if rows else 1
        tid = check(self.lib.b200ps_dense_register(self._h, name.encode(), int(shard), rows, dim))
        self.tables[name] = (tid, dim, True, shape)
        self.dense_owner[name] = int(shard)
        return tid

    def commit(self):
        if len(self.local_shards) == self.n_shards or getattr(self, "_owner", None) is not None:
            check(self.lib.b200ps_commit(self._h))
        else:
            self.sync_peers()

    def lookup(self, name):
        if name not in self.tables:
            raise _lib.PSNotFound(_lib.ENOTFOUND, "%s not in Parameter" % name)
        return self.tables[name]

    # ------------------------------------------------------------------ helpers
    def make_segs(self, items):
        """items: iterable of (table_id, n, ids_tensor|None, n_dev_tensor|None, rows_tensor)."""
        items = list(items)
        arr = (Seg * max(len(items), 1))()
        for i, (tid, n, ids, n_dev, rows) in enumerate(items):
            arr[i].table = tid
            arr[i].n = n
            arr[i].ids_dev = ids.data_ptr() if ids is not None else None
            arr[i].n_dev = n_dev.data_ptr() if n_dev is not None else None
            arr[i].rows_dev = rows.data_ptr() if rows is not None else None
        return arr, len(items)

    def _run_segs(self, fn, items):
        items = list(items)
        for i in range(0, len(items), _lib.MAX_SEGS):
            arr, n = self.make_segs(items[i:i + _lib.MAX_SEGS])
            check(fn(self._h, arr, n, self._stream()))

    def _ids(self, ids):
        t = torch.as_tensor(ids)
        if t.dtype != torch.int64:
            t = t.to(torch.int64)
        return t.to(self.device, non_blocking=True).contiguous().view(-1)

    def _f32(self, v):
        t = torch.as_tensor(v)
        if t.dtype != torch.float32:
            t = t.to(torch.float32)
        return t.to(self.device, non_blocking=True).contiguous()

    # ------------------------------------------------------------------ data path
    def pull_rows(self, requests):
        """requests: [(name, ids)] -> [float32 cuda tensor [len(ids), dim]] in ONE launch set."""
        items, outs = [], []
        for name, ids in requests:
            tid, dim, _, _ = self.lookup(name)
            ids = self._ids(ids)
            out = torch.empty((ids.numel(), dim), dtype=torch.float32, device=self.device)
            outs.append(out)
            items.append((tid, ids.numel(), ids, None, out))
        self._run_segs(self.lib.b200ps_pull_rows, items)
        return outs

    def set_rows(self, requests):
        """requests: [(name, ids, values)] ≙ SetEmbeddingVectors."""
        items = []
        for name, ids, values in requests:
            tid, dim, _, _ = self.lookup(name)
            ids = self._ids(ids)
            vals = self._f32(values).view(ids.numel(), dim)
            items.append((tid, ids.numel(), ids, None, vals))
        self._run_segs(self.lib.b200ps_set_rows, items)

    def pull_dense(self, names, into=None):
        """Dense parameters by name -> {name: float32 cuda tensor}.  `into` ({name: tensor}) makes the kernel write
        straight into the caller's tensors (contiguous float32 on this device, right size) instead of new ones."""
        outs, items = {}, []
        for name in names:
            tid, _, is_dense, shape = self.lookup(name)
            if into is not None:
                out = into[name]
                if not (out.is_cuda and out.device == self.device and out.dtype == torch.float32
                        and out.is_contiguous() and out.numel() == int(np.prod(shape))):
                    raise ValueError("pull_dense(into=): %s must be a contiguous float32 tensor of %s on %s"
                                     % (name, tuple(shape), self.device))
            else:
                out = torch.empty(shape, dtype=torch.float32, device=self.device)
            outs[name] = out
            items.append((tid, 0, None, None, out))
        self._run_segs(self.lib.b200ps_pull_dense, items)
        return outs

    def set_dense(self, named_values):
        items = []
        for name, v in named_values:
            tid, _, _, shape = self.lookup(name)
            t = self._f32(v)
            if tuple(t.shape) != tuple(shape):
                raise ValueError("shape mismatch for %s: %s vs %s" % (name, tuple(t.shape), shape))
            items.append((tid, 0, None, None, t))
        self._run_segs(self.lib.b200ps_set_dense, items)

    def slot_rows(self, name, ids, slot, values=None):
        """Read (values None) or write the optimizer slot rows of `ids` (slot 0 = parameter)."""
        tid, dim, _, _ = self.lookup(name)
        ids = self._ids(ids)
        buf = (torch.empty((ids.numel(), dim), dtype=torch.float32, device=self.device)
               if values is None else self._f32(values).view(ids.numel(), dim))
        arr, n = self.make_segs([(tid, ids.numel(), ids, None, buf)])
        check(self.lib.b200ps_slot_rows(self._h, int(slot), 0 if values is None else 1, arr, n, self._stream()))
        return buf

    def slot_dense(self, name, slot, values=None):
        tid, _, _, shape = self.lookup(name)
        buf = (torch.empty(shape, dtype=torch.float32, device=self.device)
               if values is None else self._f32(values).view(shape))
        arr, n = self.make_segs([(tid, 0, None, None, buf)])
        check(self.lib.b200ps_slot_dense(self._h, int(slot), 0 if values is None else 1, arr, n, self._stream()))
        return buf

    def push_begin(self, learning_rate, model_versions):
        mv = (ctypes.c_int32 * _lib.MAX_SHARDS)(*[int(v) for v in model_versions])
        check(self.lib.b200ps_push_begin(self._h, float(learning_rate), mv, self._stream()))

    def bump_step(self):
        check(self.lib.b200ps_bump_step(self._h, self._stream()))

    def push_rows(self, items):
        """items: [(table_id, n, ids, n_dev, grads)] unique ids per segment."""
        self._run_segs(self.lib.b200ps_push_rows, items)

    def push_dense(self, items):
        self._run_segs(self.lib.b200ps_push_dense, items)

    def push_dense_reduce(self, name, grads, scale=1.0, divide=False):
        """Sum the replica gradients `grads` left to right, then divide the sum by `scale` (divide=True, the
        sync-SGD average) or multiply it by `scale`, and apply the optimizer update -- one kernel."""
        tid, _, is_dense, _ = self.lookup(name)
        ptrs = (ctypes.c_void_p * len(grads))(*[g.data_ptr() for g in grads])
        check(self.lib.b200ps_push_dense_reduce(self._h, tid, ptrs, len(grads), float(scale), 1 if divide else 0,
                                                self._stream()))

    def push_end(self, sync=True):
        """Version++ on every shard; returns the new versions (list) when sync."""
        check(self.lib.b200ps_push_end(self._h, ctypes.c_void_p(self._pinned_versions.data_ptr()), self._stream()))
        if sync:
            torch.cuda.current_stream(self.device).synchronize()
            return self._pinned_versions[: self.n_shards].tolist()
        return None

    # ------------------------------------------------------------------ dedup
    def unique(self, ids, T=1, bounds=None):
        """tf.unique over T equal-length segments.  ids: int64 cuda [T*k].
        Returns (uniq [T*k] padded, inv int32 [T*k], n_unique int32 [T]) -- all on device.
        bounds (optional, one int per segment = the table capacity / the layer's input_dim, 0 = unknown): segments
        with a known id range are deduplicated through a direct-address position array (b200ps_unique_bounded) --
        several times faster than hashing; an id outside [0, bound) is counted as id 0 and makes check() raise."""
        ids = self._ids(ids)
        k = ids.numel() // T
        if bounds is not None and (T > _lib.MAX_SEGS or len(bounds) != T or not any(int(b) > 0 for b in bounds)):
            bounds = None
        key = None if bounds is None else (T, k, tuple(int(b) for b in bounds))
        if key is None:
            need = self.lib.b200ps_unique_workspace(T, k)
            if self._ws is None or self._ws.numel() < need:
                if self._ws is not None:
                    self._ws.record_stream(torch.cuda.current_stream(self.device))
                self._ws = torch.zeros(need, dtype=torch.uint8, device=self.device)
            ws = self._ws
        else:  # one workspace per (T, k, bounds): the direct-address arrays are laid out by the bounds
            cache = self.__dict__.setdefault("_ws_bounded", {})
            if key not in cache:  # never evicted: a captured CUDA graph may hold the address (a job has a handful of keys)
                barr = (ctypes.c_int64 * T)(*key[2])
                cache[key] = (torch.zeros(self.lib.b200ps_unique_bounded_workspace(T, k, barr), dtype=torch.uint8,
                                          device=self.device), barr)
            ws, barr = cache[key]
        uniq = torch.empty(T * k, dtype=torch.int64, device=self.device)
        inv = torch.empty(T * k, dtype=torch.int32, device=self.device)
        n_unique = torch.empty(T, dtype=torch.int32, device=self.device)
        if key is None:
            check(self.lib.b200ps_unique(self._h, ids.data_ptr(), T, k, uniq.data_ptr(), inv.data_ptr(),
                                         n_unique.data_ptr(), ws.data_ptr(), ws.numel(), self._stream()))
        else:
            check(self.lib.b200ps_unique_bounded(self._h, ids.data_ptr(), T, k, barr, uniq.data_ptr(), inv.data_ptr(),
                                                 n_unique.data_ptr(), ws.data_ptr(), ws.numel(), self._stream()))
        return uniq, inv, n_unique

    def segment_sum(self, values, inv, T, k, dim, out=None):
        values = self._f32(values)
        if out is None:
            out = torch.empty(T * k * dim, dtype=torch.float32, device=self.device)
        check(self.lib.b200ps_segment_sum(self._h, values.data_ptr(), inv.data_ptr(), T, k, dim, out.data_ptr(),
                                          self._stream()))
        return out

    def gather_rows(self, bet, inv, T, k, dim, out=None):
        if out is None:
            out = torch.empty(T * k * dim, dtype=torch.float32, device=self.device)
        check(self.lib.b200ps_gather_rows(self._h, bet.data_ptr(), inv.data_ptr(), T, k, dim, out.data_ptr(),
                                          self._stream()))
        return out

    # ------------------------------------------------------------------ state
    def snapshot(self):
        """[(version, step, initialized)] per shard, one stream sync."""
        check(self.lib.b200ps_snapshot_state(self._h, ctypes.c_void_p(self._pinned_state.data_ptr()), self._stream()))
        torch.cuda.current_stream(self.device).synchronize()
        s = self._pinned_state[: 3 * self.n_shards].view(self.n_shards, 3).tolist()
        return [(int(v), int(st), bool(i)) for v, st, i in s]

    def set_shard_state(self, shard, version=-1, step=-1, initialized=-1):
        check(self.lib.b200ps_set_shard_state(self._h, shard, version, step, initialized))

    def try_init(self, shard):
        won = ctypes.c_int()
        check(self.lib.b200ps_try_init(self._h, shard, ctypes.byref(won)))
        return bool(won.value)

    def finish_init(self, shard, version):
        check(self.lib.b200ps_finish_init(self._h, shard, int(version), self._stream()))

    def table_size(self, name, shard=None):
        tid = self.lookup(name)[0]
        total = 0
        for s in ([shard] if shard is not None else range(self.n_shards)):
            n = ctypes.c_int64()
            check(self.lib.b200ps_table_size(self._h, tid, s, ctypes.byref(n)))
            total += n.value
        return total

    def table_ids(self, name, shard):
        tid = self.lookup(name)[0]
        n = ctypes.c_int64()
        check(self.lib.b200ps_table_size(self._h, tid, shard, ctypes.byref(n)))
        ids = torch.empty(max(n.value, 1), dtype=torch.int64, device=self.device)
        check(self.lib.b200ps_table_ids(self._h, tid, shard, ids.data_ptr(), ids.numel(), ctypes.byref(n)))
        return ids[: n.value]

    def check(self):
        """Raise if a kernel flagged an error (e.g. id out of range)."""
        check(self.lib.b200ps_check(self._h))

    @property
    def launch_count(self):
        return int(self.lib.b200ps_launch_count(self._h))
