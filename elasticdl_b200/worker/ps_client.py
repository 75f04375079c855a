"""PSClient: the worker-side boundary of the parameter-server path.

Same class name, attributes, method names, argument order and return
conventions as elasticdl/python/worker/ps_client.py:87-301, so the trainer and
the Embedding layer call it unchanged.  What is different is underneath: the
"channels" are the HBM shards of a PSGroup, the per-shard request fan-out
(ps_client.py:105-120, 243-277) is the `id % N` addressing inside one CUDA
launch, and nothing is serialised.

Array types: numpy arrays / lists in -> numpy arrays out (the reference's
contract); torch CUDA tensors in -> torch CUDA tensors out (no host hop).
"""
import numpy as np
import torch

from elasticdl_b200 import _lib
from elasticdl_b200.common.hash_utils import string_to_id
from elasticdl_b200.common.tensor_utils import DeviceIds, Tensor, UniqueTensor  # noqa: F401  (Tensor re-exported as the reference module does)
from elasticdl_b200.ps.group import PSGroup


def build_ps_client(ps_group, logger=None):
    """≙ build_ps_client(ps_addrs, logger) (ps_client.py:37-84): there are no
    addresses to dial -- the group's shards are already attached -- so this only
    wraps the group.  Returns None for a falsy group like the reference does for
    an empty address list."""
    if not ps_group:
        return None
    return PSClient(ps_group)


def _is_torch(x):
    return isinstance(x, torch.Tensor)


class PSClient(object):
    def __init__(self, ps_group):
        if not isinstance(ps_group, PSGroup):
            raise TypeError("PSClient needs a PSGroup (the HBM shards); got %r" % type(ps_group))
        self.group = ps_group
        self.ps_num = ps_group.n_shards
        self.parameter_to_ps = {}
        self.ps_to_parameter = {}
        self.dense_output = "numpy"  # or "torch": keep pulled dense parameters on the device

    # ------------------------------------------------------------------ embeddings
    def pull_embedding_vectors(self, layer_name, embedding_ids):
        """Pulls and returns embedding vectors ordered by the embedding ids
        (ps_client.py:96-130)."""
        as_torch = _is_torch(embedding_ids)
        n = embedding_ids.numel() if as_torch else len(embedding_ids)
        if n == 0:
            # the reference np.concatenate()s an empty list here
            raise ValueError("need at least one array to concatenate")
        (out,) = self.group.pull_rows([(layer_name, embedding_ids)])
        if as_torch:
            return out
        self.group.check()  # device sync + out-of-range ids -> exception
        return out.cpu().numpy()

    def pull_embedding_vectors_batch(self, requests):
        """[(layer_name, ids)] -> [rows] with one launch per vector class (device
        tensors in, device tensors out).  No reference counterpart: the reference
        issues one RPC per (layer, shard)."""
        return self.group.pull_rows(requests)

    def pull_embedding_vectors_into(self, requests):
        """[(layer_name, ids int64 device [k], n_dev int32 device [1] | None, out float32 device [k, dim])]:
        the first n_dev[0] (or k) ids of every request are looked up into `out`, all requests in one
        launch and without a host read of the counts (rows past the count are left untouched)."""
        g = self.group
        items = []
        for name, ids, n_dev, out in requests:
            tid, dim, _, _ = g.lookup(name)
            items.append((tid, ids.numel(), ids, n_dev, out))
        g._run_segs(g.lib.b200ps_pull_rows, items)

    def push_embedding_table_infos(self, infos):
        """ps_client.py:289-301 -> every shard creates the tables + slot tables."""
        for info in infos:
            cap = getattr(info, "capacity", None)
            self.group.register_table(info.name, info.dim, info.initializer, cap)
        self.group.commit()

    # ------------------------------------------------------------------ dense
    def partition_dense_parameters(self, param_names, shapes=None):
        """ps_id = string_to_id(param_name) (ps_client.py:132-144).  `shapes`
        (optional, name -> shape) lets every process of a multi-process group
        register the parameters collectively up front."""
        registered = False
        for name in param_names:
            if name not in self.parameter_to_ps:
                self.parameter_to_ps[name] = string_to_id(name, self.ps_num)
                ps_id = self.parameter_to_ps[name]
                if ps_id not in self.ps_to_parameter:
                    self.ps_to_parameter[ps_id] = [name]
                else:
                    self.ps_to_parameter[ps_id].append(name)
            if shapes is not None and name not in self.group.tables:
                self.group.register_dense(name, shapes[name], self.parameter_to_ps[name])
                registered = True
        if registered:
            self.group.commit()

    def push_dense_parameters(self, parameters, ps_id, version):
        """Push dense parameters to one shard (ps_client.py:146-159 -> PushModel,
        server.go:209-221: first writer wins, later pushes are ignored)."""
        mine = [p for p in parameters if self.parameter_to_ps[p.name] == ps_id]
        registered = False
        for p in mine:
            if p.name not in self.group.tables:
                if len(self.group.local_shards) != self.group.n_shards:
                    raise RuntimeError(
                        "dense parameter %s was not registered collectively; call "
                        "partition_dense_parameters(names, shapes=...) on every rank first" % p.name)
                self.group.register_dense(p.name, tuple(np.shape(p.values)), ps_id)
                registered = True
        if registered:
            self.group.commit()
        if self.group.try_init(ps_id):
            self.group.set_dense([(p.name, p.values) for p in mine])
            self.group.finish_init(ps_id, version)

    def pull_dense_parameters(self, ps_ids, model_versions):
        """Pull dense parameters (ps_client.py:161-188).  Mutates model_versions in
        place.  Go semantics: parameters are sent when Version >= requested
        (server.go:150, quirk Q8)."""
        wanted = [ps_id for ps_id in ps_ids if ps_id in self.ps_to_parameter]
        dense_params = {}
        uninit_ps = []
        if not wanted:
            return dense_params, uninit_ps
        state = self.group.snapshot()
        names = []
        for ps_id in wanted:
            version, _, initialized = state[ps_id]
            if not initialized:
                uninit_ps.append(ps_id)
                continue
            if version >= model_versions[ps_id]:
                names.extend(n for n in self.ps_to_parameter[ps_id] if n in self.group.tables)
            model_versions[ps_id] = version
        if names:
            pulled = self.group.pull_dense(names)
            if self.dense_output == "torch":
                dense_params.update(pulled)
            else:
                for k, v in pulled.items():
                    dense_params[k] = v.cpu().numpy()
        return dense_params, uninit_ps

    # ------------------------------------------------------------------ gradients
    def _dedup(self, name, values_list, indices_list, dim):
        """merge_indexed_slices + deduplicate_indexed_slices (tensor_utils.py:31-60)
        on the device: concatenate, unique ids in first-occurrence order, summed rows."""
        g = self.group
        vals = [g._f32(v).reshape(-1, dim) for v in values_list]
        ids = [g._ids(i) for i in indices_list]
        v = vals[0] if len(vals) == 1 else torch.cat(vals, 0)
        i = ids[0] if len(ids) == 1 else torch.cat(ids, 0)
        k = i.numel()
        if v.shape[0] != k:
            raise ValueError("gradient rows (%d) and indices (%d) differ for %s" % (v.shape[0], k, name))
        uniq, inv, n_unique = g.unique(i, 1)
        gsum = g.segment_sum(v, inv, 1, k, dim)
        return uniq, n_unique, gsum, k

    def push_gradients(self, grads, edl_grads, learning_rate, model_versions, sync=True):
        """Push gradients to the PS (ps_client.py:190-287).  Two kinds:
         - gradients of normal layers (dense, or IndexedSlices of a dense parameter)
         - sparse gradients of ElasticDL embedding layers
        Every shard applies exactly one ApplyGradients and bumps its version
        (quirk Q7).  Returns (accepted, max_version).
        sync=False (device tensors only, async PS): nothing is read back -- the new versions land in
        `group._pinned_versions` when the stream gets there and the caller checks `group.check()` itself;
        returns (True, None).  This form is legal inside a CUDA-graph capture."""
        g = self.group
        if not getattr(g, "use_async", True):
            if not sync:
                raise ValueError("push_gradients(sync=False) needs an async PS group")
            return self._push_gradients_sync(grads, edl_grads, learning_rate, model_versions)
        # 1. group by name; same-name merge (ps_client.py:203-217)
        dense, indexed = {}, {}
        for grad in grads:
            if grad.name not in self.parameter_to_ps:
                raise KeyError(grad.name)  # the reference indexes parameter_to_ps[grad.name]
            if grad.indices is not None:
                indexed.setdefault(grad.name, ([], []))
                indexed[grad.name][0].append(grad.values)
                indexed[grad.name][1].append(grad.indices)
            elif grad.name in dense:
                dense[grad.name] = g._f32(dense[grad.name]) + g._f32(grad.values)
            else:
                dense[grad.name] = grad.values
        edl, already_unique = {}, {}
        for grad in edl_grads:  # ps_client.py:243-251
            edl.setdefault(grad.name, ([], []))
            edl[grad.name][0].append(grad.values)
            edl[grad.name][1].append(grad.indices)
            already_unique[grad.name] = isinstance(grad, UniqueTensor) and grad.name not in already_unique

        # validate before launching: the Go PS fails the whole ApplyGradients
        # ("grad %s not in Parameter", optimizer.go:49,59; width check kernel.go:36-38)
        # after step++ (quirk Q2)
        try:
            dense_items, row_items = [], []
            for name, v in dense.items():
                tid, _, is_dense, shape = g.lookup(name)
                t = g._f32(v)
                if t.numel() != int(np.prod(shape)):
                    raise ValueError("grad size mismatch for %s" % name)
                dense_items.append((tid, 0, None, None, t))
            for group_, is_edl in ((indexed, False), (edl, True)):
                for name, (vl, il) in group_.items():
                    tid, dim, is_dense, shape = g.lookup(name)
                    width = int(np.prod(np.shape(vl[0])[1:])) if np.ndim(vl[0]) > 1 else 1
                    if width != dim:
                        raise ValueError("grad width is not equal to embedding dim")
                    if is_edl and already_unique.get(name) and len(vl) == 1:
                        n_dev = None
                        if isinstance(il[0], DeviceIds):  # count stays on the device
                            ids_t, n_dev = il[0].ids, il[0].n_dev
                        else:
                            ids_t = g._ids(il[0])
                        row_items.append((tid, ids_t.numel(), ids_t, n_dev, g._f32(vl[0]).reshape(-1, dim)))
                        continue
                    if any(isinstance(i, DeviceIds) for i in il):
                        raise ValueError("DeviceIds gradients of %s cannot be merged with others" % name)
                    uniq, n_unique, gsum, k = self._dedup(name, vl, il, dim)
                    row_items.append((tid, k, uniq, n_unique, gsum))
        except (_lib.PSNotFound, ValueError):
            g.bump_step()
            raise

        # 2. one ApplyGradients per shard: begin (step++, lr), kernels, end (version++)
        g.push_begin(learning_rate, model_versions)
        if dense_items:
            g.push_dense(dense_items)
        if row_items:
            g.push_rows(row_items)
        versions = g.push_end(sync=sync)
        if not sync:
            return True, None
        g.check()
        return True, max(versions)

    # ------------------------------------------------------------------ sync-SGD
    def _push_gradients_sync(self, grads, edl_grads, learning_rate, model_versions):
        """Sync-SGD as the Python PS implements it (python/ps/servicer.py:168-238): pushes older
        than version - sync_version_tolerance are rejected; accepted pushes are buffered; when
        grads_to_wait of them have arrived, dense gradients are AVERAGED and sparse gradients
        SUMMED (concatenated, then deduplicated) and applied once -- the dense reduce is fused
        with the optimizer update in one kernel (b200ps_push_dense_reduce) -- and the version
        advances by one.  The buffer lives on the owning PSGroup, shared by all client views."""
        g = self.group
        owner = getattr(g, "_owner", None) or g
        state = g.snapshot()
        version = max(s[0] for s in state)
        mv = max(model_versions) if len(model_versions) else 0
        if mv < version - owner.sync_version_tolerance:  # servicer.py:168-175
            return False, version
        with owner._sync_lock:
            buf = owner._sync_buffer
            for grad in grads:
                tid, dim, is_dense, shape = g.lookup(grad.name)
                if grad.indices is not None:
                    vals, ids = buf["sparse"].setdefault(grad.name, ([], []))
                    vals.append(g._f32(grad.values).reshape(-1, dim).clone())
                    ids.append(g._ids(grad.indices).clone())
                else:
                    t = g._f32(grad.values).reshape(-1).clone()
                    if t.numel() != int(np.prod(shape)):
                        raise ValueError("grad size mismatch for %s" % grad.name)
                    buf["dense"].setdefault(grad.name, []).append(t)
            for grad in edl_grads:
                tid, dim, is_dense, shape = g.lookup(grad.name)
                vals, ids = buf["sparse"].setdefault(grad.name, ([], []))
                v = g._f32(grad.values).reshape(-1, dim)
                if v.shape[0] != g._ids(grad.indices).numel():
                    raise ValueError("grad width is not equal to embedding dim")
                vals.append(v.clone())
                ids.append(g._ids(grad.indices).clone())
            buf["n"] += 1
            if buf["n"] < owner.grads_to_wait:
                return True, version
            # apply: servicer.py:199-224
            w = owner.grads_to_wait
            g.push_begin(learning_rate, [version] * self.ps_num)
            for name, parts in buf["dense"].items():
                g.push_dense_reduce(name, parts, scale=w, divide=True)  # grad / grads_to_wait in fp32
            row_items = []
            for name, (vals, ids) in buf["sparse"].items():
                tid, dim, _, _ = g.lookup(name)
                uniq, n_unique, gsum, k = self._dedup(name, vals, ids, dim)
                row_items.append((tid, k, uniq, n_unique, gsum))
            if row_items:
                g.push_rows(row_items)
            versions = g.push_end(sync=True)
            g.check()
            buf["n"] = 0
            buf["dense"].clear()
            buf["sparse"].clear()
            return True, max(versions)
