"""ParameterServerTrainer over torch: the caller of the PS hot path.

Mirrors elasticdl/python/worker/ps_trainer.py:36-440 method for method
(`train_minibatch` -> (accepted, version, loss), `_get_model`, `_report_gradient`,
`init_variables_if_need`, local updates between pulls) with the TensorFlow pieces
restated over torch autograd:

  * `model` is a torch.nn.Module with attributes `optimizer` (a torch optimizer on
    its non-embedding parameters; its lr travels to the PS on every push,
    ps_trainer.py:275) and `loss` (callable(labels, outputs));
  * non-embedding variables are `model.named_parameters()`; ElasticDL Embedding
    layers are found by type (ps_trainer.py:66-74) and wired to
    `ps_client.pull_embedding_vectors`;
  * DenseTableEmbedding / DenseTableEmbeddingBag (layers/dense_table.py, what
    common/model_handler.py makes of torch tables of at most 2 MB) are found by type too:
    their weight is a dense PS parameter that is never pulled or pushed whole -- the
    batch's rows are pulled by id, and the gradient is pushed as those unique ids with
    their summed rows (an IndexedSlices), so rows outside the batch and their slots
    stay untouched.
"""
import numpy as np
import torch

from elasticdl_b200 import ops
from elasticdl_b200.common.tensor_utils import DT_FLOAT, DeviceIds, EmbeddingTableInfo, Tensor, UniqueTensor
from elasticdl_b200.layers.dense_table import DenseTableEmbedding, DenseTableEmbeddingBag
from elasticdl_b200.layers.embedding import Embedding
from elasticdl_b200.layers.embedding_bag import EmbeddingBag


def find_layer(model, layer_class):
    return [m for m in model.modules() if isinstance(m, layer_class)]


class _NoTiming:
    def start_record_time(self, *_):
        pass

    def end_record_time(self, *_):
        pass


class ParameterServerTrainer(object):
    """Parameter Server Trainer"""

    def __init__(self, model, ps_client, timing=None, args=None):
        self._optimizer = model.optimizer
        self._loss = model.loss
        self._model = model
        self._ps_client = ps_client
        if self._ps_client is None:
            raise ValueError("PS channels are not set up under parameter server strategy")
        self._model_versions_from_ps = [-1 for _ in range(self._ps_client.ps_num)]
        self._timing = timing or _NoTiming()
        self._get_model_steps = getattr(args, "get_model_steps", 1) if args is not None else 1
        self._non_embed_grads = None
        self._non_embed_vars = {}
        self._row_vars = {}  # dense-table weights: dense PS parameters whose rows are pulled and pushed by id
        self._evaluation_result = {}
        self._var_created = False
        self._model_version = -1
        # batched embedding lookups: None = not learnt yet, False = this model does not qualify,
        # else [(k, dim, [(layer, feature key)])] (see _learn_lookup_plan)
        self._batched_lookups = getattr(args, "batched_embedding_lookups", True) if args is not None else True
        self._lookup_plan = None if self._batched_lookups else False
        self._group_bets = []
        # CUDA-graph replay of the whole minibatch (see _train_minibatch_graphed): None = not decided yet,
        # False = this job does not qualify (stays eager), else the captured state
        self._use_cuda_graph = bool(getattr(args, "cuda_graph", False)) if args is not None else False
        self._graph_warmup = max(1, int(getattr(args, "cuda_graph_warmup", 3))) if args is not None else 3
        self._graph_state = None if self._use_cuda_graph else False
        self._eager_steps = 0
        self.graph_fallback_reason = None
        self._init_embeddings()

    # ------------------------------------------------------------------ embeddings
    def _init_embeddings(self):
        self._embedding_layers = find_layer(self._model, Embedding)
        param_names = {id(p): n for n, p in self._model.named_parameters()}
        for layer in self._embedding_layers:
            layer.set_lookup_embedding_func(self._ps_client.pull_embedding_vectors)
            if isinstance(layer, EmbeddingBag):
                layer.set_ps_group(self._ps_client.group)
            if self._is_dense_table(layer):  # its PS name is its weight's parameter name
                layer.set_embedding_weight_name(param_names[id(layer.weight)])
        self._report_embedding_info()

    @staticmethod
    def _is_dense_table(layer):
        return isinstance(layer, (DenseTableEmbedding, DenseTableEmbeddingBag))

    def _report_embedding_info(self):  # ps_trainer.py:186-214
        infos = [
            EmbeddingTableInfo(layer.embedding_weight_name, layer.output_dim, layer.embeddings_initializer,
                               DT_FLOAT, layer.input_dim)
            for layer in self._embedding_layers if not self._is_dense_table(layer)
        ]
        self._ps_client.push_embedding_table_infos(infos)

    def _set_tape_for_embedding(self, tape):
        for layer in self._embedding_layers:
            layer.set_tape(tape)

    def _reset_embedding(self):
        for layer in self._embedding_layers:
            layer.reset()
        self._group_bets = []

    # ------------------------------------------------------------------ batched lookups
    # The reference issues one lookup RPC per Embedding layer call (embedding_delegate.py:75-106), each one
    # a unique + pull of its own.  On one device that is ~6 launches and, for the exact [U, dim] BET shape,
    # two host reads per layer -- 76 layers of DeepFM make the step host-bound.  The trainer therefore
    # learns, during its first minibatch, which entry of `features` every Embedding layer is called with
    # (by object identity), and from the second minibatch on looks ALL layers up before the forward pass:
    # one unique launch and one gather per group of same-shaped layers, ONE pull launch for all tables,
    # the unique counts never leaving the device (DeviceIds).  A layer whose input is not the recorded
    # object simply takes its own per-layer path, and the plan is learnt again.
    @staticmethod
    def _feature_items(features):
        if isinstance(features, torch.Tensor):
            return [(None, features)]
        if isinstance(features, dict):
            return list(features.items())
        if isinstance(features, (list, tuple)):
            return list(enumerate(features))
        return []

    @staticmethod
    def _feature_at(features, key):
        return features if key is None else features[key]

    @staticmethod
    def _bag_stream_len(layer, src, offsets):
        """Length of the filled id stream ops.bag_prep makes of this bag input (nnz + B), None if it cannot."""
        if not (isinstance(src, torch.Tensor) and src.is_cuda and not src.is_sparse
                and src.dtype in (torch.int32, torch.int64)):
            return None
        if offsets is None:
            return src.numel() + src.shape[0] if src.dim() == 2 and src.shape[0] > 0 else None
        if not (isinstance(offsets, torch.Tensor) and offsets.is_cuda and offsets.dim() == 1 and src.dim() == 1
                and offsets.dtype in (torch.int32, torch.int64)):
            return None
        batch = offsets.numel() - (1 if layer.include_last_offset else 0)
        return src.numel() + batch if batch > 0 else None

    def _learn_lookup_plan(self, features):
        by_obj = {id(v): k for k, v in self._feature_items(features)}
        groups = {}
        for layer in self._embedding_layers:
            seen = layer._inputs_seen
            if len(seen) != 1:
                return False  # called twice (or never): keep per-layer lookups
            if isinstance(layer, EmbeddingBag):  # its ids are the stream ops.bag_prep makes of (input, offsets)
                src, offsets = seen[0]
                if id(src) not in by_obj or (offsets is not None and id(offsets) not in by_obj):
                    return False
                k = self._bag_stream_len(layer, src, offsets)
                if k is None:
                    return False
                key = (by_obj[id(src)], None if offsets is None else by_obj[id(offsets)])
                groups.setdefault(("bag", k, layer.output_dim), []).append((layer, key))
                continue
            if id(seen[0]) not in by_obj:
                return False  # called on a tensor derived from the features: keep per-layer lookups
            src = seen[0]
            if not (isinstance(src, torch.Tensor) and src.is_cuda and not src.is_sparse
                    and src.dtype == torch.int64 and src.numel() > 0):
                return False
            groups.setdefault(("rows", src.numel(), layer.output_dim), []).append((layer, by_obj[id(src)]))
        return [(k, dim, members) for (_, k, dim), members in groups.items()] or False

    def _prefetch_embeddings(self, features):
        """Look every Embedding layer of the plan up now.  Returns False (nothing done) when the features
        no longer match the plan."""
        g = self._ps_client.group
        work = []
        for k, dim, members in self._lookup_plan:
            kind = "bag" if isinstance(members[0][0], EmbeddingBag) else "rows"  # a plan group is of one kind
            srcs = []
            for layer, key in members:
                try:
                    if kind == "bag":
                        src = (self._feature_at(features, key[0]),
                               None if key[1] is None else self._feature_at(features, key[1]))
                    else:
                        src = self._feature_at(features, key)
                except (KeyError, IndexError, TypeError):
                    return False
                if kind == "bag":
                    if self._bag_stream_len(layer, *src) != k:
                        return False
                elif not (isinstance(src, torch.Tensor) and src.is_cuda and src.dtype == torch.int64
                          and not src.is_sparse and src.numel() == k):
                    return False
                srcs.append(src)
            work.append((kind, k, dim, members, srcs))
        requests, staged = [], []
        dedups = {}  # layer groups looked up with the SAME feature tensors (DeepFM's deep and wide families) share one dedup
        for kind, k, dim, members, srcs in work:
            T = len(members)
            # the layers' input_dim bounds the ids of each segment: direct-address dedup instead of hashing
            bounds = tuple(int(layer.input_dim or 0) for layer, _ in members)
            preps = [layer.prep(*src) for (layer, _), src in zip(members, srcs)] if kind == "bag" else None
            streams = [p[0] for p in preps] if kind == "bag" else srcs
            dkey = (k, tuple(id(s) for s in streams), bounds)
            if dkey not in dedups:
                flat = [s.reshape(-1) for s in streams]
                step = k * 8
                if all(f.is_contiguous() for f in flat) and all(
                        flat[t].data_ptr() == flat[0].data_ptr() + t * step for t in range(T)) and T > 1 \
                        and flat[0]._base is not None and flat[0]._base is flat[-1]._base:
                    ids = torch.as_strided(flat[0], (T * k,), (1,))  # the features are rows of one [T, k] array
                else:
                    ids = flat[0] if T == 1 else torch.cat(flat)
                dedups[dkey] = g.unique(ids, T, bounds=bounds if all(bounds) else None)
            uniq, inv, n_dev = dedups[dkey]
            bet = torch.zeros((T * k, dim), dtype=torch.float32, device=streams[0].device)
            for t, (layer, _) in enumerate(members):
                requests.append((layer.embedding_weight_name, uniq[t * k:(t + 1) * k], n_dev[t:t + 1],
                                 bet[t * k:(t + 1) * k]))
            staged.append((kind, k, dim, members, srcs, preps, uniq, inv, n_dev, bet))
        self._ps_client.pull_embedding_vectors_into(requests)
        for kind, k, dim, members, srcs, preps, uniq, inv, n_dev, bet in staged:
            T = len(members)
            bet.requires_grad_(True)
            if kind == "bag":  # each bag combines its own segment of the rows: SparseCombine over (bet, inv) slices
                for t, (layer, _) in enumerate(members):
                    _, ws, batch, nnz = preps[t]
                    layer._prefetched = (srcs[t][0], srcs[t][1], bet[t * k:(t + 1) * k], inv[t * k:(t + 1) * k], ws,
                                         batch, nnz)
            else:
                rows = ops.GatherRows.apply(bet, inv, T, k, dim).view(T, k, dim).unbind(0)
                for t, (layer, _) in enumerate(members):
                    layer._prefetched = (srcs[t], rows[t])
            self._group_bets.append((bet, uniq, n_dev, k, members))
        return True

    # ------------------------------------------------------------------ model pull
    def _get_model(self):  # ps_trainer.py:149-184
        self._timing.start_record_time("get_model")
        dense_params, uninit_ps = self._ps_client.pull_dense_parameters(
            list(range(self._ps_client.ps_num)), self._model_versions_from_ps, skip=self._row_vars)
        if len(uninit_ps) > 0:
            ps_vars = {**self._non_embed_vars, **self._row_vars}  # dense tables are initialised whole, once
            for ps_id in uninit_ps:
                parameters = [Tensor(name, ps_vars[name].detach(), None)
                              for name in self._ps_client.ps_to_parameter[ps_id]]
                self._ps_client.push_dense_parameters(parameters, ps_id, self._model_versions_from_ps[ps_id])
            ps_params, uninit = self._ps_client.pull_dense_parameters(uninit_ps, self._model_versions_from_ps,
                                                                      skip=self._row_vars)
            if len(uninit) > 0:
                raise RuntimeError("PS initialization failed")
            dense_params.update(ps_params)
        with torch.no_grad():
            for k, v in dense_params.items():
                self._non_embed_vars[k].copy_(torch.as_tensor(v).reshape(self._non_embed_vars[k].shape))
        self._model_version = max(self._model_versions_from_ps)
        self._timing.end_record_time("get_model")

    def init_variables_if_need(self, features, labels=None):  # ps_trainer.py:304-342
        if self._var_created:
            return
        row_names = {layer.embedding_weight_name for layer in self._embedding_layers if self._is_dense_table(layer)}
        params = {name: p for name, p in self._model.named_parameters() if p.requires_grad}
        self._non_embed_vars = {name: p for name, p in params.items() if name not in row_names}
        self._row_vars = {name: p for name, p in params.items() if name in row_names}
        shapes = {name: tuple(p.shape) for name, p in params.items()}
        self._ps_client.partition_dense_parameters(params.keys(), shapes=shapes)
        self._var_created = True

    def get_trainable_items(self):
        bets = [bet for (bet, _, _, _, _) in self._group_bets]
        for layer in self._embedding_layers:
            bets.extend(bet for (bet, _) in layer.embedding_and_ids)
        return list(self._non_embed_vars.values()) + bets

    # ------------------------------------------------------------------ train step
    def train_minibatch(self, features, labels, train_with_local_model=False):  # ps_trainer.py:371-385
        self.init_variables_if_need(features, labels)
        if self._graph_state is not False and not train_with_local_model:
            out = self._train_minibatch_graphed(features, labels)
            if out is not None:
                return out
        if not train_with_local_model:
            self._get_model()
        loss, grads = self._training_process_eagerly(features, labels)
        self._eager_steps += 1
        return (*self._update_global_model(grads), loss)

    # ------------------------------------------------------------------ the minibatch as ONE CUDA graph
    # args.cuda_graph=True.  The reference's step is a chain of RPCs and TF ops the worker drives one by one
    # (ps_trainer.py:371-414); on one device the same chain is ~300 kernel launches (76 lookups, the eager torch
    # model forward / backward, the push) and the step is bound by the host issuing them, not by the GPU.  After
    # `cuda_graph_warmup` eager minibatches (variables created and initialised on the PS, the lookup plan learnt,
    # every workspace at its final size) the trainer captures ONE minibatch -- pull of the dense parameters
    # straight into the model's tensors, batched lookups, forward, loss, autograd, push with the counts and the
    # versions kept on the device -- into a CUDA graph over static copies of (features, labels), and from then
    # on a minibatch is: copy the inputs in, replay, read the error word and the new versions.  Same kernels,
    # same order, same results as the eager step (tests/test_gpu_layer_trainer.py).  What does not qualify stays
    # eager, with the reason in `graph_fallback_reason`: a sync-SGD or staleness-modulated PS (the versions a push
    # carries would be baked into the graph), get_model_steps > 1, host-side or sparse features, per-layer
    # lookups (they read counts back), a learning rate or feature signature that keeps changing.
    @staticmethod
    def _rebuild_features(features, values):
        if isinstance(features, torch.Tensor):
            return values[0]
        if isinstance(features, dict):
            return dict(zip(features.keys(), values))
        return type(features)(values) if isinstance(features, tuple) else list(values)

    def _graph_signature(self, features, labels):
        items = self._feature_items(features)
        if not items:
            return None
        sig = []
        for k, v in items + [("__labels__", labels)]:
            if not (isinstance(v, torch.Tensor) and v.is_cuda and not v.is_sparse):
                return None
            sig.append((k, tuple(v.shape), v.dtype, v.device.index))
        # a schedule the push evaluates on the device is part of the captured launch; the host's lr is not used
        sched = getattr(self._ps_client.group, "lr_schedule", None)
        lr = float(self._optimizer.param_groups[0]["lr"]) if sched is None else ("lr_schedule", sched.key())
        return (type(features).__name__, tuple(sig), lr)

    @staticmethod
    def _as_one(tensors):
        """The flat view covering `tensors` when they are consecutive contiguous pieces of one storage, else None."""
        t0 = tensors[0]
        end = t0.data_ptr()
        for t in tensors:
            if not t.is_contiguous() or t.dtype != t0.dtype or t.data_ptr() != end \
                    or t.untyped_storage().data_ptr() != t0.untyped_storage().data_ptr():
                return None
            end += t.numel() * t.element_size()
        total = sum(t.numel() for t in tensors)
        return torch.as_strided(t0, (total,), (1,))

    @staticmethod
    def _static_like(tensors):
        """Static copies of `tensors`; the tensors of one dtype are carved out of ONE buffer in order, so features
        that were rows of one array stay rows of one array (the batched lookup keeps its zero-copy id view and the
        per-step input copy is one kernel per dtype)."""
        by_dtype = {}
        for i, t in enumerate(tensors):
            by_dtype.setdefault(t.dtype, []).append(i)
        out, groups = [None] * len(tensors), []
        for dt, idx in by_dtype.items():
            buf = torch.empty(sum(tensors[i].numel() for i in idx), dtype=dt, device=tensors[idx[0]].device)
            off = 0
            for i in idx:
                n = tensors[i].numel()
                out[i] = buf[off:off + n].view(tensors[i].shape)
                off += n
            groups.append((buf, idx))
        return out, groups

    @staticmethod
    def _copy_inputs(st, srcs):
        for buf, idx in st["groups"]:
            one = ParameterServerTrainer._as_one([srcs[i] for i in idx])
            if one is not None:
                buf.copy_(one)
            else:
                torch._foreach_copy_([st["statics"][i] for i in idx], [srcs[i] for i in idx])

    def _graph_eligible(self):
        g = self._ps_client.group
        if not getattr(g, "use_async", True):
            return "sync-SGD PS group"
        if getattr(g, "lr_staleness_modulation", False):
            return "lr staleness modulation needs the pulled versions on every push"
        if self._get_model_steps > 1:
            return "get_model_steps > 1"
        if self._embedding_layers and not self._lookup_plan:
            return "no batched lookup plan for this model"
        for name, p in self._non_embed_vars.items():
            if not (p.is_cuda and p.dtype == torch.float32 and p.is_contiguous() and name in g.tables):
                return "parameter %s is not a contiguous float32 device tensor registered on the PS" % name
        return None

    def _pull_dense_into_model(self):
        """_get_model without the version handshake: every dense parameter of every shard, written by the pull
        kernel straight into the model's own tensors (always the latest values; the Go PS would also resend them,
        server.go:150, because the version a worker that just pushed holds is never ahead of the shard's)."""
        c = self._ps_client
        names = [n for ps_id in sorted(c.ps_to_parameter) for n in c.ps_to_parameter[ps_id] if n in self._non_embed_vars]
        c.group.pull_dense(names, into={n: self._non_embed_vars[n].data for n in names})

    def _capture_minibatch(self, features, labels, sig):
        srcs = [v for _, v in self._feature_items(features)] + [labels]
        statics, groups = self._static_like(srcs)
        st = {"sig": sig, "statics": statics, "groups": groups}
        self._copy_inputs(st, srcs)
        s_features = self._rebuild_features(features, statics[:-1])
        self._reset_embedding()
        graph = torch.cuda.CUDAGraph()
        torch.cuda.current_stream().synchronize()
        with torch.cuda.graph(graph):
            self._pull_dense_into_model()
            loss, grads = self._training_process_eagerly(s_features, statics[-1])
            if self._embedding_layers and (not self._group_bets
                                           or any(layer.embedding_and_ids for layer in self._embedding_layers)):
                raise RuntimeError("the batched lookup plan did not cover this minibatch")
            self._report_gradient(grads, sync=False)
        self._reset_embedding()
        st.update(graph=graph, loss=loss, grads=grads)
        return st

    def _train_minibatch_graphed(self, features, labels):
        """One minibatch by graph replay; None = run this one eagerly."""
        st = self._graph_state
        sig = self._graph_signature(features, labels)
        if isinstance(st, dict) and sig == st["sig"]:
            self._pending_sig = None
            self._copy_inputs(st, [v for _, v in self._feature_items(features)] + [labels])
        else:
            if sig is None or self._eager_steps < self._graph_warmup:
                return None  # host-side / sparse inputs cannot be staged; or still warming up
            if isinstance(st, dict) and sig != getattr(self, "_pending_sig", None):
                # a one-off (the short last batch of an epoch) runs eagerly and the graph is kept; the same new
                # signature twice in a row (a new learning rate, a new batch size) is captured again
                self._pending_sig = sig
                return None
            self._pending_sig = None
            why = self._graph_eligible()
            recaptures = st["recaptures"] + 1 if isinstance(st, dict) else 0
            if why is None and recaptures > 4:
                why = "the learning rate or the feature signature keeps changing"
            if why is not None:
                self._graph_state, self.graph_fallback_reason = False, why
                return None
            stream = torch.cuda.current_stream()
            try:
                st = self._capture_minibatch(features, labels, sig)
            except Exception as err:  # anything the capture cannot hold (a host read, an allocation outside the pool)
                torch.cuda.set_stream(stream)  # a failed capture_end leaves torch on the capture stream
                self._reset_embedding()
                torch.cuda.synchronize()
                self._graph_state = False
                self.graph_fallback_reason = "capture failed: %s: %s" % (type(err).__name__, err)
                return None
            st["recaptures"] = recaptures
            self._graph_state = st
        g = self._ps_client.group
        self._timing.start_record_time("batch_process")
        st["graph"].replay()
        loss = st["loss"].clone()
        g.check()  # device sync + the error word (an id outside its table, ...)
        versions = g._pinned_versions[: g.n_shards].tolist()
        self._timing.end_record_time("batch_process")
        # the model this step trained on was pulled at (or after) the versions known before the step
        self._model_version = max(max(self._model_versions_from_ps), self._model_version)
        self._model_versions_from_ps = [int(v) for v in versions]
        return True, max(self._model_versions_from_ps), loss

    def _training_process_eagerly(self, features, labels):  # ps_trainer.py:391-400
        self._set_tape_for_embedding(True)
        prefetched = bool(self._lookup_plan) and self._prefetch_embeddings(features)
        outputs = self._model(features)
        if self._batched_lookups:
            stale = [layer for layer in self._embedding_layers if layer._prefetched is not None]
            if stale:  # a prefetched layer was not called with the recorded object (or not called at all)
                raise RuntimeError("batched embedding lookup of %s was not consumed by the model; construct the "
                                   "trainer with args.batched_embedding_lookups=False" % stale[0].name)
            if not prefetched:
                self._lookup_plan = self._learn_lookup_plan(features)
        loss = self._loss(labels, outputs)
        grads = torch.autograd.grad(loss, self.get_trainable_items(), allow_unused=True)
        return loss.detach(), grads

    def _report_gradient(self, gradients, sync=True):  # ps_trainer.py:239-280
        self._timing.start_record_time("report_gradient")
        grads = []
        names = list(self._non_embed_vars.keys())
        for i, name in enumerate(names):
            if gradients[i] is None:
                continue
            grads.append(Tensor(name, gradients[i], None))
        edl_grads = []
        bet_number = 0
        edl_embedding_grads = gradients[len(names):]
        for (bet, uniq, n_dev, k, members) in self._group_bets:  # batched lookups: one BET per layer group
            g_bet = edl_embedding_grads[bet_number]
            for t, (layer, _) in enumerate(members):
                (grads if self._is_dense_table(layer) else edl_grads).append(
                    UniqueTensor(layer.embedding_weight_name, g_bet[t * k:(t + 1) * k],
                                 DeviceIds(uniq[t * k:(t + 1) * k], n_dev[t:t + 1])))
            bet_number += 1
        edl_embedding_grads = edl_embedding_grads[bet_number:]
        bet_number = 0
        for layer in self._embedding_layers:
            for i, (_, batch_ids) in enumerate(layer.embedding_and_ids):
                (grads if self._is_dense_table(layer) else edl_grads).append(
                    UniqueTensor(layer.embedding_weight_name, edl_embedding_grads[i + bet_number], batch_ids))
            bet_number += len(layer.embedding_and_ids)
        if len(edl_embedding_grads) != bet_number:
            raise ValueError("elasticdl.layers.embedding related gradient number %d does not match the "
                             "number of its output tensor %d." % (len(edl_embedding_grads), bet_number))
        learning_rate = float(self._optimizer.param_groups[0]["lr"])
        accepted, max_version = self._ps_client.push_gradients(
            grads, edl_grads, learning_rate, self._model_versions_from_ps, **({} if sync else {"sync": False}))
        self._timing.end_record_time("report_gradient")
        return accepted, max_version

    def _update_global_model(self, grads):  # ps_trainer.py:408-414
        accepted, min_model_version = self._report_gradient(grads)
        if accepted and self._get_model_steps > 1:
            self._non_embed_grads = grads[: len(self._non_embed_vars)]
        self._reset_embedding()
        return accepted, min_model_version

    def _update_local_model(self):  # ps_trainer.py:139-147 (SSP local update of dense vars)
        if not self._non_embed_grads:
            return
        for p, g in zip(self._non_embed_vars.values(), self._non_embed_grads):
            p.grad = g
        self._optimizer.step()
        self._optimizer.zero_grad(set_to_none=True)
        self._non_embed_grads = None

    # ------------------------------------------------------------------ the worker's training loop
    def train_loop(self, batches, max_minibatch_retry_num=64, on_step=None, callbacks=None):
        """The training loop of elasticdl/python/worker/worker.py:338-370 around train_minibatch, with its
        `get_model_steps` logic (SSP, docs/designs/async_sgd.md:129-157): the dense model is pulled from the
        PS only every `get_model_steps` minibatches (and after a failed one); in between the worker trains
        with its LOCAL model, which `_update_local_model` advances with the gradients it just pushed
        (dense variables only -- embedding rows are always pulled fresh).  A minibatch whose push is not
        accepted is retried up to `max_minibatch_retry_num` times (worker.py:181-234: "Worker got stuck").
        batches: iterable of (features, labels).  Returns [(version, loss)] per minibatch.
        callbacks (elasticdl_b200.callbacks): each is given the model, and its on_train_batch_begin is called with
        the model version before every minibatch (worker.py:198).  On an async group a LearningRateScheduler over a
        declarative schedule is also installed on the PS group, whose pushes then evaluate it on the device, so that
        the graphed step needs no re-capture for it; on a sync-SGD group the schedule is evaluated on the host only,
        as the reference does.  Passing callbacks replaces the group's schedule (callbacks without a declarative
        scheduler remove one set by hand), and the schedule stays installed after train_loop returns; without
        callbacks the group's schedule is left as it is."""
        if callbacks is not None:
            from elasticdl_b200.callbacks import device_schedule

            callbacks = list(callbacks)
            for cb in callbacks:
                cb.set_model(self._model)
            group = self._ps_client.group
            group.set_lr_schedule(device_schedule(callbacks) if group.use_async else None)
        local_update_count = self._get_model_steps
        last_training_minibatch_failed = False
        out = []
        for features, labels in batches:
            if last_training_minibatch_failed or local_update_count >= self._get_model_steps:
                local_update_count = 0
                train_with_local_model = False
            else:
                train_with_local_model = True
            err_msg = ""
            try:  # _safe_process_minibatch (worker.py:274-300)
                for _ in range(max_minibatch_retry_num):
                    for cb in callbacks or ():
                        cb.on_train_batch_begin(self.get_model_version())
                    accepted, version, loss = self.train_minibatch(features, labels, train_with_local_model)
                    if accepted:
                        break
                else:
                    raise RuntimeError("Worker got stuck")
            except RuntimeError as err:
                err_msg = str(err)
            local_update_count += 1
            if err_msg:
                last_training_minibatch_failed = True
                out.append((None, None))
            else:
                last_training_minibatch_failed = False
                if local_update_count < self._get_model_steps:
                    self._update_local_model()
                out.append((version, loss))
            if on_step is not None:
                on_step(train_with_local_model, err_msg)
        return out

    # ------------------------------------------------------------------ eval / misc
    def get_model_version(self):
        return self._model_version

    def evaluate_minibatch(self, features, labels):
        with torch.no_grad():
            outputs = self._model(features)
        self._evaluation_result.setdefault("output", []).append(
            outputs if not isinstance(outputs, torch.Tensor) else outputs.cpu().numpy())
        self._evaluation_result.setdefault("label", []).append(np.asarray(torch.as_tensor(labels).cpu()))
        self._reset_embedding()

    def get_evaluation_result(self):
        return self._evaluation_result

    def reset_evaluation_result(self):
        self._evaluation_result = {}
