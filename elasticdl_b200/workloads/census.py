"""The census wide & deep model (model_zoo/census_wide_deep_model/wide_deep_functional_api.py:164-212) trained on
the parameter-server step: raw Adult rows -> census_transform -> the census tower (csrc/census_tower.cu) -> push.

Parameters, as Keras creates them (a layer without a name gets its snake-cased class name, uniquified per name by
a running count in creation order: "embedding", "embedding_1", ...; keras backend.unique_object_name), in the flat
order of include/b200_census.h:
    dense/kernel:0 [24, 16], dense/bias:0 [16], dense_1/kernel:0 [16, 8], dense_1/bias:0 [8],
    dense_2/kernel:0 [8, 4], dense_2/bias:0 [4],
    embedding/embeddings:0 [28, 1], embedding_1/embeddings:0 [75, 1]                       (wide, groups 1, 2)
    embedding_2/embeddings:0 [28, 8], embedding_3/embeddings:0 [75, 8], embedding_4/embeddings:0 [115, 8] (deep)
Every table is under 2 MB, so the reference's ModelHandler keeps it a dense Keras parameter; its gradient is an
IndexedSlices that the PS applies with the Indexed kernels (only the rows of the batch move).  Each is one dense
PS parameter here, on shard string_to_id(name), and the tables' rows are pushed with b200ps_push_rows.
"""
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib
from elasticdl_b200._lib import CensusArgs, check
from elasticdl_b200.common.hash_utils import string_to_id
from elasticdl_b200.workloads.census_features import ID_GROUP_DIMS, STRING_WIDTH, census_transform

GROUP_ROWS = tuple(ID_GROUP_DIMS[g] for g in ("group1", "group2", "group3"))  # 28, 75, 115
PARAMS = [("dense/kernel:0", (24, 16)), ("dense/bias:0", (16,)), ("dense_1/kernel:0", (16, 8)),
          ("dense_1/bias:0", (8,)), ("dense_2/kernel:0", (8, 4)), ("dense_2/bias:0", (4,)),
          ("embedding/embeddings:0", (28, 1)), ("embedding_1/embeddings:0", (75, 1)),
          ("embedding_2/embeddings:0", (28, 8)), ("embedding_3/embeddings:0", (75, 8)),
          ("embedding_4/embeddings:0", (115, 8))]
MLP_NAMES = [n for n, _ in PARAMS[:6]]
TABLE_NAMES = [n for n, _ in PARAMS[6:]]
TABLE_GROUP = (0, 1, 0, 1, 2)
TABLE_DIM = (1, 1, 8, 8, 8)
N_PARAMS, N_MLP = 2419, 572
UNIQ_OFF = (0, 28, 103, 131, 206)
N_UNIQ = 321
GSUM_OFF = (0, 28, 103, 327, 927)
N_GSUM = 1847
TILE = 256  # B200_CENSUS_TILE


def _offsets():
    out, o = {}, 0
    for n, s in PARAMS:
        out[n] = o
        o += int(np.prod(s))
    assert o == N_PARAMS and out[TABLE_NAMES[0]] == N_MLP
    assert tuple(out[n] - N_MLP for n in TABLE_NAMES) == GSUM_OFF
    return out


OFFSETS = _offsets()


def flat_views(flat):
    """{name: view of the flat buffer in the parameter's shape}."""
    return {n: flat[OFFSETS[n]:OFFSETS[n] + int(np.prod(s))].view(s) for n, s in PARAMS}


def initial_params(seed, device):
    """The reference's initialisers: Keras "uniform" embeddings U(-0.05, 0.05), glorot-uniform Dense kernels
    U(-sqrt(6 / (in + out)), +), zero biases.  float32 [2419]."""
    gen = torch.Generator(device=device).manual_seed(int(seed))
    flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=device)
    for n, v in flat_views(flat).items():
        if n.endswith("embeddings:0"):
            v.copy_((torch.rand(v.shape, generator=gen, device=device) * 2 - 1) * 0.05)
        elif n.endswith("kernel:0"):
            lim = float(np.sqrt(6.0 / (v.shape[0] + v.shape[1])))
            v.copy_((torch.rand(v.shape, generator=gen, device=device) * 2 - 1) * lim)
    return flat


def eval_metrics_fn():
    """The census model's evaluation metrics (model_zoo/census_wide_deep_model/wide_deep_functional_api.py:62-71):
    accuracy of the LOGITS thresholded at 0.5 (quirk Q12, DESIGN.md section 4) and the AUC of the probabilities."""
    from elasticdl_b200.common.evaluation_utils import zoo_eval_metrics

    return zoo_eval_metrics(0.5)


class CensusTowerCall:
    """The census tower's output buffers and workspace for batch B on `device`, and one launch over them."""

    def __init__(self, B, device):
        self.B = int(B)
        if self.B < 1:
            raise ValueError("batch size must be >= 1, not %d" % self.B)
        self.device = torch.device(device)
        self.lib = _lib.lib()
        f32 = dict(dtype=torch.float32, device=self.device)
        self.loss = torch.zeros(1, **f32)
        self.logits = torch.zeros(self.B, **f32)
        self.grads = torch.zeros(N_MLP, **f32)
        self.uniq = torch.zeros(N_UNIQ, dtype=torch.int64, device=self.device)
        self.n_unique = torch.zeros(5, dtype=torch.int32, device=self.device)
        self.gsum = torch.zeros(N_GSUM, **f32)
        self.error = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            nbytes = self.lib.b200_census_workspace_bytes(self.B)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        a = CensusArgs()
        a.B = self.B
        a.loss, a.logits, a.grads = self.loss.data_ptr(), self.logits.data_ptr(), self.grads.data_ptr()
        a.uniq, a.n_unique, a.gsum = self.uniq.data_ptr(), self.n_unique.data_ptr(), self.gsum.data_ptr()
        a.error, a.workspace, a.workspace_bytes = self.error.data_ptr(), self.workspace.data_ptr(), nbytes
        self.args = a

    def check_inputs(self, ids, labels, flat):
        B, dev = self.B, self.device

        def need(t, name, dtype, shape):
            if not (isinstance(t, torch.Tensor) and t.device == dev and t.dtype == dtype
                    and tuple(t.shape) == shape and t.is_contiguous()):
                got = (tuple(t.shape), t.dtype, t.device) if isinstance(t, torch.Tensor) else type(t)
                raise ValueError("%s must be a contiguous %s tensor of shape %s on %s, not %s"
                                 % (name, dtype, shape, dev, got))

        need(ids, "ids", torch.int32, (12, B))
        need(labels, "labels", torch.float32, (B,))
        need(flat, "params", torch.float32, (N_PARAMS,))

    def launch(self, ids, labels, flat, reference_reshape):
        """One tower launch on the current stream (no checks, no host read)."""
        a = self.args
        a.ids, a.labels, a.params = ids.data_ptr(), labels.data_ptr(), flat.data_ptr()
        a.reference_reshape = 1 if reference_reshape else 0
        with torch.cuda.device(self.device):
            rc = self.lib.b200_census_tower(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc:
            msg = self.lib.b200_census_last_error().decode("utf-8", "replace")
            raise (ValueError if rc == _lib.EINVAL else RuntimeError)("b200_census_tower failed (%d): %s" % (rc, msg))

    def check_error(self):
        """Raise PSRangeError (a ValueError) if a launch since the last check read an id outside its group, and
        clear the count.  Reads one int from the device."""
        n = int(self.error.item())
        if n:
            self.error.zero_()
            raise _lib.PSRangeError(_lib.ERANGE, "%d census ids outside [0, rows of their group) %s were read as "
                                                 "row 0" % (n, GROUP_ROWS))

    def outputs(self):
        """{loss, logits, grads, uniq [5], n_unique [5], gsum [5 segments: [rows, dim]]} (views of the buffers)."""
        out = {"loss": self.loss.reshape(()), "logits": self.logits, "grads": self.grads, "n_unique": self.n_unique,
               "uniq": [], "gsum": []}
        for t in range(5):
            rows = GROUP_ROWS[TABLE_GROUP[t]]
            out["uniq"].append(self.uniq[UNIQ_OFF[t]:UNIQ_OFF[t] + rows])
            out["gsum"].append(self.gsum[GSUM_OFF[t]:GSUM_OFF[t] + rows * TABLE_DIM[t]].view(rows, TABLE_DIM[t]))
        return out


def census_tower(ids, labels, flat, reference_reshape=False):
    """The census tower kernel on one batch: ids int32 [12, B], labels float32 [B], flat float32 [2419], all on
    one device.  Synchronises, raises ValueError for ids outside their group (after the launch, which read them
    as row 0), and returns CensusTowerCall.outputs() of fresh buffers."""
    call = CensusTowerCall(labels.shape[0] if isinstance(labels, torch.Tensor) and labels.dim() == 1 else 0,
                           flat.device if isinstance(flat, torch.Tensor) else "cuda")
    call.check_inputs(ids, labels, flat)
    call.launch(ids, labels, flat, reference_reshape)
    call.check_error()
    return call.outputs()


class CensusWideDeepEngine:
    """One async worker of the census wide & deep model on the parameter-server step.

    group: an async PSGroup without lr staleness modulation (ValueError otherwise: the captured step carries no
    pulled versions; the drop-in ParameterServerTrainer covers those modes).  register=True registers the eleven
    parameters and sets their initial values first-writer-wins (as PushModel does); register=False attaches to a
    group.clone_view() of a group where another engine registered them, for another worker thread.
    step(numeric float32 [4, B], strings uint8 [8, B, 32], labels float32 [B]) runs pull_dense (into the flat
    buffer) -> census_transform -> the tower -> push_begin -> push_dense (MLP) -> push_rows (the five tables'
    touched rows, counts on the device) -> push_end, with no host read, and returns the loss on the device.
    capture() / replay() run the same step as one CUDA graph over static inputs; a new learning rate re-captures."""

    def __init__(self, group, batch, lr, reference_reshape=False, seed=0, register=True):
        if not getattr(group, "use_async", True):
            raise ValueError("CensusWideDeepEngine trains async only: a sync-SGD group needs the drop-in trainer")
        if getattr(group, "lr_staleness_modulation", False):
            raise ValueError("CensusWideDeepEngine pushes without model versions: a group with "
                             "lr_staleness_modulation needs the drop-in trainer")
        self.B = int(batch)
        if self.B < 1:
            raise ValueError("batch size must be >= 1, not %d" % self.B)
        self.group = group if register else group.clone_view()
        g = self.group
        self.device = g.device
        self.lr = float(lr)
        self.reference_reshape = bool(reference_reshape)
        self.owner = {n: string_to_id(n, g.n_shards) for n, _ in PARAMS}
        if register:
            for n, s in PARAMS:
                g.register_dense(n, s, self.owner[n])
            g.commit()
            init = flat_views(initial_params(seed, self.device))
            for s in range(g.n_shards):  # first writer wins (PushModel, server.go:209-221)
                if s in g.local_shards and g.try_init(s):
                    mine = [(n, init[n]) for n, _ in PARAMS if self.owner[n] == s]
                    if mine:
                        g.set_dense(mine)
                    g.finish_init(s, 0)
        tids = [g.lookup(n)[0] for n, _ in PARAMS]  # PSNotFound when no engine registered them
        self.flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=self.device)
        self.views = flat_views(self.flat)
        self.ids = torch.zeros((12, self.B), dtype=torch.int32, device=self.device)
        self.transform = census_transform(torch.int32, device=self.device)
        self.tower = CensusTowerCall(self.B, self.device)
        t = self.tower
        self.pull_segs = g.make_segs([(tid, 0, None, None, self.views[n]) for tid, (n, _) in zip(tids, PARAMS)])
        self.push_dense_segs = g.make_segs([(tids[i], 0, None, None, t.grads[OFFSETS[n]:OFFSETS[n] + int(np.prod(s))])
                                            for i, (n, s) in enumerate(PARAMS[:6])])
        out = t.outputs()
        self.push_rows_segs = g.make_segs([(tids[6 + k], GROUP_ROWS[TABLE_GROUP[k]], out["uniq"][k],
                                            t.n_unique[k:k + 1], out["gsum"][k]) for k in range(5)])
        self.zero_versions = [0] * g.n_shards
        self._eval_tower = None  # evaluate()'s tower buffers (lazy)
        self.graph = None
        self._graph_lr = None
        self.steps = 0

    # ------------------------------------------------------------------ inputs
    def _check_batch(self, numeric, strings, labels):
        B, dev = self.B, self.device
        for t, name, dtype, shape in ((numeric, "numeric", torch.float32, (4, B)),
                                      (strings, "strings", torch.uint8, (8, B, STRING_WIDTH)),
                                      (labels, "labels", torch.float32, (B,))):
            if not (isinstance(t, torch.Tensor) and t.device == dev and t.dtype == dtype and tuple(t.shape) == shape
                    and t.is_contiguous()):
                got = (tuple(t.shape), t.dtype, t.device) if isinstance(t, torch.Tensor) else type(t)
                raise ValueError("%s must be a contiguous %s tensor of shape %s on %s, not %s"
                                 % (name, dtype, shape, dev, got))

    # ------------------------------------------------------------------ the step
    def _step(self, numeric, strings, ids, labels):
        g, lib = self.group, self.group.lib
        with torch.cuda.device(self.device):
            st = g._stream()
            arr, n = self.pull_segs
            check(lib.b200ps_pull_dense(g._h, arr, n, st))
            if ids is None:
                self.transform(numeric, strings, ids_out=self.ids)
                ids = self.ids
            self.tower.launch(ids, labels, self.flat, self.reference_reshape)
            g.push_begin(self.lr, self.zero_versions)
            arr, n = self.push_dense_segs
            check(lib.b200ps_push_dense(g._h, arr, n, st))
            arr, n = self.push_rows_segs
            check(lib.b200ps_push_rows(g._h, arr, n, st))
            g.push_end(sync=False)
        return self.tower.loss.reshape(())

    def step(self, numeric, strings, labels):
        """One training step from raw rows; returns the loss (device scalar, not synchronised)."""
        self._check_batch(numeric, strings, labels)
        out = self._step(numeric, strings, None, labels)
        self.steps += 1
        return out

    def step_ids(self, ids, labels):
        """One training step from the ids census_transform(torch.int32) gives: int32 [12, B]."""
        self.tower.check_inputs(ids, labels, self.flat)
        out = self._step(None, None, ids, labels)
        self.steps += 1
        return out

    def evaluate(self, numeric, strings, labels, metrics):
        """Forward only from raw rows: pull_dense -> census_transform -> the tower -> metrics.update_evaluation_metrics(
        {"logits": logits, "probs": sigmoid(logits)}, labels) (an EvaluationMetrics, e.g. of eval_metrics_fn()).
        There is no forward-only census kernel: the tower launch also computes the gradients, which evaluate()
        discards -- into buffers of its own, so the step's loss and gradients stay as they were -- and pushes
        nothing.  Returns the logits [B] on the device (overwritten by the next evaluate)."""
        self._check_batch(numeric, strings, labels)
        if self._eval_tower is None:
            self._eval_tower = CensusTowerCall(self.B, self.device)
        g = self.group
        with torch.cuda.device(self.device):
            arr, n = self.pull_segs
            check(g.lib.b200ps_pull_dense(g._h, arr, n, g._stream()))
            self.transform(numeric, strings, ids_out=self.ids)
            self._eval_tower.launch(self.ids, labels, self.flat, self.reference_reshape)
            logits = self._eval_tower.logits
            metrics.update_evaluation_metrics({"logits": logits, "probs": torch.sigmoid(logits)}, labels)
        return logits

    def check(self):
        """Raise PSRangeError (a ValueError) if a step or evaluate since the last check read an id outside its
        group (it used row 0 for it); one device read per tower."""
        if self._eval_tower is not None:
            self._eval_tower.check_error()
        self.tower.check_error()

    def set_lr(self, lr):
        """The learning rate the next pushes carry (the reference's schedule callback sets it per version);
        the captured graph is re-captured on the next replay."""
        self.lr = float(lr)

    # ------------------------------------------------------------------ CUDA graph
    def capture(self):
        """Capture one step over static inputs (self.s_numeric, self.s_strings, self.s_labels) into a CUDA graph
        on the current stream's device; the learning rate is baked in."""
        dev, B = self.device, self.B
        if self.graph is None:
            self.s_numeric = torch.zeros((4, B), dtype=torch.float32, device=dev)
            self.s_strings = torch.zeros((8, B, STRING_WIDTH), dtype=torch.uint8, device=dev)
            self.s_labels = torch.zeros(B, dtype=torch.float32, device=dev)
        torch.cuda.current_stream(dev).synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._step(self.s_numeric, self.s_strings, None, self.s_labels)
        self.graph, self._graph_lr = graph, self.lr
        return graph

    def replay(self, numeric, strings, labels):
        """step() through the captured graph (captured now if there is none or the learning rate changed)."""
        self._check_batch(numeric, strings, labels)
        if self.graph is None or self._graph_lr != self.lr:
            self.capture()
        self.s_numeric.copy_(numeric)
        self.s_strings.copy_(strings)
        self.s_labels.copy_(labels)
        self.graph.replay()
        self.steps += 1
        return self.tower.loss.reshape(())


class CensusWideDeep(torch.nn.Module):
    """The same model as a torch module for the drop-in ParameterServerTrainer: the tables are
    elasticdl_b200.layers.Embedding layers (row-sparse PS tables; only the rows of the batch are pulled and
    updated), the MLP is three torch Linear layers, both reshape modes.  forward((numeric, strings)) runs
    census_transform and sums each group's four lookups."""

    def __init__(self, lr, reference_reshape=False, optimizer="sgd"):
        super().__init__()
        from elasticdl_b200.layers import Embedding

        self.reference_reshape = bool(reference_reshape)
        self.wide = torch.nn.ModuleList([Embedding(1, input_dim=r, embeddings_initializer="uniform", name=n.split("/")[0])
                                         for n, r in zip(TABLE_NAMES[:2], GROUP_ROWS[:2])])
        self.deep = torch.nn.ModuleList([Embedding(8, input_dim=r, embeddings_initializer="uniform", name=n.split("/")[0])
                                         for n, r in zip(TABLE_NAMES[2:], GROUP_ROWS)])
        self.dense = torch.nn.ModuleList([torch.nn.Linear(24, 16), torch.nn.Linear(16, 8), torch.nn.Linear(8, 4)])
        self.transform = None  # built at the first forward (its vocabulary tables live on the device)
        opt = torch.optim.SGD if optimizer == "sgd" else torch.optim.Adam
        self.optimizer = opt(self.dense.parameters(), lr=lr)
        bce = torch.nn.BCEWithLogitsLoss()
        self.loss = lambda labels, logits: bce(logits, labels)

    def load_mlp(self, flat):
        """Copy the MLP block of a flat buffer (Keras [in, out] kernels) into the Linear layers."""
        v = flat_views(flat)
        with torch.no_grad():
            for i, lin in enumerate(self.dense):
                lin.weight.copy_(v[MLP_NAMES[2 * i]].t())
                lin.bias.copy_(v[MLP_NAMES[2 * i + 1]])

    def tower(self, wide, deep):
        """wide [2, B] and deep [3, B, 8] pooled lookups -> logits [B]."""
        B = deep.shape[1]
        x = deep.reshape(B, 24) if self.reference_reshape else deep.permute(1, 0, 2).reshape(B, 24)
        for lin in self.dense:
            x = lin(x)
        return wide.sum(0) + x.sum(1)

    def forward(self, features):
        numeric, strings = features
        if self.transform is None:
            self.transform = census_transform(torch.int64, device=numeric.device)
        ids, _ = self.transform(numeric, strings)
        wide = torch.stack([self.wide[g](ids[4 * g:4 * g + 4]).sum(0)[:, 0] for g in range(2)])
        deep = torch.stack([self.deep[g](ids[4 * g:4 * g + 4]).sum(0) for g in range(3)])
        return self.tower(wide, deep)
