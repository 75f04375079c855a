"""The frappe DeepFM model the reference's own tests train, on the parameter-server step:
ids -> dedup -> one row pull for both tables -> the frappe tower (csrc/frappe_tower.cu) -> push.

Two variants of one model (model_zoo/deepfm_edl_embedding/deepfm_edl_embedding.py:40-88 and
model_zoo/deepfm_functional_api/deepfm_functional_api.py:40-101): 10 ids per sample, zero-padded (`mask_zero`), a
64-wide deep table and a 1-wide bias table on the same ids, an FM over the masked rows, Dense(64) without
activation, Dense(1), mean sigmoid cross-entropy.  Parameters, by the names Keras gives them:
    embedding/embeddings:0 [*, 64], embedding_1/embeddings:0 [*, 1],
    dense/kernel:0 [640, 64], dense/bias:0 [64], dense_1/kernel:0 [64, 1], dense_1/bias:0 [1]
The four Dense parameters make the flat buffer of include/b200_frappe.h (41089 floats, Keras [in, out] kernels).

input_dim=None (deepfm_edl_embedding): the tables are hashed PS tables (unbounded ids, "uniform" rows created on
first pull, sharded id % N).  input_dim=5383 (deepfm_functional_api): each table is under 2 MB, so the reference
keeps it a dense Keras parameter; here it is one dense PS parameter [5383, dim] on shard string_to_id(name) whose
batch rows are pulled and pushed by id, as the census model's tables are.
"""
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib
from elasticdl_b200._lib import FrappeArgs, check
from elasticdl_b200.common.hash_utils import string_to_id

FIELDS = 10
DIM = 64
# the frappe fields and their cardinalities, as the dataset is published (not checked against data here)
FIELD_NAMES = ("user", "item", "daytime", "weekday", "isweekend", "homework", "cost", "weather", "country", "city")
FIELD_SIZES = (957, 4082, 7, 7, 2, 3, 2, 9, 80, 233)
N_IDS = sum(FIELD_SIZES)  # 5382 real ids, 1-based; 0 is the pad
INPUT_DIM = N_IDS + 1
FIELD_START = tuple(1 + int(v) for v in np.cumsum((0,) + FIELD_SIZES[:-1]))  # first id of every field
DEEP_NAME, WIDE_NAME = "embedding/embeddings:0", "embedding_1/embeddings:0"
DENSE_PARAMS = [("dense/kernel:0", (FIELDS * DIM, DIM)), ("dense/bias:0", (DIM,)), ("dense_1/kernel:0", (DIM, 1)),
                ("dense_1/bias:0", (1,))]
DENSE_NAMES = [n for n, _ in DENSE_PARAMS]
N_PARAMS = 41089  # B200_FRAPPE_PARAMS
TILE = 64  # B200_FRAPPE_TILE


def _offsets():
    out, o = {}, 0
    for n, s in DENSE_PARAMS:
        out[n] = o
        o += int(np.prod(s))
    assert o == N_PARAMS and [out[n] for n in DENSE_NAMES] == [0, 40960, 41024, 41088]
    return out


OFFSETS = _offsets()


def flat_views(flat):
    """{name: view of the flat dense buffer in the parameter's shape}."""
    return {n: flat[OFFSETS[n]:OFFSETS[n] + int(np.prod(s))].view(s) for n, s in DENSE_PARAMS}


def initial_dense(seed, device):
    """Glorot-uniform kernels U(-sqrt(6 / (in + out)), +) and zero biases, float32 [41089]."""
    gen = torch.Generator(device=device).manual_seed(int(seed))
    flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=device)
    for n, v in flat_views(flat).items():
        if n.endswith("kernel:0"):
            lim = float(np.sqrt(6.0 / (v.shape[0] + v.shape[1])))
            v.copy_((torch.rand(v.shape, generator=gen, device=device) * 2 - 1) * lim)
    return flat


def initial_table(seed, dim, device, rows=INPUT_DIM):
    """Keras "uniform" embeddings U(-0.05, 0.05), float32 [rows, dim] (the bounded variant's dense tables)."""
    gen = torch.Generator(device=device).manual_seed(int(seed) * 131 + int(dim))
    return (torch.rand((rows, dim), generator=gen, device=device) * 2 - 1) * 0.05


def synthetic_frappe_batch(B, seed, device, pad_fraction=0.0, zipf_s=1.05):
    """A frappe-shaped batch: ids int64 [B, 10] and labels float32 [B].

    Field f's ids are the contiguous 1-based range [FIELD_START[f], FIELD_START[f] + FIELD_SIZES[f]) -- 5382 ids
    in all, as the recordio generator builds its feature map -- drawn Zipf(zipf_s) within the field.  A fraction
    `pad_fraction` of the samples is left-padded (pad_sequences' default "pre"): 1..10 leading fields are 0.
    About one label in three is positive.  The frappe files themselves are not used: the cardinalities and the
    1:2 label ratio are the dataset's published description and are not checked against data here."""
    g = torch.Generator(device=device).manual_seed(int(seed))
    u = torch.rand((B, FIELDS), generator=g, device=device, dtype=torch.float64)
    rows = torch.tensor(FIELD_SIZES, device=device, dtype=torch.float64)
    a = 1.0 - zipf_s  # bounded-Pareto inverse CDF: rank in [1, N], P(rank) ~ rank^-s
    rank = torch.floor(((rows.pow(a) - 1.0) * u + 1.0).pow(1.0 / a)).clamp(min=1)
    rank = torch.minimum(rank, rows)
    ids = (rank - 1).to(torch.int64) + torch.tensor(FIELD_START, device=device, dtype=torch.int64)
    if pad_fraction > 0:
        padded = torch.rand(B, generator=g, device=device) < pad_fraction
        n_pad = torch.randint(1, FIELDS + 1, (B,), generator=g, device=device) * padded
        ids = torch.where(torch.arange(FIELDS, device=device) < n_pad.unsqueeze(1), torch.zeros_like(ids), ids)
    labels = (torch.rand(B, generator=g, device=device) < 1.0 / 3.0).float()
    return ids.contiguous(), labels


def eval_metrics_fn():
    """The frappe models' evaluation metrics (model_zoo/deepfm_edl_embedding/deepfm_edl_embedding.py:115-124,
    model_zoo/deepfm_functional_api/deepfm_functional_api.py:128-137): accuracy of logits > 0 and the AUC of the
    probabilities."""
    from elasticdl_b200.common.evaluation_utils import zoo_eval_metrics

    return zoo_eval_metrics(0.0)


class FrappeTowerCall:
    """The frappe tower's output buffers and workspace for batch B and up to `rows` unique ids on `device`, and
    one launch over them."""

    def __init__(self, B, device, rows=None):
        self.B = int(B)
        if self.B < 1:
            raise ValueError("batch size must be >= 1, not %d" % self.B)
        self.rows = int(rows) if rows is not None else FIELDS * self.B
        self.device = torch.device(device)
        self.lib = _lib.lib()
        f32 = dict(dtype=torch.float32, device=self.device)
        self.loss = torch.zeros(1, **f32)
        self.logits = torch.zeros(self.B, **f32)
        self.grads = torch.zeros(N_PARAMS, **f32)
        self.gsum_deep = torch.zeros((self.rows, DIM), **f32)
        self.gsum_wide = torch.zeros((self.rows, 1), **f32)
        nbytes = self.lib.b200_frappe_workspace_bytes(self.B)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        a = FrappeArgs()
        a.B = self.B
        a.loss, a.logits, a.grads = self.loss.data_ptr(), self.logits.data_ptr(), self.grads.data_ptr()
        a.gsum_deep, a.gsum_wide = self.gsum_deep.data_ptr(), self.gsum_wide.data_ptr()
        a.workspace, a.workspace_bytes = self.workspace.data_ptr(), nbytes
        self.args = a

    def check_inputs(self, ids, inv, n_unique, bet_deep, bet_wide, labels, flat):
        B, dev = self.B, self.device

        def need(t, name, dtype, shape):
            if not (isinstance(t, torch.Tensor) and t.device == dev and t.dtype == dtype
                    and tuple(t.shape) == shape and t.is_contiguous()):
                got = (tuple(t.shape), t.dtype, t.device) if isinstance(t, torch.Tensor) else type(t)
                raise ValueError("%s must be a contiguous %s tensor of shape %s on %s, not %s"
                                 % (name, dtype, shape, dev, got))

        need(ids, "ids", torch.int64, (B, FIELDS))
        need(inv, "inv", torch.int32, (FIELDS * B,))
        need(n_unique, "n_unique", torch.int32, (1,))
        if not (isinstance(bet_deep, torch.Tensor) and bet_deep.dim() == 2 and bet_deep.shape[0] <= self.rows):
            raise ValueError("bet_deep must be [rows <= %d, 64]" % self.rows)
        need(bet_deep, "bet_deep", torch.float32, (bet_deep.shape[0], DIM))
        need(bet_wide, "bet_wide", torch.float32, (bet_deep.shape[0], 1))
        if labels is not None:
            need(labels, "labels", torch.float32, (B,))
        need(flat, "params", torch.float32, (N_PARAMS,))

    def launch(self, ids, inv, n_unique, bet_deep, bet_wide, labels, flat, train=True):
        """One tower call (two kernels) on the current stream: no checks, no host read."""
        a = self.args
        a.ids, a.inv, a.n_unique = ids.data_ptr(), inv.data_ptr(), n_unique.data_ptr()
        a.bet_deep, a.bet_wide, a.params = bet_deep.data_ptr(), bet_wide.data_ptr(), flat.data_ptr()
        a.labels = labels.data_ptr() if labels is not None else None
        fn = self.lib.b200_frappe_tower if train else self.lib.b200_frappe_forward
        with torch.cuda.device(self.device):
            rc = fn(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        if rc:
            msg = self.lib.b200_frappe_last_error().decode("utf-8", "replace")
            raise (ValueError if rc == _lib.EINVAL else RuntimeError)("%s failed (%d): %s" % (fn.__name__, rc, msg))

    def outputs(self, n):
        """{loss, logits, grads, gsum_deep [n, 64], gsum_wide [n, 1]} (views of the buffers)."""
        return {"loss": self.loss.reshape(()), "logits": self.logits, "grads": self.grads,
                "gsum_deep": self.gsum_deep[:n], "gsum_wide": self.gsum_wide[:n]}


def frappe_tower(ids, inv, n_unique, bet_deep, bet_wide, labels, flat, train=True):
    """The frappe tower kernel on one batch: ids int64 [B, 10], the dedup's inv int32 [10 B] and n_unique int32
    [1], the unique rows bet_deep [U, 64] / bet_wide [U, 1], labels float32 [B] (None with train=False) and the
    flat dense buffer float32 [41089], all on one device.  Returns FrappeTowerCall.outputs(U) of fresh buffers."""
    B = ids.shape[0] if isinstance(ids, torch.Tensor) and ids.dim() == 2 else 0
    rows = bet_deep.shape[0] if isinstance(bet_deep, torch.Tensor) and bet_deep.dim() == 2 else 0
    call = FrappeTowerCall(B, flat.device if isinstance(flat, torch.Tensor) else "cuda", rows=max(rows, 1))
    call.check_inputs(ids, inv, n_unique, bet_deep, bet_wide, labels, flat)
    call.launch(ids, inv, n_unique, bet_deep, bet_wide, labels, flat, train)
    return call.outputs(rows)


class FrappeDeepFMEngine:
    """One async worker of the frappe DeepFM model on the parameter-server step.

    group: an async PSGroup without lr staleness modulation (ValueError otherwise: the captured step carries no
    pulled versions; the drop-in ParameterServerTrainer covers those modes).  input_dim=None: hashed tables sized
    for `expected_rows` distinct ids (the group's default when None); input_dim=5383: bounded ids, tables as dense
    PS parameters.  register=True registers the six parameters and sets the initial values of the dense ones
    first-writer-wins (as PushModel does); register=False attaches to a group.clone_view() of a group where
    another engine registered them, for another worker thread.
    step(ids int64 [B, 10], labels float32 [B]) runs pull_dense (into the flat buffer) -> dedup of the 10 B ids
    -> one pull_rows for both tables -> the tower -> push_begin -> push_dense -> push_rows (two segments, counts
    on the device) -> push_end, with no host read, and returns the loss on the device.  capture() / replay() run
    the same step as one CUDA graph over static inputs; a new learning rate re-captures."""

    def __init__(self, group, batch, lr, input_dim=None, seed=0, register=True, expected_rows=None):
        if not getattr(group, "use_async", True):
            raise ValueError("FrappeDeepFMEngine trains async only: a sync-SGD group needs the drop-in trainer")
        if getattr(group, "lr_staleness_modulation", False):
            raise ValueError("FrappeDeepFMEngine pushes without model versions: a group with "
                             "lr_staleness_modulation needs the drop-in trainer")
        self.B = int(batch)
        if self.B < 1:
            raise ValueError("batch size must be >= 1, not %d" % self.B)
        if input_dim is not None and int(input_dim) < 1:
            raise ValueError("input_dim must be None (hashed tables) or >= 1, not %r" % (input_dim,))
        self.input_dim = None if input_dim is None else int(input_dim)
        self.group = group if register else group.clone_view()
        g = self.group
        self.device = g.device
        self.lr = float(lr)
        tables = [(DEEP_NAME, DIM), (WIDE_NAME, 1)]
        self.owner = {n: string_to_id(n, g.n_shards) for n, _ in DENSE_PARAMS}
        if self.input_dim is not None:
            self.owner.update({n: string_to_id(n, g.n_shards) for n, _ in tables})
        if register:
            for n, dim in tables:
                if self.input_dim is None:
                    g.register_table(n, dim, "uniform", expected_rows=expected_rows)
                else:
                    g.register_dense(n, (self.input_dim, dim), self.owner[n])
            for n, s in DENSE_PARAMS:
                g.register_dense(n, s, self.owner[n])
            g.commit()
            init = flat_views(initial_dense(seed, self.device))
            if self.input_dim is not None:
                for n, dim in tables:
                    init[n] = initial_table(seed, dim, self.device, self.input_dim)
            for s in range(g.n_shards):  # first writer wins (PushModel, server.go:209-221)
                if s in g.local_shards and g.try_init(s):
                    mine = [(n, v) for n, v in init.items() if self.owner[n] == s]
                    if mine:
                        g.set_dense(mine)
                    g.finish_init(s, 0)
        self.tids = {n: g.lookup(n)[0] for n in [DEEP_NAME, WIDE_NAME] + DENSE_NAMES}  # PSNotFound if unregistered
        dev, B = self.device, self.B
        self.rows = FIELDS * B if self.input_dim is None else min(FIELDS * B, self.input_dim)
        self.flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=dev)
        self.views = flat_views(self.flat)
        self.uniq = torch.zeros(FIELDS * B, dtype=torch.int64, device=dev)
        self.inv = torch.zeros(FIELDS * B, dtype=torch.int32, device=dev)
        self.n_unique = torch.zeros(1, dtype=torch.int32, device=dev)
        self.bet_deep = torch.zeros((self.rows, DIM), dtype=torch.float32, device=dev)
        self.bet_wide = torch.zeros((self.rows, 1), dtype=torch.float32, device=dev)
        if self.input_dim is None:
            self.bounds = None
            nbytes = g.lib.b200ps_unique_workspace(1, FIELDS * B)
        else:
            self.bounds = (ctypes.c_int64 * 1)(self.input_dim)
            nbytes = g.lib.b200ps_unique_bounded_workspace(1, FIELDS * B, self.bounds)
        self.dedup_ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
        self.tower = FrappeTowerCall(B, dev, rows=self.rows)
        t = self.tower
        self.pull_dense_segs = g.make_segs([(self.tids[n], 0, None, None, self.views[n]) for n in DENSE_NAMES])
        self.pull_rows_segs = g.make_segs([
            (self.tids[DEEP_NAME], self.rows, self.uniq, self.n_unique, self.bet_deep),
            (self.tids[WIDE_NAME], self.rows, self.uniq, self.n_unique, self.bet_wide)])
        self.push_dense_segs = g.make_segs([(self.tids[n], 0, None, None, t.grads[OFFSETS[n]:OFFSETS[n] + int(np.prod(s))])
                                            for n, s in DENSE_PARAMS])
        self.push_rows_segs = g.make_segs([
            (self.tids[DEEP_NAME], self.rows, self.uniq, self.n_unique, t.gsum_deep),
            (self.tids[WIDE_NAME], self.rows, self.uniq, self.n_unique, t.gsum_wide)])
        self.zero_versions = [0] * g.n_shards
        self.graph = None
        self._graph_lr = None
        self.steps = 0

    # ------------------------------------------------------------------ inputs
    def _check_batch(self, ids, labels):
        B, dev = self.B, self.device
        checks = [(ids, "ids", torch.int64, (B, FIELDS))]
        if labels is not None:
            checks.append((labels, "labels", torch.float32, (B,)))
        for t, name, dtype, shape in checks:
            if not (isinstance(t, torch.Tensor) and t.device == dev and t.dtype == dtype and tuple(t.shape) == shape
                    and t.is_contiguous()):
                got = (tuple(t.shape), t.dtype, t.device) if isinstance(t, torch.Tensor) else type(t)
                raise ValueError("%s must be a contiguous %s tensor of shape %s on %s, not %s"
                                 % (name, dtype, shape, dev, got))

    # ------------------------------------------------------------------ the step
    def _pull(self, ids, st, mark):
        """pull_dense -> dedup of the 10 B ids -> one pull_rows for both tables on the unique ids."""
        g, lib = self.group, self.group.lib
        arr, n = self.pull_dense_segs
        check(lib.b200ps_pull_dense(g._h, arr, n, st))
        mark("pull_dense")
        k, ws = FIELDS * self.B, self.dedup_ws
        if self.bounds is None:
            check(lib.b200ps_unique(g._h, ids.data_ptr(), 1, k, self.uniq.data_ptr(), self.inv.data_ptr(),
                                    self.n_unique.data_ptr(), ws.data_ptr(), ws.numel(), st))
        else:  # an id outside [0, input_dim) is read as id 0 and makes check() raise
            check(lib.b200ps_unique_bounded(g._h, ids.data_ptr(), 1, k, self.bounds, self.uniq.data_ptr(),
                                            self.inv.data_ptr(), self.n_unique.data_ptr(), ws.data_ptr(), ws.numel(),
                                            st))
        mark("dedup")
        arr, n = self.pull_rows_segs
        check(lib.b200ps_pull_rows(g._h, arr, n, st))
        mark("pull")

    def _step(self, ids, labels, ev=None):
        g, lib = self.group, self.group.lib

        def mark(name):  # an event after each part of the step
            if ev is not None:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                ev.setdefault(name, []).append(e)

        with torch.cuda.device(self.device):
            st = g._stream()
            mark("start")
            self._pull(ids, st, mark)
            self.tower.launch(ids, self.inv, self.n_unique, self.bet_deep, self.bet_wide, labels, self.flat)
            mark("tower")
            g.push_begin(self.lr, self.zero_versions)
            arr, n = self.push_dense_segs
            check(lib.b200ps_push_dense(g._h, arr, n, st))
            arr, n = self.push_rows_segs
            check(lib.b200ps_push_rows(g._h, arr, n, st))
            g.push_end(sync=False)
            mark("push")
        return self.tower.loss.reshape(())

    def step(self, ids, labels, ev=None):
        """One training step; returns the loss (device scalar, not synchronised).  ev (optional dict): CUDA events
        recorded after pull_dense, dedup, pull, tower and push (and one at the start) on the launching stream."""
        self._check_batch(ids, labels)
        out = self._step(ids, labels, ev)
        self.steps += 1
        return out

    def predict(self, ids):
        """Logits [B] of the current parameters (pull_dense -> dedup -> pull -> the tower's forward-only
        instance); the pulled rows are not pushed.  Returns a fresh tensor, not synchronised."""
        self._check_batch(ids, None)
        with torch.cuda.device(self.device):
            self._pull(ids, self.group._stream(), lambda name: None)
            self.tower.launch(ids, self.inv, self.n_unique, self.bet_deep, self.bet_wide, None, self.flat, train=False)
        return self.tower.logits.clone()

    def evaluate(self, ids, labels, metrics):
        """The forward of predict() on one batch, then metrics.update_evaluation_metrics({"logits": logits,
        "probs": sigmoid(logits)}, labels) (an EvaluationMetrics, e.g. of eval_metrics_fn()).  Pushes nothing.
        Returns the tower's logits buffer [B] (not a copy: the next step, predict or evaluate overwrites it)."""
        self._check_batch(ids, labels)
        with torch.cuda.device(self.device):
            self._pull(ids, self.group._stream(), lambda name: None)
            self.tower.launch(ids, self.inv, self.n_unique, self.bet_deep, self.bet_wide, None, self.flat, train=False)
            logits = self.tower.logits
            metrics.update_evaluation_metrics({"logits": logits, "probs": torch.sigmoid(logits)}, labels)
        return logits

    def check(self):
        """Raise PSRangeError (a ValueError) if a step since the last check met an id outside [0, input_dim) (the
        step used row 0 for it) or a hashed table ran out of slots; synchronises the device."""
        self.group.check()

    def set_lr(self, lr):
        """The learning rate the next pushes carry; the captured graph is re-captured on the next replay."""
        self.lr = float(lr)

    # ------------------------------------------------------------------ CUDA graph
    def capture(self):
        """Capture one step over static inputs (self.s_ids, self.s_labels) into a CUDA graph on the current
        stream's device; the learning rate is baked in."""
        dev, B = self.device, self.B
        if self.graph is None:
            self.s_ids = torch.zeros((B, FIELDS), dtype=torch.int64, device=dev)
            self.s_labels = torch.zeros(B, dtype=torch.float32, device=dev)
        torch.cuda.current_stream(dev).synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._step(self.s_ids, self.s_labels)
        self.graph, self._graph_lr = graph, self.lr
        return graph

    def replay(self, ids, labels):
        """step() through the captured graph (captured now if there is none or the learning rate changed)."""
        self._check_batch(ids, labels)
        if self.graph is None or self._graph_lr != self.lr:
            self.capture()
        self.s_ids.copy_(ids)
        self.s_labels.copy_(labels)
        self.graph.replay()
        self.steps += 1
        return self.tower.loss.reshape(())


class FrappeDeepFM(torch.nn.Module):
    """The same model as a drop-in ParameterServerTrainer user writes it: two elasticdl_b200.layers.Embedding
    layers (64 and 1 wide, mask_zero=True, input_length=10) called with the features tensor itself -- so the
    trainer's batched, graphed lookup plan applies -- the mask applied from the layer's compute_mask, the FM, and
    Dense(64) -> Dense(1) as torch linear maps.  The Dense weights are held as Keras-named, Keras-shaped parameters
    (dense/kernel:0 [640, 64], ...), so the trainer registers the same PS parameters FrappeDeepFMEngine does and
    the two paths can hand state to each other."""

    def __init__(self, lr=0.1, input_dim=None, optimizer="sgd"):
        super().__init__()
        from elasticdl_b200.layers import Embedding

        self.deep = Embedding(DIM, input_dim=input_dim, embeddings_initializer="uniform", mask_zero=True,
                              input_length=FIELDS, name=DEEP_NAME.split("/")[0])
        self.wide = Embedding(1, input_dim=input_dim, embeddings_initializer="uniform", mask_zero=True,
                              input_length=FIELDS, name=WIDE_NAME.split("/")[0])
        for n, s in DENSE_PARAMS:
            self.register_parameter(n, torch.nn.Parameter(torch.zeros(s)))
        self.load_mlp(initial_dense(0, "cpu"))
        opt = torch.optim.SGD if optimizer == "sgd" else torch.optim.Adam
        self.optimizer = opt([p for n, p in self.named_parameters() if n in DENSE_NAMES], lr=lr)
        bce = torch.nn.BCEWithLogitsLoss()
        self.loss = lambda labels, logits: bce(logits, labels)

    def load_mlp(self, flat):
        """Copy a flat dense buffer (include/b200_frappe.h layout) into the Dense parameters."""
        v = flat_views(flat)
        with torch.no_grad():
            for n in DENSE_NAMES:
                getattr(self, n).copy_(v[n])

    def tower(self, e, w, mask):
        """Rows e [B, 10, 64], w [B, 10, 1] and the mask [B, 10] -> logits [B]."""
        m = mask.unsqueeze(2).to(e.dtype)
        e = e * m
        w = w * m
        first = w.sum((1, 2))
        S = e.sum(1)
        second = 0.5 * (S * S - (e * e).sum(1)).sum(1)
        x = e.reshape(e.shape[0], FIELDS * DIM)  # Flatten: f-major
        h = torch.nn.functional.linear(x, getattr(self, "dense/kernel:0").t(), getattr(self, "dense/bias:0"))
        deep = torch.nn.functional.linear(h, getattr(self, "dense_1/kernel:0").t(), getattr(self, "dense_1/bias:0"))
        return first + second + deep[:, 0]

    def forward(self, features):
        return self.tower(self.deep(features), self.wide(features), self.deep.compute_mask(features))
