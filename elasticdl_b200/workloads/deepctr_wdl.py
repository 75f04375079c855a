"""deepctr's WDL model (model_zoo/deepctr/wdl.py:19-75) trained on the parameter-server step: raw Criteo-shaped
rows -> Hash(10000) of C1..C26 (b200feat_transform) -> the deepctr WDL tower (csrc/deepctr_wdl_tower.cu) ->
push_dense of all 61 parameters.

The model: WDL(fixlen, fixlen, task="binary") over 26 SparseFeat("C<j>", vocabulary_size=10000, embedding_dim=4,
use_hash=True) and 13 DenseFeat("I<i>", 1); the loss is the batch mean of Keras binary_crossentropy on p plus the
tables' and the linear kernel's l2(1e-5) (the reference trainer adds model.losses, worker/ps_trainer.py:397-398);
Adam(learning_rate=0.001).  Every table is under 2 MB, so the reference keeps it an ordinary Keras variable
(common/model_handler.py:98-102) whose gradient, the lookup's IndexedSlices plus the dense 2 lambda W, TF
aggregates into a dense tensor: the PS updates every row of every table at every step (DESIGN.md section 4, Q28).

deepctr is third-party and unpinned (model_zoo/requirements.txt).  The names, shapes, initialisers and
regularizers below are RECALLED from deepctr's source, not read from it (Q27).
"""
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib
from elasticdl_b200._lib import DeepctrWdlArgs, check
from elasticdl_b200.common.hash_utils import string_to_id
from elasticdl_b200.workloads.async_engine import AsyncEngine, check_tensor

FIELDS, DENSE, ROWS, DIM = 26, 13, 10000, 4   # B200_DEEPCTR_WDL_FIELDS, _DENSE, _ROWS, _DIM
F = FIELDS * DIM + DENSE                      # 117
HIDDEN = (256, 128, 64)                       # dnn_hidden_units (before deepctr 0.9: (128, 128), not built)
TILE = 64                                     # B200_DEEPCTR_WDL_TILE
STRING_WIDTH = 8                              # Criteo hex ids
L2_REG = 1e-5                                 # l2_reg_embedding = l2_reg_linear

# the 61 parameters in flat order (RECALLED names): the deep tables, the linear tables, then the dense block
DEEP_NAMES = ["sparse_emb_C%d/embeddings:0" % j for j in range(1, FIELDS + 1)]
LINEAR_NAMES = ["linear0sparse_emb_C%d/embeddings:0" % j for j in range(1, FIELDS + 1)]
DNN_PARAMS = [("linear/linear_kernel:0", (DENSE, 1)),
              ("dnn/kernel0:0", (F, HIDDEN[0])), ("dnn/bias0:0", (HIDDEN[0],)),
              ("dnn/kernel1:0", (HIDDEN[0], HIDDEN[1])), ("dnn/bias1:0", (HIDDEN[1],)),
              ("dnn/kernel2:0", (HIDDEN[1], HIDDEN[2])), ("dnn/bias2:0", (HIDDEN[2],)),
              ("dense/kernel:0", (HIDDEN[2], 1)), ("prediction_layer/global_bias:0", (1,))]
PARAMS = ([(n, (ROWS, DIM)) for n in DEEP_NAMES] + [(n, (ROWS, 1)) for n in LINEAR_NAMES] + DNN_PARAMS)
NAMES = [n for n, _ in PARAMS]
N_PARAMS, N_TABLES = 1371438, 1300000  # B200_DEEPCTR_WDL_PARAMS; floats of the 52 tables
ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", 1e-3)


def _offsets():
    out, o = {}, 0
    for n, s in PARAMS:
        out[n] = o
        o += int(np.prod(s))
    assert len(PARAMS) == 61 and o == N_PARAMS and out["linear/linear_kernel:0"] == N_TABLES
    return out


OFFSETS = _offsets()


def flat_views(flat):
    """{name: view of the flat buffer in the parameter's shape}."""
    return {n: flat[OFFSETS[n]:OFFSETS[n] + int(np.prod(s))].view(s) for n, s in PARAMS}


def initial_params(seed, device):
    """The recalled initialisers: deep tables N(0, 1e-4) (deepctr's init_std 1e-4), linear tables zero
    (get_linear_logit replaces the initializer with Zeros), kernels glorot_normal (a normal of stddev
    sqrt(2 / (in + out)) truncated at two stddevs), biases zero.  float32 [1371438]."""
    gen = torch.Generator(device=device).manual_seed(int(seed))
    flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=device)
    for n, v in flat_views(flat).items():
        if n in DEEP_NAMES:
            v.copy_(torch.randn(v.shape, generator=gen, device=device) * 1e-4)
        elif "kernel" in n:
            std = float(np.sqrt(2.0 / (v.shape[0] + v.shape[1]))) / 0.87962566103423978  # keras truncated-normal
            x = torch.randn(v.shape, generator=gen, device=device)
            while True:
                bad = x.abs() > 2
                if not bool(bad.any()):
                    break
                x[bad] = torch.randn(int(bad.sum()), generator=gen, device=device)
            v.copy_(x * std)
    return flat


def optimizer():
    """The zoo's optimizer, Adam(learning_rate=0.001), as (PS type, argument string, lr)."""
    return ADAM


def eval_metrics_fn():
    """{"probs": {"auc": AUC}} (model_zoo/deepctr/wdl.py: {"auc": AUC()} over the model's output p)."""
    from elasticdl_b200.common.evaluation_utils import AUC

    return {"probs": {"auc": AUC()}}


def transform(device=None):
    """FeatureTransform: Hash(10000) of the 26 string columns (tf.strings.to_hash_bucket_fast, "" an ordinary
    bucket: Q30) -> ids int32 [26, B]; the 13 dense columns pass through untouched."""
    from elasticdl_b200.preprocessing.layers import FeatureTransform

    return FeatureTransform([{"kind": "hash", "column": j, "num_bins": ROWS} for j in range(FIELDS)], (),
                            torch.int32, device=device)


def synthetic_batch(B, seed, device, empty_fraction=None):
    """Criteo-shaped raw rows from dac_ctr_features.synthetic_raw_batch: dense float32 [13, B] (its integer
    counts as float32, wdl.py parses I* as float32), strings uint8 [26, B, 8] (about 3 % empty, or a fraction
    `empty_fraction` emptied), labels float32 [B] (about 25 % positive)."""
    from elasticdl_b200.workloads.dac_ctr_features import synthetic_raw_batch

    numeric, strings, _ = synthetic_raw_batch(B, seed, device)
    if empty_fraction is not None:
        g = torch.Generator(device=strings.device).manual_seed(int(seed) + 11)
        drop = torch.rand(strings.shape[:2], generator=g, device=strings.device) < empty_fraction
        strings = strings.masked_fill(drop.unsqueeze(2), 0)
    g = torch.Generator(device=strings.device).manual_seed(int(seed) + 13)
    labels = (torch.rand(B, generator=g, device=strings.device) < 0.25).float()
    return numeric.float().contiguous(), strings.contiguous(), labels


class DeepctrWdlCall:
    """The tower's output buffers and workspace for batch B on `device`, and one launch over them."""

    def __init__(self, B, device):
        self.B = int(B)
        if self.B < 1:
            raise ValueError("batch size must be >= 1, not %d" % self.B)
        self.device = torch.device(device)
        self.lib = _lib.lib()
        f32 = dict(dtype=torch.float32, device=self.device)
        self.loss = torch.zeros(1, **f32)
        self.logits = torch.zeros(self.B, **f32)
        self.grads = torch.zeros(N_PARAMS, **f32)
        self.error = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            nbytes = self.lib.b200_deepctr_wdl_workspace_bytes(self.B)
        if not nbytes:
            raise ValueError("batch size must be in [1, 4194304], not %d" % self.B)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        a = DeepctrWdlArgs()
        a.B = self.B
        a.loss, a.logits, a.grads = self.loss.data_ptr(), self.logits.data_ptr(), self.grads.data_ptr()
        a.error, a.workspace, a.workspace_bytes = self.error.data_ptr(), self.workspace.data_ptr(), nbytes
        self.args = a

    def check_inputs(self, ids, dense, labels, flat):
        """labels may be None (the forward)."""
        check_tensor(ids, "ids", torch.int32, (FIELDS, self.B), self.device)
        check_tensor(dense, "dense", torch.float32, (DENSE, self.B), self.device)
        if labels is not None:
            check_tensor(labels, "labels", torch.float32, (self.B,), self.device)
        check_tensor(flat, "params", torch.float32, (N_PARAMS,), self.device)

    def launch(self, ids, dense, labels, flat, train=True):
        """One training call (train=False: the forward, logits only) on the current stream (no checks, no host
        read)."""
        a = self.args
        a.ids, a.dense, a.params = ids.data_ptr(), dense.data_ptr(), flat.data_ptr()
        a.labels = labels.data_ptr() if labels is not None else None
        fn = self.lib.b200_deepctr_wdl_tower if train else self.lib.b200_deepctr_wdl_forward
        with torch.cuda.device(self.device):
            rc = fn(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        _lib.check_call(rc, fn.__name__, self.lib.b200_deepctr_wdl_last_error)

    def check_error(self):
        """Raise PSRangeError (a ValueError) if a launch since the last check read an id outside [0, 10000), and
        clear the count.  Reads one int from the device."""
        n = int(self.error.item())
        if n:
            self.error.zero_()
            raise _lib.PSRangeError(_lib.ERANGE, "%d deepctr WDL ids outside [0, 10000) were read as row 0" % n)

    def outputs(self):
        return {"loss": self.loss.reshape(()), "logits": self.logits, "grads": self.grads}


def deepctr_wdl_tower(ids, dense, labels, flat, train=True):
    """The tower on one batch: ids int32 [26, B], dense float32 [13, B], labels float32 [B] (None with
    train=False), flat float32 [1371438], all on one device.  Raises ValueError for ids outside [0, 10000) (after
    the launch, which read them as row 0).  Returns DeepctrWdlCall.outputs() of fresh buffers."""
    B = dense.shape[1] if isinstance(dense, torch.Tensor) and dense.dim() == 2 else 0
    call = DeepctrWdlCall(B, flat.device if isinstance(flat, torch.Tensor) else "cuda")
    call.check_inputs(ids, dense, labels, flat)
    call.launch(ids, dense, labels, flat, train)
    call.check_error()
    return call.outputs()


class DeepctrWdlEngine(AsyncEngine):
    """One async worker of deepctr's WDL on the parameter-server step.

    group: an async PSGroup, as AsyncEngine takes it.  register=True registers the 61 dense parameters, each on
    shard string_to_id(name, N), and sets their initial values, initial_params(seed), first-writer-wins (as
    PushModel does); register=False attaches to a group.clone_view() of a group where another engine registered
    them, for another worker thread.  step(dense float32 [13, B], strings uint8 [26, B, 8], labels float32 [B])
    runs pull_dense (all 61 parameters into the flat buffer) -> Hash(10000) -> the tower -> push_begin ->
    push_dense of all 61 gradients -> push_end, with no host read, and returns the loss on the device.
    capture() / replay() run the same step as one CUDA graph; lr_schedule: as AsyncEngine takes it."""

    def __init__(self, group, batch, lr, seed=0, register=True, lr_schedule=None):
        super().__init__(group, batch, lr, register, lr_schedule)
        g, dev, B = self.group, self.device, self.B
        self.inputs = [("dense", torch.float32, (DENSE, B)), ("strings", torch.uint8, (FIELDS, B, STRING_WIDTH)),
                       ("labels", torch.float32, (B,))]
        self.owner = {n: string_to_id(n, g.n_shards) for n in NAMES}
        if register:
            for n, s in PARAMS:
                g.register_dense(n, s, self.owner[n])
            g.commit()
            g.init_dense(flat_views(initial_params(seed, dev)).items())
        tids = {n: g.lookup(n)[0] for n in NAMES}  # PSNotFound when no engine registered them
        self.flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=dev)
        self.views = flat_views(self.flat)
        self.ids = torch.zeros((FIELDS, B), dtype=torch.int32, device=dev)
        self.transform = transform(dev)
        self.tower = t = DeepctrWdlCall(B, dev)
        grads = flat_views(t.grads)
        self.pull_segs = g.make_segs([(tids[n], 0, None, None, self.views[n]) for n in NAMES])
        self.push_dense_segs = g.make_segs([(tids[n], 0, None, None, grads[n]) for n in NAMES])
        self._eval_tower = None

    def _push(self, st):
        """push_begin -> push_dense (every parameter, whole) -> push_end: no push_rows."""
        g = self.group
        g.push_begin(self.lr, self.zero_versions)
        check(g.lib.b200ps_push_dense(g._h, *self.push_dense_segs, st))
        g.push_end(sync=False)

    def _pull(self, dense, strings, st):
        check(self.group.lib.b200ps_pull_dense(self.group._h, *self.pull_segs, st))
        self.transform(dense, strings, ids_out=self.ids)

    def _step(self, dense, strings, labels):
        with torch.cuda.device(self.device):
            st = self.group._stream()
            self._pull(dense, strings, st)
            self.tower.launch(self.ids, dense, labels, self.flat)
            self._push(st)
        return self.tower.loss.reshape(())

    def evaluate(self, dense, strings, labels, metrics):
        """The forward only: pull_dense -> Hash -> the tower's forward form -> metrics.update_evaluation_metrics(
        {"logits": logits, "probs": sigmoid(logits)}, labels) (an EvaluationMetrics, e.g. of eval_metrics_fn()).
        Pushes nothing.  Returns the logits [B] on the device (overwritten by the next evaluate)."""
        self._check_batch(dense, strings, labels)
        if self._eval_tower is None:
            self._eval_tower = DeepctrWdlCall(self.B, self.device)
        t = self._eval_tower
        with torch.cuda.device(self.device):
            self._pull(dense, strings, self.group._stream())
            t.launch(self.ids, dense, None, self.flat, train=False)
            metrics.update_evaluation_metrics({"logits": t.logits, "probs": torch.sigmoid(t.logits)}, labels)
        return t.logits

    def check(self):
        """Raise PSRangeError (a ValueError) if a step or evaluate since the last check read an id outside
        [0, 10000); one device read per tower.  Hash ids are always in range, so this guards the buffers."""
        if self._eval_tower is not None:
            self._eval_tower.check_error()
        self.tower.check_error()


def keras_bce_mean(labels, p):
    """tf.keras.losses.binary_crossentropy on probabilities, batch mean (DESIGN.md section 4, Q19): clip to
    [1e-7, 1 - 1e-7] (no gradient where the clip is active), -(y log(p + 1e-7) + (1 - y) log(1 - p + 1e-7))."""
    eps = float(np.float32(1e-7))
    pc = torch.clamp(p, eps, float(np.float32(1.0) - np.float32(eps)))
    return (-(labels * torch.log(pc + eps) + (1.0 - labels) * torch.log(1.0 - pc + eps))).mean()


class DeepctrWdl(torch.nn.Module):
    """The same model as a torch module for the drop-in ParameterServerTrainer.  Its 52 tables are plain
    torch.nn.Embedding parameters, so the trainer pulls and pushes them whole, as the reference does with Keras
    variables under 2 MB (Q29).  forward({"ids": int64 [26, B], "dense": float32 [13, B]}) returns p [B]; loss is
    the clipped BCE mean plus regularization()."""

    def __init__(self, lr=None, optimizer="adam"):
        super().__init__()
        self.deep = torch.nn.ModuleList([torch.nn.Embedding(ROWS, DIM) for _ in range(FIELDS)])
        self.linear = torch.nn.ModuleList([torch.nn.Embedding(ROWS, 1) for _ in range(FIELDS)])
        self.dnn_params = torch.nn.ParameterList([torch.nn.Parameter(torch.zeros(s)) for _, s in DNN_PARAMS])
        self.load_flat(initial_params(0, "cpu"))
        lr = ADAM[2] if lr is None else lr
        opt = torch.optim.Adam if optimizer == "adam" else torch.optim.SGD
        self.optimizer = opt(self.parameters(), lr=lr)
        self.loss = lambda labels, p: keras_bce_mean(labels, p) + self.regularization()

    def ordered(self):
        """The parameters in the flat order of PARAMS."""
        return [e.weight for e in self.deep] + [e.weight for e in self.linear] + list(self.dnn_params)

    def load_flat(self, flat):
        with torch.no_grad():
            for p, (n, _) in zip(self.ordered(), PARAMS):
                p.copy_(flat_views(flat)[n])

    def regularization(self):
        """1e-5 (sum of the tables' squares + |w_lin|^2): the l2 regularizers of every table and the linear
        kernel, over whole tables."""
        s = sum((e.weight * e.weight).sum() for e in self.deep) + sum((e.weight * e.weight).sum() for e in self.linear)
        w = self.dnn_params[0]
        return L2_REG * (s + (w * w).sum())

    def forward(self, features):
        ids, dense = features["ids"], features["dense"]
        x = torch.cat([self.deep[j](ids[j]) for j in range(FIELDS)] + [dense.t()], 1)
        wl, W0, b0, W1, b1, W2, b2, wd, gb = self.dnn_params
        h = torch.relu(x @ W0 + b0)
        h = torch.relu(h @ W1 + b1)
        h = torch.relu(h @ W2 + b2)
        lin = sum(self.linear[j](ids[j])[:, 0] for j in range(FIELDS)) + (dense.t() @ wl)[:, 0]
        return torch.sigmoid((h @ wd)[:, 0] + lin + gb)
