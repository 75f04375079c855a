"""deepctr's DeepFMEstimator (model_zoo/deepctr/deepfm_estimator.py) trained on the parameter-server step: raw
Criteo-shaped rows -> categorical_column_with_hash_bucket(C<j>, 1000) of C1..C26, "" dropped (b200feat_transform,
id -1) -> the deepctr DeepFM tower (csrc/deepctr_deepfm_tower.cu) -> push_dense to two groups: the dnn scope (26
embedding tables, the 117-256-128-64 DNN and its logit kernel) on TF1 Adagrad(0.01), the linear scope (26 hashed
weight columns, 13 numeric weights, bias_weights) on TF1 Ftrl(0.005), as deepctr's two minimize calls do.

The model: DeepFMEstimator(linear, dnn, task="binary") over embedding_column(hash_bucket(C<j>, 1000), 4) and
numeric_column(I<i>) for the DNN and FM, and hash_bucket(C<j>, 1000) and numeric_column(I<i>) for the linear model;
the TF1 head's loss is the batch sum of sigmoid_cross_entropy on the logits plus the regularisation loss,
1e-5 l2_loss of each looked-up embedding and of every linear variable but bias_weights.  batch_size = 64.

deepctr is third-party and unpinned.  Its defaults, TF1's initialisers and optimizer defaults, and the variable names
below are RECALLED, not read from their source (DESIGN.md section 4, Q31-Q35).
"""
import csv
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib
from elasticdl_b200._lib import DeepctrDeepfmArgs, check
from elasticdl_b200.common.hash_utils import string_to_id
from elasticdl_b200.workloads.async_engine import AsyncEngine, check_tensor, truncated_normal

FIELDS, DENSE, ROWS, DIM = 26, 13, 1000, 4   # B200_DEEPCTR_DEEPFM_FIELDS, _DENSE, _ROWS, _DIM
F = FIELDS * DIM + DENSE                     # 117
HIDDEN = (256, 128, 64)                      # dnn_hidden_units
TILE = 64                                    # B200_DEEPCTR_DEEPFM_TILE
STRING_WIDTH = 8                             # Criteo hex ids
L2_REG = 1e-5                                # l2_reg_embedding = l2_reg_linear
BATCH_SIZE = 64                              # deepfm_estimator.py's batch_size
ADAGRAD_LR, FTRL_LR = 0.01, 0.005

# the 73 parameters in flat order (RECALLED TF1-style names): the dnn group, then the linear group
EMB_NAMES = ["dnn/input_from_feature_columns/C%d_embedding/embedding_weights:0" % j for j in range(1, FIELDS + 1)]
DNN_PARAMS = [("dnn/dnn/kernel0:0", (F, HIDDEN[0])), ("dnn/dnn/bias0:0", (HIDDEN[0],)),
              ("dnn/dnn/kernel1:0", (HIDDEN[0], HIDDEN[1])), ("dnn/dnn/bias1:0", (HIDDEN[1],)),
              ("dnn/dnn/kernel2:0", (HIDDEN[1], HIDDEN[2])), ("dnn/dnn/bias2:0", (HIDDEN[2],)),
              ("dnn/dense/kernel:0", (HIDDEN[2], 1))]
LIN_NAMES = ["linear/linear_model/C%d/weights:0" % j for j in range(1, FIELDS + 1)]
NUM_NAMES = ["linear/linear_model/I%d/weights:0" % i for i in range(1, DENSE + 1)]
BIAS_NAME = "linear/linear_model/bias_weights:0"
DNN_GROUP = [(n, (ROWS, DIM)) for n in EMB_NAMES] + DNN_PARAMS
LINEAR_GROUP = [(n, (ROWS, 1)) for n in LIN_NAMES] + [(n, (1, 1)) for n in NUM_NAMES] + [(BIAS_NAME, (1,))]
PARAMS = DNN_GROUP + LINEAR_GROUP
NAMES = [n for n, _ in PARAMS]
DNN_NAMES = [n for n, _ in DNN_GROUP]
LINEAR_NAMES = [n for n, _ in LINEAR_GROUP]
N_PARAMS, N_DNN_GROUP = 201438, 175424  # B200_DEEPCTR_DEEPFM_PARAMS, _DNN_FLOATS


def _offsets():
    out, o = {}, 0
    for n, s in PARAMS:
        out[n] = o
        o += int(np.prod(s))
    assert len(PARAMS) == 73 and o == N_PARAMS and out[LIN_NAMES[0]] == N_DNN_GROUP
    return out


OFFSETS = _offsets()


def flat_views(flat):
    """{name: view of the flat buffer in the parameter's shape}."""
    return {n: flat[OFFSETS[n]:OFFSETS[n] + int(np.prod(s))].view(s) for n, s in PARAMS}


def initial_params(seed, device):
    """The recalled initialisers: embedding tables truncated_normal(stddev = 1/sqrt(4)) (embedding_column's
    default), DNN and logit kernels glorot_normal (Keras' truncated normal of stddev sqrt(2 / (in + out))), biases
    and the whole linear model zero (linear_model's zeros).  float32 [201438]."""
    gen = torch.Generator(device=device).manual_seed(int(seed))
    flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=device)
    for n, v in flat_views(flat).items():
        if n in EMB_NAMES:
            v.copy_(truncated_normal(v.shape, 1.0 / np.sqrt(DIM), gen, device))
        elif n.startswith("dnn/") and "kernel" in n:
            v.copy_(truncated_normal(v.shape, float(np.sqrt(2.0 / (v.shape[0] + v.shape[1]))) / 0.87962566103423978,
                                     gen, device))
    return flat


def optimizers():
    """deepctr's defaults as PS (type, argument string) pairs: (linear, dnn) = (Ftrl(0.005) with
    initial_accumulator_value 0.1 and no l1 / l2 / shrinkage, Adagrad(0.01) with no epsilon).  TF1's Adagrad
    starts its accumulator at 0.1: DeepctrDeepfmEngine writes that when it registers the dnn group."""
    return (("Ftrl", "learning_rate=%g;initial_accumulator_value=0.1;l1_regularization_strength=0.0;"
                     "l2_regularization_strength=0.0;l2_shrinkage_regularization_strength=0.0;beta=0.0;" % FTRL_LR),
            ("Adagrad", "learning_rate=%g;epsilon=0.0;" % ADAGRAD_LR))


def eval_metrics_fn():
    """deepctr's binary head metrics: AUC (200 thresholds) and prediction/mean of p, LogLoss (the unweighted mean
    cross-entropy) of the logits, label/mean.  The engine's evaluate feeds {"logits", "probs"}."""
    from elasticdl_b200.common.evaluation_utils import AUC

    def logloss(labels, logits):
        return logits.clamp(min=0) - logits * labels + torch.log1p(torch.exp(-logits.abs()))

    def prediction_mean(labels, probs):
        return probs

    def label_mean(labels, probs):
        return labels

    return {"probs": {"AUC": AUC(), "prediction/mean": prediction_mean, "label/mean": label_mean},
            "logits": {"LogLoss": logloss}}


def transform(device=None):
    """FeatureTransform: categorical_column_with_hash_bucket(C<j>, 1000) of the 26 string columns (Fingerprint64 %
    1000, as tf.strings.to_hash_bucket_fast; an empty cell is dropped: id -1) -> ids int32 [26, B]."""
    from elasticdl_b200.preprocessing.layers import FeatureTransform

    return FeatureTransform([{"kind": "hash", "column": j, "num_bins": ROWS, "absent": True} for j in range(FIELDS)],
                            (), torch.int32, device=device)


def read_criteo_csv(path):
    """deepfm_estimator.py's read_csv: skip the header row; label int, I1..I13 float (an empty cell 0), C1..C26
    strings.  Returns (dense float32 [13, N], strings uint8 [26, N, 8] (zero-padded; "" all zeros), labels float32
    [N]) on the CPU.  ValueError for a string longer than 8 bytes or a row without 40 cells."""
    labels, dense, strings = [], [], []
    with open(path, newline="") as fh:
        for i, row in enumerate(csv.reader(fh)):
            if i == 0:
                continue
            if len(row) != 1 + DENSE + FIELDS:
                raise ValueError("row %d has %d cells, not %d" % (i, len(row), 1 + DENSE + FIELDS))
            labels.append(int(row[0]))
            dense.append([float(v) if v else 0.0 for v in row[1:1 + DENSE]])
            cells = [v.encode() for v in row[1 + DENSE:]]
            if any(len(c) > STRING_WIDTH for c in cells):
                raise ValueError("row %d: a string cell is longer than %d bytes" % (i, STRING_WIDTH))
            strings.append([c.ljust(STRING_WIDTH, b"\0") for c in cells])
    n = len(labels)
    s = np.frombuffer(b"".join(b"".join(r) for r in strings), dtype=np.uint8).reshape(n, FIELDS, STRING_WIDTH)
    return (torch.tensor(dense, dtype=torch.float32).reshape(n, DENSE).t().contiguous(),
            torch.from_numpy(s.transpose(1, 0, 2).copy()), torch.tensor(labels, dtype=torch.float32))


def synthetic_batch(B, seed, device, empty_fraction=None):
    """Criteo-shaped raw rows from dac_ctr_features.synthetic_raw_batch: dense float32 [13, B] (its integer
    counts as float32), strings uint8 [26, B, 8] (about 3 % empty, or a fraction `empty_fraction` emptied), labels
    float32 [B] (about 25 % positive)."""
    from elasticdl_b200.workloads.dac_ctr_features import synthetic_raw_batch

    numeric, strings, _ = synthetic_raw_batch(B, seed, device)
    if empty_fraction is not None:
        g = torch.Generator(device=strings.device).manual_seed(int(seed) + 11)
        drop = torch.rand(strings.shape[:2], generator=g, device=strings.device) < empty_fraction
        strings = strings.masked_fill(drop.unsqueeze(2), 0)
    g = torch.Generator(device=strings.device).manual_seed(int(seed) + 13)
    labels = (torch.rand(B, generator=g, device=strings.device) < 0.25).float()
    return numeric.float().contiguous(), strings.contiguous(), labels


class DeepctrDeepfmCall:
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
            nbytes = self.lib.b200_deepctr_deepfm_workspace_bytes(self.B)
        if not nbytes:
            raise ValueError("batch size must be in [1, 4194304], not %d" % self.B)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        a = DeepctrDeepfmArgs()
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
        fn = self.lib.b200_deepctr_deepfm_tower if train else self.lib.b200_deepctr_deepfm_forward
        with torch.cuda.device(self.device):
            rc = fn(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        _lib.check_call(rc, fn.__name__, self.lib.b200_deepctr_deepfm_last_error)

    def check_error(self):
        """Raise PSRangeError (a ValueError) if a launch since the last check read an id outside [-1, 1000), and
        clear the count.  Reads one int from the device."""
        n = int(self.error.item())
        if n:
            self.error.zero_()
            raise _lib.PSRangeError(_lib.ERANGE, "%d deepctr DeepFM ids outside [-1, 1000) were read as absent" % n)

    def outputs(self):
        return {"loss": self.loss.reshape(()), "logits": self.logits, "grads": self.grads}


def deepctr_deepfm_tower(ids, dense, labels, flat, train=True):
    """The tower on one batch: ids int32 [26, B] (-1 absent), dense float32 [13, B], labels float32 [B] (None with
    train=False), flat float32 [201438], all on one device.  Raises ValueError for ids outside [-1, 1000) (after the
    launch, which read them as absent).  Returns DeepctrDeepfmCall.outputs() of fresh buffers."""
    B = dense.shape[1] if isinstance(dense, torch.Tensor) and dense.dim() == 2 else 0
    call = DeepctrDeepfmCall(B, flat.device if isinstance(flat, torch.Tensor) else "cuda")
    call.check_inputs(ids, dense, labels, flat)
    call.launch(ids, dense, labels, flat, train)
    call.check_error()
    return call.outputs()


class DeepctrDeepfmEngine(AsyncEngine):
    """One async worker of deepctr's DeepFMEstimator on the parameter-server step, over two groups: `dnn_group`
    (Adagrad in the model: the 26 embedding tables, the DNN and its logit kernel) and `linear_group` (Ftrl: the
    linear model's 40 variables); optimizers() gives both.

    register=True registers each group's dense parameters, each on shard string_to_id(name, N) of its group, sets
    their initial values, initial_params(seed), first-writer-wins (as PushModel does), and on an Adagrad dnn group
    sets the accumulators to TF1's initial 0.1 (the PS starts them at 0).  register=False attaches to clone_view()s
    of groups where another engine registered them, for another worker thread.  step(dense float32 [13, B], strings
    uint8 [26, B, 8], labels float32 [B]) runs pull_dense (all 73 parameters into the flat buffer) -> hash -> the
    tower -> for each group push_begin -> push_dense of its gradients -> push_end, with no host read, and returns
    the summed loss on the device.  capture() / replay() run the same step as one CUDA graph.  Learning rates are
    per group (set_lr); a device learning-rate schedule is not supported."""

    def __init__(self, dnn_group, linear_group, batch, seed=0, register=True, dnn_lr=ADAGRAD_LR,
                 linear_lr=FTRL_LR):
        self._check_group(linear_group)
        super().__init__(dnn_group, batch, dnn_lr, register)
        self.linear_group = linear_group if register else linear_group.clone_view()
        if self.linear_group.device != self.device:
            raise ValueError("the dnn and linear groups are on %s and %s" % (self.device, self.linear_group.device))
        self.linear_lr = float(linear_lr)
        self.linear_zero_versions = [0] * self.linear_group.n_shards
        dev, B = self.device, self.B
        self.inputs = [("dense", torch.float32, (DENSE, B)), ("strings", torch.uint8, (FIELDS, B, STRING_WIDTH)),
                       ("labels", torch.float32, (B,))]
        groups = ((self.group, DNN_GROUP), (self.linear_group, LINEAR_GROUP))
        self.owner = {n: string_to_id(n, g.n_shards) for g, params in groups for n, _ in params}
        if register:
            init = flat_views(initial_params(seed, dev))
            for g, params in groups:
                for n, s in params:
                    g.register_dense(n, s, self.owner[n])
                g.commit()
                g.init_dense([(n, init[n]) for n, _ in params])
            if self.group.opt_type == "Adagrad":
                for n, s in DNN_GROUP:
                    self.group.slot_dense(n, 1, torch.full(s, 0.1, device=dev))
        self.flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=dev)
        self.views = flat_views(self.flat)
        self.ids = torch.zeros((FIELDS, B), dtype=torch.int32, device=dev)
        self.transform = transform(dev)
        self.tower = t = DeepctrDeepfmCall(B, dev)
        grads = flat_views(t.grads)
        self.segs = []  # (group, pull segments, push segments), the dnn group first
        for g, params in groups:
            tids = {n: g.lookup(n)[0] for n, _ in params}  # PSNotFound when no engine registered them
            self.segs.append((g, g.make_segs([(tids[n], 0, None, None, self.views[n]) for n, _ in params]),
                              g.make_segs([(tids[n], 0, None, None, grads[n]) for n, _ in params])))
        self._eval_tower = None

    def set_lr(self, dnn_lr, linear_lr=None):
        """The learning rates the next pushes carry (linear_lr None keeps the linear group's); the captured graph is
        re-captured on the next replay."""
        self.lr = float(dnn_lr)
        if linear_lr is not None:
            self.linear_lr = float(linear_lr)

    def set_lr_schedule(self, schedule):
        raise ValueError("DeepctrDeepfmEngine pushes to two groups with their own learning rates: a device "
                         "learning-rate schedule is not supported")

    def _graph_key(self):
        return (self.lr, self.linear_lr)

    def _push(self, st):
        """For each group: push_begin -> push_dense (every parameter, whole) -> push_end."""
        for (g, _, push), lr, versions in zip(self.segs, (self.lr, self.linear_lr),
                                              (self.zero_versions, self.linear_zero_versions)):
            g.push_begin(lr, versions)
            check(g.lib.b200ps_push_dense(g._h, *push, st))
            g.push_end(sync=False)

    def _pull(self, dense, strings, st):
        for g, pull, _ in self.segs:
            check(g.lib.b200ps_pull_dense(g._h, *pull, st))
        self.transform(dense, strings, ids_out=self.ids)

    def _step(self, dense, strings, labels):
        with torch.cuda.device(self.device):
            st = self.group._stream()
            self._pull(dense, strings, st)
            self.tower.launch(self.ids, dense, labels, self.flat)
            self._push(st)
        return self.tower.loss.reshape(())

    def evaluate(self, dense, strings, labels, metrics):
        """The forward only: pull_dense -> hash -> the tower's forward form -> metrics.update_evaluation_metrics(
        {"logits": logits, "probs": sigmoid(logits)}, labels) (an EvaluationMetrics, e.g. of eval_metrics_fn()).
        Pushes nothing.  Returns the logits [B] on the device (overwritten by the next evaluate)."""
        self._check_batch(dense, strings, labels)
        if self._eval_tower is None:
            self._eval_tower = DeepctrDeepfmCall(self.B, self.device)
        t = self._eval_tower
        with torch.cuda.device(self.device):
            self._pull(dense, strings, self.group._stream())
            t.launch(self.ids, dense, None, self.flat, train=False)
            metrics.update_evaluation_metrics({"logits": t.logits, "probs": torch.sigmoid(t.logits)}, labels)
        return t.logits

    def check(self):
        """Raise PSRangeError (a ValueError) if a step or evaluate since the last check read an id outside
        [-1, 1000); one device read per tower.  Hashed ids are always in range, so this guards the buffers."""
        if self._eval_tower is not None:
            self._eval_tower.check_error()
        self.tower.check_error()
