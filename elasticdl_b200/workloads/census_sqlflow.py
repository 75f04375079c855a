"""The census_model_sqlflow wide & deep models (model_zoo/census_model_sqlflow/wide_and_deep/, five files, one
model) trained on the parameter-server step: raw rows -> the fused feature-id transform of the model's id rule
(census_sqlflow_features) -> the census_sqlflow tower (csrc/census_sqlflow_tower.cu) -> push.

Per group, SparseEmbedding(combiner="mean") / embedding_column averages the rows of the ids that are present; a
group with none pools to zero.  Wide: groups 1 and 2, dim 1; deep: groups 1..3, dim 8; Dense 24 -> 16 -> 8 -> 4
with no activation; logit = the sum of the wide outputs and h3; the mean sigmoid cross-entropy.

MODELS lists the five files: the id rule each uses and whether its DNN input is the tf.reshape of the list of the
three deep embeddings (quirk Q11) or their concatenation.  Parameter names (param_names()), in the flat order of
include/b200_census_sqlflow.h, are the reference's variable names as Keras and the feature columns create them;
they are recalled from TF's naming rules (a layer without a name gets its snake-cased class name, uniquified by a
running count in creation order; embedding_column's weight is <DenseFeatures layer>/<column name>_embedding/
embedding_weights, the column name of concatenated_categorical_column being its sorted inputs' names joined by
"_C_", feature_column.py:141-147) and not verified here.  Every table is under 2 MB, so the reference keeps it a
dense parameter; here each is one dense PS parameter whose batch rows are pushed with b200ps_push_rows.
"""
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib
from elasticdl_b200._lib import CsqlArgs, check
from elasticdl_b200.common.hash_utils import string_to_id
from elasticdl_b200.workloads.async_engine import AsyncEngine, check_tensor
from elasticdl_b200.workloads.census_sqlflow_features import GROUP_DIMS, STRING_WIDTH, transform, _check_variant

# model file -> (id rule, reference_reshape)
MODELS = {
    "wide_deep_functional_keras": ("keras", True),                  # :65 tf.reshape(deep_embeddings, (-1, 24))
    "wide_deep_functional_tensor_interface_keras": ("keras", False),  # :233 ConcatenateWithOffset(offsets=None)
    "wide_deep_subclass_keras": ("keras", False),                   # :177 ConcatenateWithOffset(offsets=None)
    "wide_deep_functional_fc": ("fc", True),                        # :76 tf.reshape(deep_embeddings, (-1, 24))
    "wide_deep_functional_tensor_interface_fc": ("fc", False),      # :255 one DenseFeatures (Q26)
}
SHAPES = [(24, 16), (16,), (16, 8), (8,), (8, 4), (4,), (27, 1), (73, 1), (27, 8), (73, 8), (113, 8)]
MLP_NAMES = ["dense/kernel:0", "dense/bias:0", "dense_1/kernel:0", "dense_1/bias:0", "dense_2/kernel:0",
             "dense_2/bias:0"]
# the concatenated columns' names: their inputs' names (a bucketized column is <key>_bucketized), sorted
FC_COLUMNS = ("capital_gain_bucketized_C_capital_loss_bucketized_C_hours_per_week_bucketized_C_workclass",
              "education_C_marital_status_C_occupation_C_relationship",
              "age_bucketized_C_native_country_C_race_C_sex")
# the five tables' names (wide group 1, wide group 2, deep groups 1..3), recalled as the module docstring says; "fc"
# holds wide_deep_functional_fc's five DenseFeatures layers (the tensor-interface file has two)
TABLE_NAMES = {
    "keras": ["sparse_embedding/embeddings:0"] + ["sparse_embedding_%d/embeddings:0" % i for i in range(1, 5)],
    "fc": ["dense_features%s/%s_embedding/embedding_weights:0" % ("_%d" % k if k else "", FC_COLUMNS[g])
           for k, g in enumerate((0, 1, 0, 1, 2))],
}
TABLE_GROUP = (0, 1, 0, 1, 2)
TABLE_DIM = (1, 1, 8, 8, 8)
N_PARAMS, N_MLP = 2376, 572
UNIQ_OFF = (0, 27, 100, 127, 200)
N_UNIQ = 313
GSUM_OFF = (0, 27, 100, 316, 900)
N_GSUM = 1804
TILE = 256  # B200_CSQL_TILE
OFFSETS = [int(v) for v in np.cumsum([0] + [int(np.prod(s)) for s in SHAPES])[:-1]]
assert OFFSETS[6] == N_MLP and sum(int(np.prod(s)) for s in SHAPES) == N_PARAMS
assert tuple(o - N_MLP for o in OFFSETS[6:]) == GSUM_OFF


def model_of(model):
    """(variant, reference_reshape) of a MODELS name."""
    if model not in MODELS:
        raise ValueError("unknown model %r: one of %s" % (model, sorted(MODELS)))
    return MODELS[model]


def param_names(variant):
    """The eleven parameter names of `variant` in flat order."""
    _check_variant(variant)
    return MLP_NAMES + TABLE_NAMES[variant]


def flat_views(flat):
    """The [shape] views of a flat buffer in flat order: all eleven of the parameters, the MLP's six of its
    572-float gradient."""
    return [flat[o:o + int(np.prod(s))].view(s) for o, s in zip(OFFSETS, SHAPES) if o + int(np.prod(s)) <= flat.numel()]


def initial_params(seed, device):
    """The reference's initialisers: "uniform" embeddings U(-0.05, 0.05) (SparseEmbedding's default), glorot-uniform
    Dense kernels, zero biases.  float32 [2376]."""
    gen = torch.Generator(device=device).manual_seed(int(seed))
    flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=device)
    for i, v in enumerate(flat_views(flat)):
        if i >= 6:
            v.copy_((torch.rand(v.shape, generator=gen, device=device) * 2 - 1) * 0.05)
        elif i % 2 == 0:
            lim = float(np.sqrt(6.0 / (v.shape[0] + v.shape[1])))
            v.copy_((torch.rand(v.shape, generator=gen, device=device) * 2 - 1) * lim)
    return flat


def optimizer():
    """The zoo's optimizer, Adam(learning_rate=0.001) (wide_deep_functional_keras.py:263-264), as the PS's
    (optimizer type, argument string, lr)."""
    return ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", 1e-3)


def eval_metrics_fn():
    """wide_deep_functional_keras.py:267-276: accuracy of the LOGITS thresholded at 0.5 (quirk Q12, as in the
    census model) and the AUC of the probabilities."""
    from elasticdl_b200.common.evaluation_utils import zoo_eval_metrics

    return zoo_eval_metrics(0.5)


def callbacks():
    """wide_deep_functional_keras.py:279-288: 3e-4 below version 5000, 2e-4 below 12000, then 1e-4, as a
    declarative schedule the push evaluates on the device; versions are integers, so `< 5000` is `<= 4999`."""
    from elasticdl_b200.callbacks import LearningRateScheduler, PiecewiseConstantDecay

    return [LearningRateScheduler(PiecewiseConstantDecay([4999, 11999], [3e-4, 2e-4, 1e-4]))]


class CsqlTowerCall:
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
        self.grads = torch.zeros(N_MLP, **f32)
        self.uniq = torch.zeros(N_UNIQ, dtype=torch.int64, device=self.device)
        self.n_unique = torch.zeros(5, dtype=torch.int32, device=self.device)
        self.gsum = torch.zeros(N_GSUM, **f32)
        self.error = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            nbytes = self.lib.b200_csql_workspace_bytes(self.B)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        a = CsqlArgs()
        a.B = self.B
        a.loss, a.logits, a.grads = self.loss.data_ptr(), self.logits.data_ptr(), self.grads.data_ptr()
        a.uniq, a.n_unique, a.gsum = self.uniq.data_ptr(), self.n_unique.data_ptr(), self.gsum.data_ptr()
        a.error, a.workspace, a.workspace_bytes = self.error.data_ptr(), self.workspace.data_ptr(), nbytes
        self.args = a

    def check_inputs(self, ids, labels, flat):
        check_tensor(ids, "ids", torch.int32, (12, self.B), self.device)
        if labels is not None:
            check_tensor(labels, "labels", torch.float32, (self.B,), self.device)
        check_tensor(flat, "params", torch.float32, (N_PARAMS,), self.device)

    def launch(self, ids, labels, flat, reference_reshape, train=True):
        """One tower launch (train=False: the forward form, logits only) on the current stream (no checks, no host
        read)."""
        a = self.args
        a.ids, a.params = ids.data_ptr(), flat.data_ptr()
        a.labels = labels.data_ptr() if labels is not None else None
        a.reference_reshape = 1 if reference_reshape else 0
        fn = self.lib.b200_csql_tower if train else self.lib.b200_csql_forward
        with torch.cuda.device(self.device):
            rc = fn(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        _lib.check_call(rc, fn.__name__, self.lib.b200_csql_last_error)

    def check_error(self):
        """Raise PSRangeError (a ValueError) if a launch since the last check read an id outside [-1, rows of its
        group), and clear the count.  Reads one int from the device."""
        n = int(self.error.item())
        if n:
            self.error.zero_()
            raise _lib.PSRangeError(_lib.ERANGE, "%d census_sqlflow ids outside [-1, rows of their group) %s were "
                                                 "read as absent" % (n, GROUP_DIMS))

    def outputs(self):
        """{loss, logits, grads, uniq [5], n_unique [5], gsum [5 segments: [rows, dim]]} (views of the buffers)."""
        out = {"loss": self.loss.reshape(()), "logits": self.logits, "grads": self.grads, "n_unique": self.n_unique,
               "uniq": [], "gsum": []}
        for t in range(5):
            rows = GROUP_DIMS[TABLE_GROUP[t]]
            out["uniq"].append(self.uniq[UNIQ_OFF[t]:UNIQ_OFF[t] + rows])
            out["gsum"].append(self.gsum[GSUM_OFF[t]:GSUM_OFF[t] + rows * TABLE_DIM[t]].view(rows, TABLE_DIM[t]))
        return out


def census_sqlflow_tower(ids, labels, flat, reference_reshape=False, train=True):
    """The tower kernel on one batch: ids int32 [12, B] (-1 = absent), labels float32 [B] (None with train=False),
    flat float32 [2376], all on one device.  Synchronises, raises ValueError for ids outside [-1, rows) (after the
    launch, which read them as absent), and returns CsqlTowerCall.outputs() of fresh buffers."""
    B = ids.shape[1] if isinstance(ids, torch.Tensor) and ids.dim() == 2 else 0
    call = CsqlTowerCall(B, flat.device if isinstance(flat, torch.Tensor) else "cuda")
    call.check_inputs(ids, labels, flat)
    call.launch(ids, labels, flat, reference_reshape, train)
    call.check_error()
    return call.outputs()


class CensusSqlflowEngine(AsyncEngine):
    """One async worker of a census_model_sqlflow wide & deep model on the parameter-server step.

    group: an async PSGroup, as AsyncEngine takes it.  model: a MODELS name, which sets the id rule and the reshape
    mode.  register=True registers the eleven parameters under the model's names and sets their initial values
    first-writer-wins (as PushModel does); register=False attaches to a group.clone_view() of a group where
    another engine registered them, for another worker thread.
    step(numeric float32 [4, B], strings uint8 [8, B, 32], labels float32 [B]) runs pull_dense (into the flat
    buffer) -> the feature transform -> the tower -> push_begin -> push_dense (MLP) -> push_rows (the five tables'
    touched rows, counts on the device) -> push_end, with no host read, and returns the loss on the device.
    capture() / replay() run the same step as one CUDA graph over static inputs.  lr_schedule: a schedule to
    install, as AsyncEngine.set_lr_schedule does (callbacks()[0].schedule is the zoo's)."""

    def __init__(self, group, model, batch, lr, seed=0, register=True, lr_schedule=None):
        self.variant, self.reference_reshape = model_of(model)
        super().__init__(group, batch, lr, register, lr_schedule)
        g, B = self.group, self.B
        self.inputs = [("numeric", torch.float32, (4, B)), ("strings", torch.uint8, (8, B, STRING_WIDTH)),
                       ("labels", torch.float32, (B,))]
        self.names = param_names(self.variant)
        self.owner = {n: string_to_id(n, g.n_shards) for n in self.names}
        if register:
            for n, s in zip(self.names, SHAPES):
                g.register_dense(n, s, self.owner[n])
            g.commit()
            g.init_dense(zip(self.names, flat_views(initial_params(seed, self.device))))
        tids = [g.lookup(n)[0] for n in self.names]  # PSNotFound when no engine registered them
        self.flat = torch.zeros(N_PARAMS, dtype=torch.float32, device=self.device)
        views = flat_views(self.flat)
        self.ids = torch.zeros((12, B), dtype=torch.int32, device=self.device)
        self.transform = transform(self.variant, device=self.device)
        self.tower = t = CsqlTowerCall(B, self.device)
        self.pull_segs = g.make_segs([(tid, 0, None, None, v) for tid, v in zip(tids, views)])
        self.push_dense_segs = g.make_segs([(tids[i], 0, None, None, v) for i, v in enumerate(flat_views(t.grads))])
        out = t.outputs()
        self.push_rows_segs = g.make_segs([(tids[6 + k], GROUP_DIMS[TABLE_GROUP[k]], out["uniq"][k],
                                            t.n_unique[k:k + 1], out["gsum"][k]) for k in range(5)])
        self._eval_tower = None  # evaluate()'s logits buffer (lazy)

    def _pull(self, numeric, strings, st):
        check(self.group.lib.b200ps_pull_dense(self.group._h, *self.pull_segs, st))
        self.transform(numeric, strings, ids_out=self.ids)

    def _step(self, numeric, strings, labels):
        with torch.cuda.device(self.device):
            st = self.group._stream()
            self._pull(numeric, strings, st)
            self.tower.launch(self.ids, labels, self.flat, self.reference_reshape)
            self._push(st)
        return self.tower.loss.reshape(())

    def step(self, numeric, strings, labels):
        """One training step from raw rows; returns the loss (device scalar, not synchronised)."""
        self._check_batch(numeric, strings, labels)
        out = self._step(numeric, strings, labels)
        self.steps += 1
        return out

    def evaluate(self, numeric, strings, labels, metrics):
        """The forward only: pull_dense -> the transform -> the tower's forward form -> metrics.update_evaluation_
        metrics({"logits": logits, "probs": sigmoid(logits)}, labels) (an EvaluationMetrics, e.g. of
        eval_metrics_fn()).  Pushes nothing.  Returns the logits [B] on the device (overwritten by the next
        evaluate)."""
        self._check_batch(numeric, strings, labels)
        if self._eval_tower is None:
            self._eval_tower = CsqlTowerCall(self.B, self.device)
        with torch.cuda.device(self.device):
            self._pull(numeric, strings, self.group._stream())
            self._eval_tower.launch(self.ids, None, self.flat, self.reference_reshape, train=False)
            logits = self._eval_tower.logits
            metrics.update_evaluation_metrics({"logits": logits, "probs": torch.sigmoid(logits)}, labels)
        return logits

    def check(self):
        """Raise PSRangeError (a ValueError) if a step or evaluate since the last check read an id outside its
        group (read as absent); one device read per tower."""
        if self._eval_tower is not None:
            self._eval_tower.check_error()
        self.tower.check_error()


def sparse_group_ids(ids, g):
    """Group g's four id rows of ids [12, B] as the SparseTensor [B, 4] the reference's SparseEmbedding takes: a
    COO tensor holding every cell, absent ones as -1 (safe_embedding_lookup_sparse prunes them)."""
    B = ids.shape[1]
    rows = torch.arange(B, device=ids.device).repeat_interleave(4)
    cols = torch.arange(4, device=ids.device).repeat(B)
    vals = ids[4 * g:4 * g + 4].t().reshape(-1).to(torch.int64)
    return torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, (B, 4))


class CensusSqlflowWideDeep(torch.nn.Module):
    """The same model as a torch module for the drop-in ParameterServerTrainer: the tables are
    elasticdl_b200.layers.Embedding layers with combiner="mean" over sparse ids (row-sparse PS tables under the
    model's names; safe_embedding_lookup_sparse prunes the absent ids and zeroes an empty group), the MLP is three
    torch Linear layers.  forward((numeric, strings)) runs the model's feature transform."""

    def __init__(self, model, lr, optimizer="sgd"):
        super().__init__()
        from elasticdl_b200.layers import Embedding

        self.variant, self.reference_reshape = model_of(model)
        tables = []
        for n, g, d in zip(TABLE_NAMES[self.variant], TABLE_GROUP, TABLE_DIM):
            e = Embedding(d, input_dim=GROUP_DIMS[g], embeddings_initializer="uniform", combiner="mean",
                          name=n.rsplit("/", 1)[0])
            e.set_embedding_weight_name(n)
            tables.append(e)
        self.wide = torch.nn.ModuleList(tables[:2])
        self.deep = torch.nn.ModuleList(tables[2:])
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
                lin.weight.copy_(v[2 * i].t())
                lin.bias.copy_(v[2 * i + 1])

    def forward(self, features):
        numeric, strings = features
        if self.transform is None:
            self.transform = transform(self.variant, device=numeric.device)
        ids, _ = self.transform(numeric, strings)
        sp = [sparse_group_ids(ids, g) for g in range(3)]
        wide = self.wide[0](sp[0])[:, 0] + self.wide[1](sp[1])[:, 0]
        deep = torch.stack([self.deep[g](sp[g]) for g in range(3)])  # [3, B, 8]
        B = deep.shape[1]
        x = deep.reshape(B, 24) if self.reference_reshape else deep.permute(1, 0, 2).reshape(B, 24)
        for lin in self.dense:
            x = lin(x)
        return wide + x.sum(1)
