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
import numpy as np
import torch

from elasticdl_b200._lib import CsqlArgs
from elasticdl_b200.workloads.census import TABLE_DIM, TABLE_GROUP, TowerCall, TowerSpec, WideDeepEngine, WideDeepTwin
from elasticdl_b200.workloads.census_sqlflow_features import GROUP_DIMS, transform, _check_variant

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


SPEC = TowerSpec("b200_csql", CsqlArgs, GROUP_DIMS, UNIQ_OFF, N_UNIQ, GSUM_OFF, N_GSUM, N_PARAMS, N_MLP,
                 "census_sqlflow ids outside [-1, rows of their group) %s were read as absent" % (GROUP_DIMS,), True)


class CsqlTowerCall(TowerCall):
    """The tower's output buffers and workspace for batch B on `device`, and one launch over them."""

    spec = SPEC


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


class CensusSqlflowEngine(WideDeepEngine):
    """One async worker of a census_model_sqlflow wide & deep model on the parameter-server step (census.
    WideDeepEngine), from raw rows through the feature transform of the model's id rule.

    group: an async PSGroup, as AsyncEngine takes it.  model: a MODELS name, which sets the id rule and the reshape
    mode.  register=True registers the eleven parameters under the model's names and sets their initial values
    first-writer-wins (as PushModel does); register=False attaches to a group.clone_view() of a group where
    another engine registered them, for another worker thread.  lr_schedule: a schedule to install, as
    AsyncEngine.set_lr_schedule does (callbacks()[0].schedule is the zoo's).  evaluate() runs the tower's forward
    form."""

    def __init__(self, group, model, batch, lr, seed=0, register=True, lr_schedule=None):
        self.variant, self.reference_reshape = model_of(model)
        super().__init__(group, batch, lr, register, lr_schedule)
        self._setup(param_names(self.variant), SHAPES, initial_params, seed,
                    transform(self.variant, device=self.device), CsqlTowerCall, register)


def sparse_group_ids(ids, g):
    """Group g's four id rows of ids [12, B] as the SparseTensor [B, 4] the reference's SparseEmbedding takes: a
    COO tensor holding every cell, absent ones as -1 (safe_embedding_lookup_sparse prunes them)."""
    B = ids.shape[1]
    rows = torch.arange(B, device=ids.device).repeat_interleave(4)
    cols = torch.arange(4, device=ids.device).repeat(B)
    vals = ids[4 * g:4 * g + 4].t().reshape(-1).to(torch.int64)
    return torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, (B, 4))


class CensusSqlflowWideDeep(WideDeepTwin):
    """The same model as a torch module for the drop-in ParameterServerTrainer: the tables are
    elasticdl_b200.layers.Embedding layers with combiner="mean" over sparse ids (row-sparse PS tables under the
    model's names; safe_embedding_lookup_sparse prunes the absent ids and zeroes an empty group), the MLP is three
    torch Linear layers.  forward((numeric, strings)) runs the model's feature transform."""

    def __init__(self, model, lr, optimizer="sgd"):
        from elasticdl_b200.layers import Embedding

        variant, reference_reshape = model_of(model)
        tables = []
        for n, g, d in zip(TABLE_NAMES[variant], TABLE_GROUP, TABLE_DIM):
            e = Embedding(d, input_dim=GROUP_DIMS[g], embeddings_initializer="uniform", combiner="mean",
                          name=n.rsplit("/", 1)[0])
            e.set_embedding_weight_name(n)
            tables.append(e)
        super().__init__(tables[:2], tables[2:], lr, reference_reshape, optimizer)
        self.variant = variant

    def forward(self, features):
        numeric, strings = features
        if self.transform is None:
            self.transform = transform(self.variant, device=numeric.device)
        ids, _ = self.transform(numeric, strings)
        sp = [sparse_group_ids(ids, g) for g in range(3)]
        wide = torch.stack([self.wide[g](sp[g])[:, 0] for g in range(2)])
        deep = torch.stack([self.deep[g](sp[g]) for g in range(3)])  # [3, B, 8]
        return self.tower(wide, deep)
