"""The model zoo's embedding-column DNNs on the parameter-server step: census_dnn_model
(model_zoo/census_dnn_model/census_functional_api.py:19-55 with census_feature_columns.py:19-62),
heart_functional_api (model_zoo/heart_functional_api/heart_functional_api.py:19-96) and census_model_sqlflow's
DNNClassifier (model_zoo/census_model_sqlflow/dnn/census_functional.py:28-70 with census_feature_column.py:35-67).

All three are raw columns -> DenseFeatures -> Dense(16, relu) -> Dense(16, relu) -> Dense(1, sigmoid).
DenseFeatures holds numeric_column (pass-through), bucketized_column (a left-closed one-hot) and an embedding_column
over categorical_column_with_hash_bucket.  Where the column is ElasticDL's (feature_column/feature_column.py:24-221:
census_dnn_model, heart), the trainer registers it as a PS embedding table named
dense_features/<key>_embedding/embedding_weights:0 with the "uniform" initializer whatever the column's own
initializer is (worker/ps_trainer.py:76-92, 200-211), so its rows are created when first pulled.  Where it is
TF's (census_model_sqlflow), the PS strategy swaps it for ElasticDL's only above 2 MB
(common/model_handler.py:98-127): a smaller table stays a Keras variable of that name, a dense PS parameter the
worker initialises, updated by the Indexed kernels on the batch's rows only (Q36).  One layout table per model says
where each column sits in x and which kind each table is; the tower kernel (csrc/fc_dnn_tower.cu) reads the same
rows and writes the same row gradients for both kinds.

The step: pull_dense (the MLP) -> FeatureTransform (FarmHash buckets, Discretization) -> empty strings to the fill
id 0 -> per-table dedup -> one pull_rows of the batch's unique rows -> the tower -> push_dense + push_rows ->
push_end.  Quirks Q16-Q20 and Q36 of DESIGN.md section 4 are what the layouts reproduce.
"""
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib
from elasticdl_b200._lib import FcDnnArgs, FcLayout, check
from elasticdl_b200.common.hash_utils import string_to_id
from elasticdl_b200.workloads.async_engine import AsyncEngine, check_tensor, truncated_normal
from elasticdl_b200.workloads.census_features import STRING_WIDTH, synthetic_raw_batch

NUMERIC, BUCKET, EMBEDDING = 0, 1, 2  # B200_FC_NUMERIC, B200_FC_BUCKET, B200_FC_EMBEDDING
PS_TABLE, DENSE_TABLE = "ps", "dense"  # a table's kind: a hashed PS embedding table, or a dense PS parameter
HIDDEN = 16
TILE = 64  # B200_FC_DNN_TILE


def mlp_shapes(F):
    """The Dense layers' parameters in the flat order of include/b200_fc_dnn.h (Keras [in, out] kernels)."""
    return [("dense/kernel:0", (F, HIDDEN)), ("dense/bias:0", (HIDDEN,)), ("dense_1/kernel:0", (HIDDEN, HIDDEN)),
            ("dense_1/bias:0", (HIDDEN,)), ("dense_2/kernel:0", (HIDDEN, 1)), ("dense_2/bias:0", (1,))]


MLP_NAMES = [n for n, _ in mlp_shapes(1)]


def table_name(key):
    """feature_column.py:81-91: the column is <key>_embedding, its DenseFeatures layer dense_features."""
    return "dense_features/%s_embedding/embedding_weights:0" % key


class Layout:
    """One model's DenseFeatures layout.

    numeric_keys / string_keys: the order of the rows of the numeric float32 [n, B] and strings uint8 [m, B, 32]
    inputs.  tables: [(key, hash buckets, dim)], table k hashing string column string_keys.index(key).  buckets:
    [(key, boundaries)], Discretization of a numeric column.  columns: DenseFeatures' concatenation order, as
    [(column name, kind, key)] -- quirk Q17: sorted by column name, recalled from TF's feature_column_v2 and not
    verified here.  loss_mean: True = the gradients are batch means, False = batch sums (Q16).  table_kinds: per
    table, PS_TABLE (default: a hashed PS table with "uniform" rows created when pulled) or DENSE_TABLE (a dense
    [rows, dim] PS parameter initialised from TF's embedding_column default, truncated_normal(0, 1/sqrt(dim)),
    first writer wins, and updated on the pushed rows only: Q36)."""

    def __init__(self, name, numeric_keys, string_keys, tables, buckets, columns, loss_mean, optimizer,
                 table_kinds=None):
        self.name = name
        self.numeric_keys, self.string_keys = tuple(numeric_keys), tuple(string_keys)
        self.tables, self.buckets, self.columns = list(tables), list(buckets), list(columns)
        self.loss_mean = bool(loss_mean)
        self.optimizer = optimizer  # (PS optimizer type, its argument string, lr) of the model zoo entry
        self.table_names = [table_name(k) for k, _, _ in self.tables]
        self.table_kinds = list(table_kinds) if table_kinds is not None else [PS_TABLE] * len(self.tables)
        if len(self.table_kinds) != len(self.tables) or not set(self.table_kinds) <= {PS_TABLE, DENSE_TABLE}:
            raise ValueError("table_kinds must give %r or %r for each of the %d tables, not %r"
                             % (PS_TABLE, DENSE_TABLE, len(self.tables), table_kinds))
        blocks, off = [], 0
        for _, kind, key in self.columns:
            if kind == NUMERIC:
                src, width = self.numeric_keys.index(key), 1
            elif kind == BUCKET:
                i = [k for k, _ in self.buckets].index(key)
                src, width = len(self.tables) + i, len(self.buckets[i][1]) + 1
            else:
                src = [k for k, _, _ in self.tables].index(key)
                width = self.tables[src][2]
            blocks.append((kind, src, width, off))
            off += width
        self.blocks, self.F = blocks, off
        self.mlp = mlp_shapes(self.F)
        self.n_mlp = HIDDEN * self.F + 305
        self.xoff = {src: o for kind, src, _, o in blocks if kind == EMBEDDING}
        self.row_off = np.cumsum([0] + [r * d for _, r, d in self.tables]).tolist()
        self.c = self._c_layout()

    def spec(self):
        """The layout as plain data (oracle/fc_dnn_oracle.py takes it)."""
        return {"F": self.F, "blocks": list(self.blocks), "tables": [(r, d) for _, r, d in self.tables],
                "loss_mean": self.loss_mean, "table_kinds": list(self.table_kinds)}

    def _c_layout(self):
        c = FcLayout()
        c.F, c.n_blocks, c.n_tables, c.loss_mean = self.F, len(self.blocks), len(self.tables), int(self.loss_mean)
        for k, (key, rows, dim) in enumerate(self.tables):
            c.table_rows[k], c.table_dim[k], c.table_string[k] = rows, dim, self.string_keys.index(key)
        for i, (kind, src, width, off) in enumerate(self.blocks):
            c.blocks[i].kind, c.blocks[i].src, c.blocks[i].width, c.blocks[i].offset = kind, src, width, off
        return c

    def groups(self):
        """The FeatureTransform specs: the tables' hash groups (ids rows 0 .. T-1), then the bucket groups."""
        out = [{"kind": "hash", "column": self.string_keys.index(k), "num_bins": r} for k, r, _ in self.tables]
        out += [{"kind": "discretize", "column": self.numeric_keys.index(k), "bins": [float(v) for v in b]}
                for k, b in self.buckets]
        return out

    def transform(self, device=None):
        """FeatureTransform of groups(): ids int32 [T + n_buckets, B]."""
        from elasticdl_b200.preprocessing.layers import FeatureTransform

        return FeatureTransform(self.groups(), (), torch.int32, device=device)

    def flat_views(self, flat):
        out, o = {}, 0
        for n, s in self.mlp:
            k = int(np.prod(s))
            out[n] = flat[o:o + k].view(s)
            o += k
        return out

    def initial_mlp(self, seed, device):
        """Glorot-uniform kernels U(-sqrt(6 / (in + out)), +), zero biases: float32 [16 F + 305]."""
        gen = torch.Generator(device=device).manual_seed(int(seed))
        flat = torch.zeros(self.n_mlp, dtype=torch.float32, device=device)
        for n, v in self.flat_views(flat).items():
            if n.endswith("kernel:0"):
                lim = float(np.sqrt(6.0 / (v.shape[0] + v.shape[1])))
                v.copy_((torch.rand(v.shape, generator=gen, device=device) * 2 - 1) * lim)
        return flat

    def initial_tables(self, seed):
        """The DENSE_TABLE tables' initial values, {name: float32 [rows, dim] on the CPU}: TF's embedding_column
        default truncated_normal(mean 0, stddev 1/sqrt(dim)), draws outside two stddevs redrawn, from one CPU
        generator seeded `seed` and drawn in table order (the same values on every device)."""
        gen = torch.Generator().manual_seed(int(seed))
        return {n: truncated_normal((r, d), 1.0 / np.sqrt(d), gen, "cpu")
                for n, kind, (_, r, d) in zip(self.table_names, self.table_kinds, self.tables) if kind == DENSE_TABLE}


CENSUS_CATEGORICAL = ["workclass", "education", "marital-status", "occupation", "relationship", "race", "sex",
                      "native-country"]
CENSUS_NUMERIC = ["age", "capital-gain", "capital-loss", "hours-per-week"]
# census_feature_columns.py:40-57; loss census_functional_api.py:33-35 (per-sample, never reduced: Q16);
# optimizer census_functional_api.py:38-39 (Adam() defaults)
CENSUS_DNN = Layout(
    "census_dnn_model", CENSUS_NUMERIC, CENSUS_CATEGORICAL,
    tables=[(k, 64, 16) for k in CENSUS_CATEGORICAL], buckets=[],
    columns=[("age", NUMERIC, "age"), ("capital-gain", NUMERIC, "capital-gain"),
             ("capital-loss", NUMERIC, "capital-loss"), ("education_embedding", EMBEDDING, "education"),
             ("hours-per-week", NUMERIC, "hours-per-week"),
             ("marital-status_embedding", EMBEDDING, "marital-status"),
             ("native-country_embedding", EMBEDDING, "native-country"),
             ("occupation_embedding", EMBEDDING, "occupation"), ("race_embedding", EMBEDDING, "race"),
             ("relationship_embedding", EMBEDDING, "relationship"), ("sex_embedding", EMBEDDING, "sex"),
             ("workclass_embedding", EMBEDDING, "workclass")],
    loss_mean=False,
    optimizer=("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", 1e-3))
HEART_NUMERIC = ["age", "trestbps", "chol", "thalach", "oldpeak", "slope", "ca"]
HEART_AGE_BOUNDARIES = [18, 25, 30, 35, 40, 45, 50, 55, 60, 65]
# heart_functional_api.py:22-42; loss :60-63 (both reshaped to [-1]: a batch mean, Q16); optimizer :66-67
HEART = Layout(
    "heart_functional_api", HEART_NUMERIC, ["thal"],
    tables=[("thal", 100, 8)], buckets=[("age", HEART_AGE_BOUNDARIES)],
    columns=[("age_bucketized", BUCKET, "age"), ("ca", NUMERIC, "ca"), ("chol", NUMERIC, "chol"),
             ("oldpeak", NUMERIC, "oldpeak"), ("slope", NUMERIC, "slope"), ("thal_embedding", EMBEDDING, "thal"),
             ("thalach", NUMERIC, "thalach"), ("trestbps", NUMERIC, "trestbps")],
    loss_mean=True,
    optimizer=("SGD", "learning_rate=1e-06;momentum=0.0;nesterov=false;", 1e-6))
# census_model_sqlflow/dnn: census_feature_column.py:35-53, TF's embedding_column(categorical_column_with_hash_bucket(
# key, 64), dimension=16) after the four numeric_columns, so the same DenseFeatures as census_dnn_model; loss
# census_functional.py:51-53 (binary_crossentropy(expand_dims(labels, 1), p): per-sample, never reduced, Q16);
# optimizer :56-57 (Adam() defaults).  Its 64 x 16 tables (4 KB) stay Keras variables under the PS strategy (Q36).
CENSUS_SQLFLOW_DNN = Layout(
    "census_model_sqlflow_dnn", CENSUS_NUMERIC, CENSUS_CATEGORICAL,
    tables=[(k, 64, 16) for k in CENSUS_CATEGORICAL], buckets=[], columns=CENSUS_DNN.columns,
    loss_mean=False, optimizer=CENSUS_DNN.optimizer, table_kinds=[DENSE_TABLE] * len(CENSUS_CATEGORICAL))
LAYOUTS = {"census_dnn_model": CENSUS_DNN, "heart_functional_api": HEART,
           "census_model_sqlflow_dnn": CENSUS_SQLFLOW_DNN}
for _l in LAYOUTS.values():
    assert [c for c, _, _ in _l.columns] == sorted(c for c, _, _ in _l.columns)  # Q17
assert (CENSUS_DNN.F, CENSUS_DNN.n_mlp, HEART.F, HEART.n_mlp) == (132, 2417, 25, 705)
assert (CENSUS_SQLFLOW_DNN.F, CENSUS_SQLFLOW_DNN.n_mlp) == (132, 2417)


def layout_of(model):
    if isinstance(model, Layout):
        return model
    if model not in LAYOUTS:
        raise ValueError("unknown model %r: one of %s" % (model, sorted(LAYOUTS)))
    return LAYOUTS[model]


def synthetic_census_batch(B, seed, device, empty_fraction=0.05):
    """synthetic_raw_batch's Adult-shaped raw rows, with a fraction `empty_fraction` of every string column
    emptied: numeric float32 [4, B], strings uint8 [8, B, 32]."""
    numeric, strings, _, _ = synthetic_raw_batch(B, seed, device)
    if empty_fraction > 0:
        g = torch.Generator(device=strings.device).manual_seed(int(seed) + 7)
        drop = torch.rand(strings.shape[:2], generator=g, device=strings.device) < empty_fraction
        strings = strings.masked_fill(drop.unsqueeze(2), 0)
    return numeric, strings.contiguous()


def synthetic_heart_batch(B, seed, device, empty_fraction=0.05):
    """Heart-disease-shaped raw rows: numeric float32 [7, B] (HEART_NUMERIC order, integral values in the UCI
    data's ranges; oldpeak in tenths), strings uint8 [1, B, 32] (thal: "normal", "fixed", "reversible", a few
    others and about `empty_fraction` empty), labels float32 [B] (about 27 % positive)."""
    rng = np.random.RandomState(seed)
    num = np.stack([rng.randint(29, 78, B), rng.randint(94, 201, B), rng.randint(126, 565, B),
                    rng.randint(71, 203, B), rng.randint(0, 63, B) / 10.0, rng.randint(0, 3, B),
                    rng.randint(0, 4, B)]).astype(np.float32)
    k = min(len(HEART_AGE_BOUNDARIES), B)
    num[0, rng.choice(B, k, replace=False)] = HEART_AGE_BOUNDARIES[:k]  # the left-closed edges
    pool = np.array(["normal", "fixed", "reversible", "1", "2", ""], dtype=object)
    p = np.array([0.5, 0.1, 0.3, 0.05, 0.05 - min(empty_fraction, 0.05), min(empty_fraction, 0.05)])
    thal = pool[rng.choice(len(pool), B, p=p / p.sum())]
    from elasticdl_b200.preprocessing.layers import encode_strings

    strings = encode_strings([[str(v) for v in thal]], STRING_WIDTH, device="cpu")
    labels = (rng.rand(B) < 0.27).astype(np.float32)
    return (torch.from_numpy(num).to(device), strings.to(device).contiguous(), torch.from_numpy(labels).to(device))


def eval_metrics_fn(model):
    """The model's eval_metrics_fn as an EvaluationMetrics dict over the outputs {"logits", "probs"}.
    census_dnn_model (census_functional_api.py:42-48) and census_model_sqlflow_dnn (census_functional.py:60-66):
    accuracy of round(p) against the int label; tf.round rounds half to even, so round(p) = 1 iff p > 0.5 iff the
    logit > 0.  heart_functional_api (heart_functional_api.py:89-96): argmax of
    the [B, 1] output over axis 1 is always 0, so its "accuracy" is the share of label-0 samples (Q20)."""
    from elasticdl_b200.common.evaluation_utils import zoo_eval_metrics

    if layout_of(model) in (CENSUS_DNN, CENSUS_SQLFLOW_DNN):
        return {"logits": {"accuracy": zoo_eval_metrics(0.0)["logits"]["accuracy"]}}

    def heart_accuracy(labels, predictions):
        return torch.zeros_like(predictions.reshape(-1), dtype=torch.int32) == labels.reshape(-1).int()

    return {"logits": {"accuracy": heart_accuracy}}


def fill_empty(layout, ids, strings):
    """Rows 0 .. T-1 of ids int32 [G, B] (the tables' hash buckets) := 0 where the table's string is empty, in
    place (Q18): the string column drops "" and safe_embedding_lookup_sparse looks the empty row up as id 0."""
    lib = _lib.lib()
    B = ids.shape[1]
    with torch.cuda.device(ids.device):
        rc = lib.b200_fc_dnn_fill_empty(ctypes.byref(layout.c), ctypes.c_void_p(ids.data_ptr()),
                                        ctypes.c_void_p(strings.data_ptr()), B, strings.shape[2],
                                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    _lib.check_call(rc, "b200_fc_dnn_fill_empty", lib.b200_fc_dnn_last_error)
    return ids


class FcDnnTowerCall:
    """The tower's output buffers and workspace for one layout and batch B on `device`, and one launch over
    them."""

    def __init__(self, layout, B, device):
        self.layout = layout_of(layout)
        self.B = int(B)
        if self.B < 1:
            raise ValueError("batch size must be >= 1, not %d" % self.B)
        self.device = torch.device(device)
        self.lib = _lib.lib()
        L = self.layout
        f32 = dict(dtype=torch.float32, device=self.device)
        self.loss = torch.zeros(1, **f32)
        self.logits = torch.zeros(self.B, **f32)
        self.grads = torch.zeros(L.n_mlp, **f32)
        self.gsum = torch.zeros(max(L.row_off[-1], 1), **f32)
        with torch.cuda.device(self.device):
            nbytes = self.lib.b200_fc_dnn_workspace_bytes(ctypes.byref(L.c), self.B)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        a = FcDnnArgs()
        a.B, a.n_numeric, a.n_ids, a.n_strings, a.W = (self.B, len(L.numeric_keys), len(L.tables) + len(L.buckets),
                                                       len(L.string_keys), STRING_WIDTH)
        a.loss, a.logits, a.grads, a.gsum = (self.loss.data_ptr(), self.logits.data_ptr(), self.grads.data_ptr(),
                                             self.gsum.data_ptr())
        a.workspace, a.workspace_bytes = self.workspace.data_ptr(), nbytes
        self.args = a

    def table_view(self, buf, k):
        """Table k's [rows, dim] block of a rows / gsum buffer."""
        L = self.layout
        _, r, d = L.tables[k]
        return buf[L.row_off[k]:L.row_off[k] + r * d].view(r, d)

    def check_inputs(self, numeric, ids, strings, inv, n_unique, rows, labels, flat):
        L, B, dev = self.layout, self.B, self.device
        T = len(L.tables)
        check_tensor(numeric, "numeric", torch.float32, (len(L.numeric_keys), B), dev)
        check_tensor(ids, "ids", torch.int32, (T + len(L.buckets), B), dev)
        check_tensor(strings, "strings", torch.uint8, (len(L.string_keys), B, STRING_WIDTH), dev)
        check_tensor(inv, "inv", torch.int32, (T, B), dev)
        check_tensor(n_unique, "n_unique", torch.int32, (T,), dev)
        check_tensor(rows, "rows", torch.float32, (self.gsum.numel(),), dev)
        if labels is not None:
            check_tensor(labels, "labels", torch.float32, (B,), dev)
        check_tensor(flat, "params", torch.float32, (L.n_mlp,), dev)

    def launch(self, numeric, ids, strings, inv, n_unique, rows, labels, flat, train=True):
        """One tower launch on the current stream (no checks, no host read)."""
        a = self.args
        a.numeric, a.ids, a.strings = numeric.data_ptr(), ids.data_ptr(), strings.data_ptr()
        a.inv, a.n_unique, a.rows = inv.data_ptr(), n_unique.data_ptr(), rows.data_ptr()
        a.labels = labels.data_ptr() if labels is not None else None
        a.params = flat.data_ptr()
        fn = self.lib.b200_fc_dnn_tower if train else self.lib.b200_fc_dnn_forward
        with torch.cuda.device(self.device):
            rc = fn(ctypes.byref(self.layout.c), ctypes.byref(a),
                    ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        _lib.check_call(rc, fn.__name__, self.lib.b200_fc_dnn_last_error)

    def outputs(self, n_unique=None):
        """{loss, logits, grads, gsum: [table k's [rows, dim] block]} (views of the buffers); with n_unique (a
        list of ints), each gsum block is cut to its first n_unique[k] rows."""
        gs = [self.table_view(self.gsum, k) for k in range(len(self.layout.tables))]
        if n_unique is not None:
            gs = [g[:int(n)] for g, n in zip(gs, n_unique)]
        return {"loss": self.loss.reshape(()), "logits": self.logits, "grads": self.grads, "gsum": gs}


def fc_dnn_tower(model, numeric, ids, strings, inv, n_unique, rows, labels, flat, train=True):
    """The tower kernel on one batch, all on one device: numeric float32 [n, B], ids int32 [T + buckets, B] (the
    bucket rows are read), strings uint8 [m, B, 32], inv int32 [T, B] and n_unique int32 [T] of the per-table
    dedup, rows float32 (every table's [rows, dim] block back to back), labels float32 [B] (None with
    train=False) and the flat MLP float32 [16 F + 305].  Returns FcDnnTowerCall.outputs() of fresh buffers."""
    L = layout_of(model)
    B = numeric.shape[1] if isinstance(numeric, torch.Tensor) and numeric.dim() == 2 else 0
    call = FcDnnTowerCall(L, B, flat.device if isinstance(flat, torch.Tensor) else "cuda")
    call.check_inputs(numeric, ids, strings, inv, n_unique, rows, labels, flat)
    call.launch(numeric, ids, strings, inv, n_unique, rows, labels, flat, train)
    return call.outputs()


class FeatureColumnDNNEngine(AsyncEngine):
    """One async worker of census_dnn_model, heart_functional_api or census_model_sqlflow_dnn on the
    parameter-server step.

    group: an async PSGroup, as AsyncEngine takes it.  model: one of LAYOUTS (or a Layout).  register=True
    registers the MLP's six dense parameters and the embedding-column tables, a PS_TABLE as a hashed "uniform"
    table, a DENSE_TABLE as a dense [rows, dim] parameter (initial values of both dense kinds first-writer-wins, as
    PushModel does: Layout.initial_mlp(seed) and initial_tables(seed)); register=False attaches to a
    group.clone_view() of a group where another engine registered them, for another worker thread.  Both table
    kinds go through the same pull_rows and push_rows launches; on a dense parameter push_rows is the Indexed
    update of the batch's unique rows and their slots (Q36).
    step(numeric float32 [n, B], strings uint8 [m, B, 32], labels float32 [B]) runs pull_dense -> the feature
    transform -> empty strings to id 0 -> the per-table dedup -> one pull_rows of the unique rows -> the tower ->
    push_begin -> push_dense -> push_rows (counts on the device) -> push_end, with no host read, and returns the
    loss on the device (a batch sum for the census models, a mean for heart_functional_api: Q16).  capture() /
    replay() run the same step as one CUDA graph over static inputs.  lr_schedule: as AsyncEngine takes it."""

    def __init__(self, group, model, batch, lr, seed=0, register=True, lr_schedule=None):
        self.layout = L = layout_of(model)
        super().__init__(group, batch, lr, register, lr_schedule)
        g, dev, B = self.group, self.device, self.B
        T = len(L.tables)
        self.inputs = [("numeric", torch.float32, (len(L.numeric_keys), B)),
                       ("strings", torch.uint8, (len(L.string_keys), B, STRING_WIDTH)),
                       ("labels", torch.float32, (B,))]
        self.owner = {n: string_to_id(n, g.n_shards)
                      for n in MLP_NAMES + [t for t, kind in zip(L.table_names, L.table_kinds) if kind == DENSE_TABLE]}
        if register:
            for n, kind, (_, rows, dim) in zip(L.table_names, L.table_kinds, L.tables):
                if kind == PS_TABLE:
                    g.register_table(n, dim, "uniform", expected_rows=max(4 * rows, 1024))
                else:
                    g.register_dense(n, (rows, dim), self.owner[n])
            for n, s in L.mlp:
                g.register_dense(n, s, self.owner[n])
            g.commit()
            g.init_dense(list(L.flat_views(L.initial_mlp(seed, dev)).items()) + list(L.initial_tables(seed).items()))
        self.tids = {n: g.lookup(n)[0] for n in L.table_names + MLP_NAMES}  # PSNotFound if unregistered
        self.flat = torch.zeros(L.n_mlp, dtype=torch.float32, device=dev)
        self.views = L.flat_views(self.flat)
        self.transform = L.transform(dev)
        self.ids = torch.zeros((T + len(L.buckets), B), dtype=torch.int32, device=dev)
        self.uniq = torch.zeros(max(T, 1) * B, dtype=torch.int64, device=dev)
        self.inv = torch.zeros((T, B), dtype=torch.int32, device=dev)
        self.n_unique = torch.zeros(max(T, 1), dtype=torch.int32, device=dev)[:T]
        self.tower = t = FcDnnTowerCall(L, B, dev)
        self.rows = torch.zeros_like(t.gsum)
        self.bounds = (ctypes.c_int64 * max(T, 1))(*[r for _, r, _ in L.tables])
        nbytes = g.lib.b200ps_unique_bounded_workspace(T, B, self.bounds) if T else 0
        self.dedup_ws = torch.zeros(max(nbytes, 1), dtype=torch.uint8, device=dev)

        def segs(buf):  # one segment per table: its unique ids, count and [rows, dim] block of `buf`
            return [(self.tids[n], min(B, r), self.uniq[k * B:(k + 1) * B], self.n_unique[k:k + 1], t.table_view(buf, k))
                    for k, (n, (_, r, _)) in enumerate(zip(L.table_names, L.tables))]

        self.pull_dense_segs = g.make_segs([(self.tids[n], 0, None, None, self.views[n]) for n in MLP_NAMES])
        self.pull_rows_segs = g.make_segs(segs(self.rows))
        off, items = 0, []
        for n, s in L.mlp:
            k = int(np.prod(s))
            items.append((self.tids[n], 0, None, None, t.grads[off:off + k]))
            off += k
        self.push_dense_segs = g.make_segs(items)
        self.push_rows_segs = g.make_segs(segs(t.gsum))
        self._eval_tower = None

    # ------------------------------------------------------------------ the step
    def _pull(self, numeric, strings, st):
        """pull_dense -> transform -> empty strings to id 0 -> dedup -> one pull_rows of the unique rows."""
        g, lib, L = self.group, self.group.lib, self.layout
        arr, n = self.pull_dense_segs
        check(lib.b200ps_pull_dense(g._h, arr, n, st))
        self.transform(numeric, strings, ids_out=self.ids)
        T = len(L.tables)
        if T:
            fill_empty(L, self.ids, strings)
            ws = self.dedup_ws
            check(lib.b200ps_unique_bounded_i32(g._h, self.ids.data_ptr(), T, self.B, self.bounds,
                                                self.uniq.data_ptr(), self.inv.data_ptr(), self.n_unique.data_ptr(),
                                                ws.data_ptr(), ws.numel(), st))
            arr, n = self.pull_rows_segs
            check(lib.b200ps_pull_rows(g._h, arr, n, st))

    def _step(self, numeric, strings, labels):
        with torch.cuda.device(self.device):
            st = self.group._stream()
            self._pull(numeric, strings, st)
            self.tower.launch(numeric, self.ids, strings, self.inv, self.n_unique, self.rows, labels, self.flat)
            self._push(st)
        return self.tower.loss.reshape(())

    def evaluate(self, numeric, strings, labels, metrics):
        """The forward only: the step's pulls (rows are created by the pull, as the reference's evaluation
        lookups create them), the tower's forward form, then metrics.update_evaluation_metrics({"logits": logits,
        "probs": sigmoid(logits)}, labels) (an EvaluationMetrics, e.g. of eval_metrics_fn(model)).  Pushes
        nothing.  Returns the logits [B] on the device (overwritten by the next evaluate)."""
        self._check_batch(numeric, strings, labels)
        if self._eval_tower is None:
            self._eval_tower = FcDnnTowerCall(self.layout, self.B, self.device)
        with torch.cuda.device(self.device):
            self._pull(numeric, strings, self.group._stream())
            self._eval_tower.launch(numeric, self.ids, strings, self.inv, self.n_unique, self.rows, None, self.flat,
                                    train=False)
            logits = self._eval_tower.logits
            metrics.update_evaluation_metrics({"logits": logits, "probs": torch.sigmoid(logits)}, labels)
        return logits

    def check(self):
        """Raise if a step since the last check flagged an error on the group (e.g. a hashed table ran out of
        slots); synchronises the device."""
        self.group.check()


def twin_features(model, numeric, strings, transform=None):
    """The drop-in twin's features from raw rows: {"numeric": float32 [n, B], "buckets": int64 [n_buckets, B],
    "present": float32 [T, B] (0 where the table's string is empty), <key>: int64 [B] hash bucket per table, 0
    where empty}.  Each table's ids are a feature of their own, so the trainer's batched lookup plan (and its
    CUDA graph) applies."""
    L = layout_of(model)
    transform = transform or L.transform(numeric.device)
    ids, _ = transform(numeric, strings)
    T = len(L.tables)
    if T:
        fill_empty(L, ids, strings)
    present = torch.stack([strings[L.string_keys.index(k), :, 0] != 0 for k, _, _ in L.tables]).float() if T else \
        torch.zeros((0, numeric.shape[1]), device=numeric.device)
    out = {"numeric": numeric, "buckets": ids[T:].long().contiguous(), "present": present.contiguous()}
    for k, (key, _, _) in enumerate(L.tables):
        out[key] = ids[k].long().contiguous()
    return out


class FeatureColumnDNN(torch.nn.Module):
    """The same model as a torch module for the drop-in ParameterServerTrainer: per embedding column, a PS_TABLE is
    an elasticdl_b200.layers.Embedding under the reference's table name (a hashed "uniform" PS table) and a
    DENSE_TABLE a torch.nn.Embedding(rows, dim) whose weight is also this module's parameter of the table's name,
    so that ParameterServerModelHandler keeps it as a DenseTableEmbedding (at most 2 MB) and the trainer pulls and
    pushes its rows by id under that name (Q36).  Empty-string rows are zeroed, and the three Dense layers are
    Keras-named parameters (dense/kernel:0 [F, 16], ...), so that the trainer registers the same PS parameters, with
    the same update kinds, as the engine does.  forward(twin_features(...)) returns the probability [B]; the loss is
    the Keras clipped binary cross-entropy, summed (the census models) or averaged (heart_functional_api)."""

    def __init__(self, model, lr=None, optimizer=None):
        super().__init__()
        from elasticdl_b200.layers import Embedding

        L = self.layout = layout_of(model)
        self.tables = torch.nn.ModuleList()
        for kind, (key, rows, dim) in zip(L.table_kinds, L.tables):
            if kind == PS_TABLE:
                e = Embedding(dim, embeddings_initializer="uniform", name="%s_embedding" % key)
                e.set_embedding_weight_name(table_name(key))
            else:  # registered here first, so named_parameters() gives the weight the table's name
                e = torch.nn.Embedding(rows, dim)
                self.register_parameter(table_name(key), e.weight)
            self.tables.append(e)
        for n, s in L.mlp:
            self.register_parameter(n, torch.nn.Parameter(torch.zeros(s)))
        self.load_mlp(L.initial_mlp(0, "cpu"))
        self.load_tables(L.initial_tables(0))
        lr = L.optimizer[2] if lr is None else lr
        opt = torch.optim.Adam if (optimizer or L.optimizer[0]).lower() == "adam" else torch.optim.SGD
        self.optimizer = opt([getattr(self, n) for n in MLP_NAMES], lr=lr)
        self.loss = lambda labels, p: keras_bce(labels, p, L.loss_mean)

    def load_mlp(self, flat):
        v = self.layout.flat_views(flat)
        with torch.no_grad():
            for n in MLP_NAMES:
                getattr(self, n).copy_(v[n])

    def load_tables(self, tables):
        """Copy {table name: [rows, dim]} into the DENSE_TABLE weights."""
        with torch.no_grad():
            for n, v in tables.items():
                getattr(self, n).copy_(v)

    def dense_features(self, features):
        L = self.layout
        numeric, buckets, present = features["numeric"], features["buckets"], features["present"]
        cols = []
        for _, kind, key in L.columns:
            if kind == NUMERIC:
                cols.append(numeric[L.numeric_keys.index(key)].unsqueeze(1))
            elif kind == BUCKET:
                i = [k for k, _ in L.buckets].index(key)
                width = len(L.buckets[i][1]) + 1
                cols.append((buckets[i].unsqueeze(1) == torch.arange(width, device=buckets.device)).to(numeric.dtype))
            else:
                k = [t for t, _, _ in L.tables].index(key)
                cols.append(self.tables[k](features[key]) * present[k].unsqueeze(1))
        return torch.cat(cols, 1)

    def forward(self, features):
        x = self.dense_features(features)
        h = torch.relu(x @ getattr(self, "dense/kernel:0") + getattr(self, "dense/bias:0"))
        h = torch.relu(h @ getattr(self, "dense_1/kernel:0") + getattr(self, "dense_1/bias:0"))
        z = (h @ getattr(self, "dense_2/kernel:0") + getattr(self, "dense_2/bias:0"))[:, 0]
        return torch.sigmoid(z)


def keras_bce(labels, p, mean):
    """tf.keras.losses.binary_crossentropy on probabilities (Q19): clip to [1e-7, 1 - 1e-7] (no gradient where
    the clip is active), -(y log(p + 1e-7) + (1 - y) log(1 - p + 1e-7)); the batch mean or sum (Q16)."""
    eps = float(np.float32(1e-7))  # the float32 constants Keras computes with, also in a float64 check
    pc = torch.clamp(p, eps, float(np.float32(1.0) - np.float32(eps)))
    l = -(labels * torch.log(pc + eps) + (1.0 - labels) * torch.log(1.0 - pc + eps))  # noqa: E741
    return l.mean() if mean else l.sum()
