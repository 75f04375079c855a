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
import collections
import ctypes

import numpy as np
import torch

from elasticdl_b200 import _lib
from elasticdl_b200._lib import CensusArgs, check
from elasticdl_b200.common.hash_utils import string_to_id
from elasticdl_b200.workloads.async_engine import AsyncEngine, check_tensor
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


def callbacks():
    """The census model's learning-rate schedule (model_zoo/census_wide_deep_model/wide_deep_functional_api.py:74-83:
    3e-4 below version 5000, 2e-4 below 12000, then 1e-4) as a declarative schedule the push evaluates on the
    device; versions are integers, so `< 5000` is `<= 4999`."""
    from elasticdl_b200.callbacks import LearningRateScheduler, PiecewiseConstantDecay

    return [LearningRateScheduler(PiecewiseConstantDecay([4999, 11999], [3e-4, 2e-4, 1e-4]))]


# What a census-style wide & deep tower's entry points and buffers depend on (SPEC here, census_sqlflow.SPEC):
# the entry points' prefix and argument struct, the groups' rows, the push_rows segments' offsets and sizes, the
# flat sizes, what the range error says after its count, and whether a forward-only entry point (<prefix>_forward)
# exists.
TowerSpec = collections.namedtuple("TowerSpec", "prefix args group_rows uniq_off n_uniq gsum_off n_gsum n_params n_mlp "
                                                "range_error forward")
SPEC = TowerSpec("b200_census", CensusArgs, GROUP_ROWS, UNIQ_OFF, N_UNIQ, GSUM_OFF, N_GSUM, N_PARAMS, N_MLP,
                 "census ids outside [0, rows of their group) %s were read as row 0" % (GROUP_ROWS,), False)


class TowerCall:
    """A census-style tower's output buffers and workspace for batch B on `device`, and one launch over them; a
    subclass sets `spec`, a TowerSpec."""

    spec = None

    def __init__(self, B, device):
        self.B = int(B)
        if self.B < 1:
            raise ValueError("batch size must be >= 1, not %d" % self.B)
        self.device = torch.device(device)
        self.lib = _lib.lib()
        sp = self.spec
        f32 = dict(dtype=torch.float32, device=self.device)
        self.loss = torch.zeros(1, **f32)
        self.logits = torch.zeros(self.B, **f32)
        self.grads = torch.zeros(sp.n_mlp, **f32)
        self.uniq = torch.zeros(sp.n_uniq, dtype=torch.int64, device=self.device)
        self.n_unique = torch.zeros(5, dtype=torch.int32, device=self.device)
        self.gsum = torch.zeros(sp.n_gsum, **f32)
        self.error = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            nbytes = getattr(self.lib, sp.prefix + "_workspace_bytes")(self.B)
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        a = sp.args()
        a.B = self.B
        a.loss, a.logits, a.grads = self.loss.data_ptr(), self.logits.data_ptr(), self.grads.data_ptr()
        a.uniq, a.n_unique, a.gsum = self.uniq.data_ptr(), self.n_unique.data_ptr(), self.gsum.data_ptr()
        a.error, a.workspace, a.workspace_bytes = self.error.data_ptr(), self.workspace.data_ptr(), nbytes
        self.args = a

    def check_inputs(self, ids, labels, flat):
        """labels may be None where the tower has a forward form."""
        check_tensor(ids, "ids", torch.int32, (12, self.B), self.device)
        if labels is not None or not self.spec.forward:
            check_tensor(labels, "labels", torch.float32, (self.B,), self.device)
        check_tensor(flat, "params", torch.float32, (self.spec.n_params,), self.device)

    def launch(self, ids, labels, flat, reference_reshape, train=True):
        """One tower launch (train=False: the forward form, logits only) on the current stream (no checks, no host
        read)."""
        if not (train or self.spec.forward):
            raise ValueError("%s has no forward form" % self.spec.prefix)
        a = self.args
        a.ids, a.params = ids.data_ptr(), flat.data_ptr()
        a.labels = labels.data_ptr() if labels is not None else None
        a.reference_reshape = 1 if reference_reshape else 0
        fn = getattr(self.lib, self.spec.prefix + ("_tower" if train else "_forward"))
        with torch.cuda.device(self.device):
            rc = fn(ctypes.byref(a), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        _lib.check_call(rc, fn.__name__, getattr(self.lib, self.spec.prefix + "_last_error"))

    def check_error(self):
        """Raise PSRangeError (a ValueError) if a launch since the last check read an id outside its group, and
        clear the count.  Reads one int from the device."""
        n = int(self.error.item())
        if n:
            self.error.zero_()
            raise _lib.PSRangeError(_lib.ERANGE, "%d %s" % (n, self.spec.range_error))

    def outputs(self):
        """{loss, logits, grads, uniq [5], n_unique [5], gsum [5 segments: [rows, dim]]} (views of the buffers)."""
        out = {"loss": self.loss.reshape(()), "logits": self.logits, "grads": self.grads, "n_unique": self.n_unique,
               "uniq": [], "gsum": []}
        sp = self.spec
        for t in range(5):
            rows = sp.group_rows[TABLE_GROUP[t]]
            out["uniq"].append(self.uniq[sp.uniq_off[t]:sp.uniq_off[t] + rows])
            out["gsum"].append(self.gsum[sp.gsum_off[t]:sp.gsum_off[t] + rows * TABLE_DIM[t]].view(rows, TABLE_DIM[t]))
        return out


class CensusTowerCall(TowerCall):
    """The census tower's output buffers and workspace for batch B on `device`, and one launch over them."""

    spec = SPEC


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


def _split(flat, shapes):
    """Views of consecutive blocks of `flat` in `shapes`."""
    out, o = [], 0
    for s in shapes:
        out.append(flat[o:o + int(np.prod(s))].view(s))
        o += int(np.prod(s))
    return out


class WideDeepEngine(AsyncEngine):
    """One async worker of a census-style wide & deep model on the parameter-server step: the body of
    CensusWideDeepEngine and census_sqlflow.CensusSqlflowEngine.

    step(numeric float32 [4, B], strings uint8 [8, B, 32], labels float32 [B]) runs pull_dense (into the flat
    buffer) -> the feature transform -> the tower -> push_begin -> push_dense (MLP) -> push_rows (the five tables'
    touched rows, counts on the device) -> push_end, with no host read, and returns the loss on the device.
    capture() / replay() run the same step as one CUDA graph over static inputs; a new learning rate re-captures.
    A subclass runs AsyncEngine.__init__, sets `reference_reshape` and calls _setup()."""

    def _setup(self, names, shapes, initial_params, seed, transform, tower, register):
        """names, shapes: the eleven parameters in flat order; register=True registers them and sets their initial
        values, initial_params(seed, device), first-writer-wins (as PushModel does).  transform: the model's feature
        transform (raw rows -> int32 ids [12, B]); tower: its TowerCall class."""
        g, B = self.group, self.B
        self.inputs = [("numeric", torch.float32, (4, B)), ("strings", torch.uint8, (8, B, STRING_WIDTH)),
                       ("labels", torch.float32, (B,))]
        self.names = names
        self.owner = {n: string_to_id(n, g.n_shards) for n in names}
        if register:
            for n, s in zip(names, shapes):
                g.register_dense(n, s, self.owner[n])
            g.commit()
            g.init_dense(zip(names, _split(initial_params(seed, self.device), shapes)))
        tids = [g.lookup(n)[0] for n in names]  # PSNotFound when no engine registered them
        self.flat = torch.zeros(tower.spec.n_params, dtype=torch.float32, device=self.device)
        self.ids = torch.zeros((12, B), dtype=torch.int32, device=self.device)
        self.transform = transform
        self.tower = t = tower(B, self.device)
        self.pull_segs = g.make_segs([(tid, 0, None, None, v) for tid, v in zip(tids, _split(self.flat, shapes))])
        self.push_dense_segs = g.make_segs([(tid, 0, None, None, v)
                                            for tid, v in zip(tids, _split(t.grads, shapes[:6]))])
        out = t.outputs()
        self.push_rows_segs = g.make_segs([(tids[6 + k], t.spec.group_rows[TABLE_GROUP[k]], out["uniq"][k],
                                            t.n_unique[k:k + 1], out["gsum"][k]) for k in range(5)])
        self._eval_tower = None  # evaluate()'s tower buffers (lazy)

    def _pull(self, numeric, strings, st):
        check(self.group.lib.b200ps_pull_dense(self.group._h, *self.pull_segs, st))
        if numeric is not None:
            self.transform(numeric, strings, ids_out=self.ids)

    def _step(self, numeric, strings, labels, ids=None):
        with torch.cuda.device(self.device):
            st = self.group._stream()
            self._pull(numeric, strings, st)
            self.tower.launch(self.ids if ids is None else ids, labels, self.flat, self.reference_reshape)
            self._push(st)
        return self.tower.loss.reshape(())

    def evaluate(self, numeric, strings, labels, metrics):
        """Forward only from raw rows: pull_dense -> the transform -> the tower -> metrics.update_evaluation_metrics(
        {"logits": logits, "probs": sigmoid(logits)}, labels) (an EvaluationMetrics, e.g. of eval_metrics_fn()).
        A tower without a forward form runs its training launch, whose gradients evaluate() discards -- into
        buffers of its own, so the step's loss and gradients stay as they were.  Pushes nothing.  Returns the
        logits [B] on the device (overwritten by the next evaluate)."""
        self._check_batch(numeric, strings, labels)
        if self._eval_tower is None:
            self._eval_tower = type(self.tower)(self.B, self.device)
        t = self._eval_tower
        with torch.cuda.device(self.device):
            self._pull(numeric, strings, self.group._stream())
            if t.spec.forward:
                t.launch(self.ids, None, self.flat, self.reference_reshape, train=False)
            else:
                t.launch(self.ids, labels, self.flat, self.reference_reshape)
            metrics.update_evaluation_metrics({"logits": t.logits, "probs": torch.sigmoid(t.logits)}, labels)
        return t.logits

    def check(self):
        """Raise PSRangeError (a ValueError) if a step or evaluate since the last check read an id outside its
        group; one device read per tower."""
        if self._eval_tower is not None:
            self._eval_tower.check_error()
        self.tower.check_error()


class CensusWideDeepEngine(WideDeepEngine):
    """One async worker of the census wide & deep model on the parameter-server step (WideDeepEngine), from raw
    Adult rows through census_transform.

    group: an async PSGroup, as AsyncEngine takes it.  register=True registers the eleven parameters and sets their
    initial values first-writer-wins (as PushModel does); register=False attaches to a group.clone_view() of a
    group where another engine registered them, for another worker thread.  lr_schedule: a schedule to install, as
    AsyncEngine.set_lr_schedule does.  There is no forward-only census kernel: evaluate() runs the training launch
    into buffers of its own."""

    def __init__(self, group, batch, lr, reference_reshape=False, seed=0, register=True, lr_schedule=None):
        super().__init__(group, batch, lr, register, lr_schedule)
        self.reference_reshape = bool(reference_reshape)
        self._setup([n for n, _ in PARAMS], [s for _, s in PARAMS], initial_params, seed,
                    census_transform(torch.int32, device=self.device), CensusTowerCall, register)
        self.views = flat_views(self.flat)

    def step_ids(self, ids, labels):
        """One training step from the ids census_transform(torch.int32) gives: int32 [12, B]."""
        self.tower.check_inputs(ids, labels, self.flat)
        out = self._step(None, None, labels, ids)
        self.steps += 1
        return out


class WideDeepTwin(torch.nn.Module):
    """What the census-style models' torch twins share: the MLP (three torch Linear layers, with their optimizer),
    the loss and the tower over pooled lookups.  wide, deep: the subclass's wide and deep tables."""

    def __init__(self, wide, deep, lr, reference_reshape, optimizer):
        super().__init__()
        self.reference_reshape = bool(reference_reshape)
        self.wide = torch.nn.ModuleList(wide)
        self.deep = torch.nn.ModuleList(deep)
        self.dense = torch.nn.ModuleList([torch.nn.Linear(24, 16), torch.nn.Linear(16, 8), torch.nn.Linear(8, 4)])
        self.transform = None  # built at the first forward (its vocabulary tables live on the device)
        opt = torch.optim.SGD if optimizer == "sgd" else torch.optim.Adam
        self.optimizer = opt(self.dense.parameters(), lr=lr)
        bce = torch.nn.BCEWithLogitsLoss()
        self.loss = lambda labels, logits: bce(logits, labels)

    def load_mlp(self, flat):
        """Copy the MLP block of a flat buffer (Keras [in, out] kernels) into the Linear layers."""
        v = _split(flat, [s for _, s in PARAMS[:6]])
        with torch.no_grad():
            for i, lin in enumerate(self.dense):
                lin.weight.copy_(v[2 * i].t())
                lin.bias.copy_(v[2 * i + 1])

    def tower(self, wide, deep):
        """wide [2, B] and deep [3, B, 8] pooled lookups -> logits [B]."""
        B = deep.shape[1]
        x = deep.reshape(B, 24) if self.reference_reshape else deep.permute(1, 0, 2).reshape(B, 24)
        for lin in self.dense:
            x = lin(x)
        return wide.sum(0) + x.sum(1)


class CensusWideDeep(WideDeepTwin):
    """The same model as a torch module for the drop-in ParameterServerTrainer: the tables are
    elasticdl_b200.layers.Embedding layers (row-sparse PS tables; only the rows of the batch are pulled and
    updated), the MLP is three torch Linear layers, both reshape modes.  forward((numeric, strings)) runs
    census_transform and sums each group's four lookups."""

    def __init__(self, lr, reference_reshape=False, optimizer="sgd"):
        from elasticdl_b200.layers import Embedding

        wide = [Embedding(1, input_dim=r, embeddings_initializer="uniform", name=n.split("/")[0])
                for n, r in zip(TABLE_NAMES[:2], GROUP_ROWS[:2])]
        deep = [Embedding(8, input_dim=r, embeddings_initializer="uniform", name=n.split("/")[0])
                for n, r in zip(TABLE_NAMES[2:], GROUP_ROWS)]
        super().__init__(wide, deep, lr, reference_reshape, optimizer)

    def forward(self, features):
        numeric, strings = features
        if self.transform is None:
            self.transform = census_transform(torch.int64, device=numeric.device)
        ids, _ = self.transform(numeric, strings)
        wide = torch.stack([self.wide[g](ids[4 * g:4 * g + 4]).sum(0)[:, 0] for g in range(2)])
        deep = torch.stack([self.deep[g](ids[4 * g:4 * g + 4]).sum(0) for g in range(3)])
        return self.tower(wide, deep)
