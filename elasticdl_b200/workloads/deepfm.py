"""DeepFM on Criteo-shaped data over the HBM parameter server: the workload of
BASELINE.json configs[1] (model_zoo/dac_ctr/deepfm_model.py:20-109, utils.py:17-41,
feature_config.py:61-195, feature_transform.py:33,102-110).

38 id groups (12 bucketised integer features + 26 hashed categorical features
capped at 1e6 buckets), one id per group per sample, two embedding tables per
group (wide dim 1, deep dim 8) -> 76 PS tables, 5 549 416 rows per family; dense
tower DNN[16,4] over 13 + 38*8 inputs, FM over the 38x8 deep embeddings, linear
part = sum of wide embeddings + Dense(1)(dense features); Adam lr 1e-3.

`DeepFMPSEngine.step` is one pass of the hot path: pull dense -> unique ids
(first-occurrence) -> pull rows (one launch for all 76 tables; with row_source="table" the
tile tower reads the rows from the tables itself and there is no pull) -> gather -> tower
fwd/bwd (torch, library GEMMs) -> segment-sum of per-occurrence gradients -> push (dense +
76 tables, fused Adam) -> version++.  No host sync inside the step; nothing but
ids/features/labels comes from the host.
"""
import collections
import ctypes
import math

import torch

from elasticdl_b200._lib import DEEPFM_DCN_SCRATCH, DEEPFM_TILE_MAXG, DEEPFM_TILE_SCRATCH, MAX_SEGS, check

# model_zoo/dac_ctr/feature_config.py:61-75 (len(boundaries)+1 buckets; I4 is not in FEATURE_GROUPS)
INT_BUCKETS = [5, 10, 9, 10, 9, 9, 10, 10, 3, 6, 2, 9]
# feature_config.py:123-150 distinct counts, capped by MAX_HASHING_BUCKET_SIZE = 1e6 (feature_transform.py:33)
CAT_COUNTS = [1460, 582, 9264260, 2046299, 305, 24, 12506, 633, 3, 91211, 5670, 7659856, 3194, 27, 14876,
              5031503, 10, 5624, 2171, 4, 6477624, 18, 15, 272811, 105, 138075]
GROUP_ROWS = INT_BUCKETS + [min(c, 1000000) for c in CAT_COUNTS]
N_GROUPS = len(GROUP_ROWS)  # 38
N_DENSE = 13
DEEP_DIM = 8
assert N_GROUPS == 38 and sum(GROUP_ROWS) == 5549416


class DeepFMTower(torch.nn.Module):
    """deepfm_model.py:61-109 without the embedding lookups."""

    def __init__(self, n_groups=N_GROUPS, deep_dim=DEEP_DIM, n_dense=N_DENSE, hidden=(16, 4)):
        super().__init__()
        self.n_groups, self.deep_dim = n_groups, deep_dim
        self.dense_linear = torch.nn.Linear(n_dense, 1, bias=False)
        dims = [n_dense + n_groups * deep_dim] + list(hidden)
        self.dnn = torch.nn.ModuleList([torch.nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])])
        self.dnn_logit = torch.nn.Linear(dims[-1], 1, bias=False)

    def forward(self, dense, wide, deep):
        """dense [B,13], wide [B,G], deep [B,G,D] -> logits [B]."""
        B = dense.shape[0]
        x = torch.cat([dense, deep.reshape(B, -1)], 1)
        for layer in self.dnn:
            x = torch.relu(layer(x))
        dnn_logit = self.dnn_logit(x).squeeze(1)
        linear_logit = wide.sum(1) + self.dense_linear(dense).squeeze(1)
        s = deep.sum(1)  # FM: 0.5 * sum_d[(sum_f e)^2 - sum_f e^2]  (deepfm_edl_embedding.py:50-56)
        fm = 0.5 * (s * s - (deep * deep).sum(1)).sum(1)
        return linear_logit + dnn_logit + fm


class WideDeepTower(DeepFMTower):
    """wide_deep_model.py:62-107 without the embedding lookups: DeepFMTower without the FM term (the same
    parameters, under the same names, so the flat layout is DeepFM's)."""

    def forward(self, dense, wide, deep):
        """dense [B,13], wide [B,G], deep [B,G,D] -> logits [B]."""
        B = dense.shape[0]
        x = torch.cat([dense, deep.reshape(B, -1)], 1)
        for layer in self.dnn:
            x = torch.relu(layer(x))
        dnn_logit = self.dnn_logit(x).squeeze(1)
        linear_logit = wide.sum(1) + self.dense_linear(dense).squeeze(1)
        return linear_logit + dnn_logit


class DCNTower(torch.nn.Module):
    """dcn_model.py:53-95 without the embedding lookups: the same DNN[16, 4] and linear part as DeepFMTower, FM
    replaced by a CrossNet over x0 = [dense | deep] (deepctr's CrossNet, "vector" parameterization, DCN paper eq. 3:
    x_{l+1} = x0 * (x_l . w_l) + b_l + x_l; kernels glorot-normal, biases zero) and one bias-free output unit over
    [dnn_out | x_L].  regularization() is the l2 term the model adds to its loss (model.losses)."""

    def __init__(self, n_groups=N_GROUPS, deep_dim=DEEP_DIM, n_dense=N_DENSE, hidden=(16, 4), cross_layers=2,
                 l2_reg=1e-5):
        super().__init__()
        self.n_groups, self.deep_dim, self.l2_reg = n_groups, deep_dim, l2_reg
        n_in = n_dense + n_groups * deep_dim
        self.dense_linear = torch.nn.Linear(n_dense, 1, bias=False)
        dims = [n_in] + list(hidden)
        self.dnn = torch.nn.ModuleList([torch.nn.Linear(a, b) for a, b in zip(dims[:-1], dims[1:])])
        self.out = torch.nn.Linear(dims[-1] + n_in, 1, bias=False)
        # keras glorot_normal of a [n_in, 1] kernel: truncated normal, std sqrt(2 / (n_in + 1)) / 0.8796
        std = math.sqrt(2.0 / (n_in + 1)) / 0.87962566103423978
        self.cross_w = torch.nn.Parameter(torch.nn.init.trunc_normal_(torch.empty(cross_layers, n_in), 0.0, std,
                                                                      -2 * std, 2 * std))
        self.cross_b = torch.nn.Parameter(torch.zeros(cross_layers, n_in))

    def forward(self, dense, wide, deep):
        """dense [B,13], wide [B,G], deep [B,G,D] -> logits [B]."""
        B = dense.shape[0]
        x0 = torch.cat([dense, deep.reshape(B, -1)], 1)
        h = x0
        for layer in self.dnn:
            h = torch.relu(layer(h))
        x = x0
        for w, b in zip(self.cross_w, self.cross_b):
            x = x0 * (x @ w).unsqueeze(1) + b + x
        deep_cross_logit = self.out(torch.cat([h, x], 1)).squeeze(1)
        linear_logit = wide.sum(1) + self.dense_linear(dense).squeeze(1)
        return linear_logit + deep_cross_logit

    def regularization(self):
        return self.l2_reg * (self.cross_w * self.cross_w).sum()


class XDeepFMTower(WideDeepTower):
    """xdeepfm_model.py:55-107 without the embedding lookups: WideDeepTower (its parameters under the same names)
    plus a Compressed Interaction Network over the deep rows X0 = deep [B, G, D] (deepctr's CIN with
    layer_size=(128, 128), activation="relu", split_half=True) and its Dense(1) over the 192 pooled channels:
        Z_k[b, d, i H_k + j] = X0[b, i, d] X_k[b, j, d],   C_k = relu(W_k Z_k + b_k)   [B, 128, D],
        X_1 = C_0[:, :64],  p = [C_0[:, 64:] | C_1].sum(d),  logit = Wide & Deep + exfm(p).
    Filters glorot-uniform over (K, 128), biases zero.  regularization() is the filters' l2 term.  Needs G >= 2: with
    one field the reference builds a different model (no CIN)."""

    def __init__(self, n_groups=N_GROUPS, deep_dim=DEEP_DIM, n_dense=N_DENSE, hidden=(16, 4), layer_size=(128, 128),
                 l2_reg=1e-5):
        super().__init__(n_groups, deep_dim, n_dense, hidden)
        self.l2_reg = l2_reg
        h0, h1 = layer_size
        k0, k1 = n_groups * n_groups, n_groups * (h0 // 2)

        def glorot(rows, cols):
            lim = math.sqrt(6.0 / (rows + cols))
            return torch.nn.Parameter(torch.empty(rows, cols).uniform_(-lim, lim))

        self.cin_w0, self.cin_b0 = glorot(h0, k0), torch.nn.Parameter(torch.zeros(h0))
        self.cin_w1, self.cin_b1 = glorot(h1, k1), torch.nn.Parameter(torch.zeros(h1))
        self.exfm = torch.nn.Linear(h0 // 2 + h1, 1)
        with torch.no_grad():
            self.exfm.weight.copy_(glorot(1, h0 // 2 + h1))
            self.exfm.bias.zero_()

    def cin(self, deep):
        """deep [B, G, D] -> p [B, 192]."""
        B, G, D = deep.shape
        x, direct = deep, []
        for k, (w, b) in enumerate(((self.cin_w0, self.cin_b0), (self.cin_w1, self.cin_b1))):
            z = torch.einsum("bid,bjd->bdij", deep, x).reshape(B, D, G * x.shape[1])
            c = torch.relu(torch.matmul(z, w.t()) + b).transpose(1, 2)  # [B, 128, D]
            if k == 0:
                x, c = c[:, :c.shape[1] // 2], c[:, c.shape[1] // 2:]
            direct.append(c)
        return torch.cat(direct, 1).sum(2)

    def forward(self, dense, wide, deep):
        """dense [B,13], wide [B,G], deep [B,G,D] -> logits [B]."""
        return super().forward(dense, wide, deep) + self.exfm(self.cin(deep)).squeeze(1)

    def regularization(self):
        return self.l2_reg * ((self.cin_w0 * self.cin_w0).sum() + (self.cin_w1 * self.cin_w1).sum())


TOWERS = {"deepfm": DeepFMTower, "dcn": DCNTower, "wide_deep": WideDeepTower, "xdeepfm": XDeepFMTower}


def eval_metrics_fn():
    """The dac_ctr models' evaluation metrics (model_zoo/dac_ctr/elasticdl_train.py:51-60): accuracy of the
    LOGITS thresholded at 0.5 (quirk Q12, DESIGN.md section 4) and the AUC of the probabilities."""
    from elasticdl_b200.common.evaluation_utils import zoo_eval_metrics

    return zoo_eval_metrics(0.5)


def synthetic_batch(batch, seed, device, dist="zipf", zipf_s=1.05, group_rows=GROUP_ROWS):
    """SURVEY.md section 8d config 2: bucket ids uniform, categorical ids Zipf(s) over the
    table's rows (or uniform), dense features N(0,1), labels Bernoulli(0.25).
    Returns ids [G, B] int64 (group-major, like the reference's per-group id tensors)."""
    g = torch.Generator(device=device).manual_seed(seed)
    G = len(group_rows)
    u = torch.rand((G, batch), generator=g, device=device, dtype=torch.float64)
    rows = torch.tensor(group_rows, device=device, dtype=torch.float64).unsqueeze(1)
    if dist == "zipf":
        # bounded-Pareto inverse CDF: rank in [1, N], P(rank) ~ rank^-s
        a = 1.0 - zipf_s
        rank = torch.floor(((rows.pow(a) - 1.0) * u + 1.0).pow(1.0 / a))
        ids = (rank - 1.0).clamp_(min=0)
        ids = torch.minimum(ids, rows - 1)
        small = rows < 64  # the bucketised integer groups are uniform
        ids = torch.where(small.expand_as(ids), torch.floor(u * rows), ids)
    else:
        ids = torch.floor(u * rows)
    ids = ids.to(torch.int64)
    dense = torch.randn((batch, N_DENSE), generator=g, device=device)
    labels = (torch.rand(batch, generator=g, device=device) < 0.25).float()
    return ids, dense, labels


def id_widths(group_rows):
    """Bytes per id of every group on the wire: a table with at most 256 / 65536 rows needs one / two."""
    return [1 if r <= 256 else (2 if r <= 65536 else 4) for r in group_rows]


def _ids_layout(B, widths):
    """[(byte offset, width)] of the per-group id segments (each padded to 16 bytes) and the total."""
    off, out = 0, []
    for w in widths:
        out.append((off, w))
        off += (B * w + 15) // 16 * 16
    return out, off


def packed_nbytes(G, B, widths=None):
    """One training batch as ONE buffer: [ids, group by group at their own width | dense fp32 B x 13 | labels fp32 B].
    widths=None: int32 ids."""
    widths = widths or [4] * G
    return _ids_layout(B, widths)[1] + 4 * B * N_DENSE + 4 * B


def packed_views(buf, G, B, widths=None):
    """(ids, dense fp32 [B, 13], labels fp32 [B]) views of a packed uint8 buffer; ids is an int32 [G, B] view
    when every width is 4 and the segments need no padding (B % 4 == 0), else the uint8 id region itself (the
    dedup kernel reads it with the widths)."""
    widths = widths or [4] * G
    a = _ids_layout(B, widths)[1]
    b = a + 4 * B * N_DENSE
    ids = buf[:a].view(torch.int32).view(G, B) if all(w == 4 for w in widths) and B % 4 == 0 else buf[:a]
    return ids, buf[a:b].view(torch.float32).view(B, N_DENSE), buf[b:b + 4 * B].view(torch.float32)


_NP_UINT = {1: torch.uint8, 2: torch.int16, 4: torch.int32}


def check_id_widths(ids, widths):
    """Raise ValueError unless every id of group g (ids [G, B]) fits widths[g] bytes: 0 <= id < min(256**w, 2**31)
    (4-byte ids are read back as int32 on the int32 transport).  Narrowing is a plain cast, so an id outside that
    range would wrap around onto another, valid row; the dedup kernel can only range-check what it reads."""
    lo, hi = (t.tolist() for t in torch.aminmax(ids, dim=1))
    for g, (w, a, b) in enumerate(zip(widths, lo, hi)):
        lim = min(256 ** w, 2 ** 31)
        if a < 0 or b >= lim:
            raise ValueError("id group %d: id %d does not fit its %d-byte ids (0 <= id < %d)"
                             % (g, a if a < 0 else b, w, lim))


def pack_batch(ids, dense, labels, pin=False, widths=None):
    """Pack (ids int64/int32 [G, B], dense [B, 13], labels [B]) into one uint8 buffer on the same device
    (pin=True: pinned host memory).  ids are narrowed to `widths` bytes per group (default int32: every
    dac_ctr table has fewer than 2^31 rows); the device widens them again inside the dedup kernel
    (b200ps_unique_bounded_i32 / b200ps_unique_packed), so the PS sees the same int64 ids.  An id that does
    not fit its group's width raises ValueError (check_id_widths)."""
    G, B = ids.shape
    widths = widths or [4] * G
    check_id_widths(ids, widths)
    layout, a = _ids_layout(B, widths)
    buf = torch.zeros(packed_nbytes(G, B, widths), dtype=torch.uint8, device="cpu" if pin else ids.device)
    if pin:
        buf = buf.pin_memory()
    for g, (off, w) in enumerate(layout):
        # unsigned narrowing: two's complement of the low bytes (uint16 as int16 bits)
        seg = buf[off:off + B * w].view(_NP_UINT[w])
        v = ids[g].to(torch.int64)
        if w == 2:
            v = torch.where(v >= 32768, v - 65536, v)
        seg.copy_(v.to(_NP_UINT[w]))
    _, v_dense, v_labels = packed_views(buf, G, B, widths)
    v_dense.copy_(dense)
    v_labels.copy_(labels)
    return buf


def flat_order(tower):
    """[(parameter, padded size or None)] of the tower in its flat layout (include/b200_deepfm.h)."""
    order = [(tower.dense_linear.weight, 16), (tower.dnn[0].weight, None), (tower.dnn[0].bias, None),
             (tower.dnn[1].weight, None), (tower.dnn[1].bias, None)]
    if isinstance(tower, DCNTower):
        return order + [(tower.out.weight, None), (tower.cross_w, None), (tower.cross_b, None)]
    order.append((tower.dnn_logit.weight, None))
    if isinstance(tower, XDeepFMTower):
        order += [(tower.cin_w0, None), (tower.cin_b0, None), (tower.cin_w1, None), (tower.cin_b1, None),
                  (tower.exfm.weight, None), (tower.exfm.bias, None)]
    return order


def flatten_tower(tower, flat):
    """Re-point the tower's parameters at views of one flat buffer laid out as
    include/b200_deepfm.h documents: DeepFM and Wide & Deep [w_dense 13 (+3 pad) | w1 | b1 | w2 | b2 | w3], DCN
    [w_dense 13 (+3 pad) | w1 | b1 | w2 | b2 | w_out | w_0 w_1 | b_0 b_1], xDeepFM Wide & Deep's then
    [W_0 | b_0 | W_1 | b_1 | w_ex | b_ex]."""
    order = flat_order(tower)
    off, views = 0, []
    with torch.no_grad():
        for p, padded in order:
            n = p.numel()
            flat[off:off + n].copy_(p.reshape(-1))
            p.data = flat[off:off + n].view(p.shape)
            views.append((off, n))
            off += padded or n
    return views


class HostFeeder:
    """Pinned-host batches -> staging slots on a copy stream -> the captured step.
    A batch travels as ONE packed buffer (pack_batch: int32 ids | dense | labels) = one H2D copy;
    submit() also takes the three separate tensors (three copies, ids narrowed on the device).
    lookahead=True drives engine.step_ahead_graph: slot k's dense/labels train while slot k+1's
    ids are deduplicated, so two batches must have landed before a step starts (depth >= 3)."""

    def __init__(self, engine, depth=2, lookahead=False):
        self.lookahead = bool(lookahead)
        if self.lookahead:
            depth = max(depth, 3)
            if engine.graphs_ahead is None:
                engine.capture_ahead()
        elif getattr(engine, "graph", None) is None:
            engine.capture()
        self.started = False
        self.e = engine
        dev, G, B = engine.device, engine.G, engine.B
        self.depth = depth
        self.slots = [torch.empty(packed_nbytes(G, B, engine.widths), dtype=torch.uint8, device=dev) for _ in range(depth)]
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.ready = [torch.cuda.Event() for _ in range(depth)]
        self.free = [torch.cuda.Event() for _ in range(depth)]
        self.head = self.tail = 0

    def submit(self, *host_batch):
        """Enqueue the H2D copy of one batch (pinned host memory) on the copy stream:
        submit(packed) or submit(ids, dense, labels)."""
        k = self.head % self.depth
        with torch.cuda.stream(self.copy_stream):
            if self.head >= self.depth:
                self.copy_stream.wait_event(self.free[k])
            if len(host_batch) == 1:
                self.slots[k].copy_(host_batch[0], non_blocking=True)
            else:
                self.e._fill(self.slots[k], host_batch)
            self.ready[k].record(self.copy_stream)
        self.head += 1

    def run_next(self):
        """Run one step on the oldest submitted batch; returns the loss (device scalar)."""
        k = self.tail % self.depth
        main = torch.cuda.current_stream(self.e.device)
        main.wait_event(self.ready[k])
        if not self.lookahead:
            loss = self.e.step_graph(self.slots[k])
        else:
            if not self.started:
                self.e.prepare_packed(self.slots[k])
                self.started = True
            k1 = k
            if self.tail + 1 < self.head:  # the next batch was submitted: its ids are deduplicated now
                k1 = (self.tail + 1) % self.depth
                main.wait_event(self.ready[k1])
            loss = self.e.step_ahead_graph(self.slots[k1])
        self.free[k].record(main)
        self.tail += 1
        return loss


def _tower_error(lib):
    """Why the last failed tower call failed (b200_deepfm_last_error)."""
    return lib.b200_deepfm_last_error().decode("utf-8", "replace")


# What DeepFMPSEngine calls for its model on its tower kind (tower_calls): fwd_bwd, the one-call training step (None
# on tower="torch"); prologue / main, the tile tower's training step split in two (None elsewhere); forward,
# predict()'s tower; param_count(G), the flat parameter count; scratch(G, B), the floats the tile tower needs of
# `scratch`; regularized, whether the torch loss adds tower.regularization().
TowerCalls = collections.namedtuple("TowerCalls", "fwd_bwd prologue main forward param_count scratch regularized")


def tower_calls(lib, model, tower):
    tile = tower == "tile"
    return {
        "deepfm": TowerCalls(
            {"tile": lib.b200_deepfm_fwd_bwd_tile, "fused": lib.b200_deepfm_fwd_bwd,
             "mma": lib.b200_deepfm_fwd_bwd_mma}.get(tower),
            lib.b200_deepfm_tile_prologue if tile else None, lib.b200_deepfm_tile_main if tile else None,
            lib.b200_deepfm_forward_tile if tile else lib.b200_deepfm_forward,
            lib.b200_deepfm_param_count, lambda G, B: DEEPFM_TILE_SCRATCH, False),
        "dcn": TowerCalls(
            lib.b200_deepfm_dcn_fwd_bwd_tile if tile else None,
            lib.b200_deepfm_dcn_tile_prologue if tile else None, lib.b200_deepfm_dcn_tile_main if tile else None,
            lib.b200_deepfm_dcn_forward_tile,
            lib.b200_deepfm_dcn_param_count, lambda G, B: DEEPFM_DCN_SCRATCH, True),
        "wide_deep": TowerCalls(
            lib.b200_deepfm_wide_deep_fwd_bwd_tile if tile else None,
            lib.b200_deepfm_wide_deep_tile_prologue if tile else None,
            lib.b200_deepfm_wide_deep_tile_main if tile else None,
            lib.b200_deepfm_wide_deep_forward_tile,
            lib.b200_deepfm_param_count, lambda G, B: DEEPFM_TILE_SCRATCH, False),
        "xdeepfm": TowerCalls(
            lib.b200_deepfm_xdeepfm_fwd_bwd_tile if tile else None,
            lib.b200_deepfm_xdeepfm_tile_prologue if tile else None,
            lib.b200_deepfm_xdeepfm_tile_main if tile else None,
            lib.b200_deepfm_xdeepfm_forward_tile,
            lib.b200_deepfm_xdeepfm_param_count, lib.b200_deepfm_xdeepfm_scratch_floats, True),
    }[model]


def resolve_row_source(row_source, tower, n_shards, exchange, paired):
    """DeepFMPSEngine's row_source: "table" (the tower reads the table records) needs the tile tower and every
    record on this GPU in its own slab -- one shard, the direct exchange, unpaired tables."""
    assert row_source in ("auto", "table", "pull")
    table_ok = tower == "tile" and n_shards == 1 and exchange == "direct" and not paired
    if row_source == "auto":
        return "table" if table_ok else "pull"
    if row_source == "table" and not table_ok:
        raise ValueError('row_source="table" needs the tile tower, one shard, the direct exchange and unpaired tables')
    return row_source


class DeepFMPSEngine:
    def __init__(self, group, batch, lr=1e-3, init_std=0.01, seed=7, group_rows=GROUP_ROWS, deep_dim=DEEP_DIM,
                 init_rows=True, tower="tile", paired=None, exchange=None, id_transport="int32", row_source="auto",
                 model="deepfm"):
        """tower="tile": rows of 32 samples gathered once into shared memory, forward / backward / parameter
        gradients from the tile (csrc/deepfm_tower2.cu);
        tower="fused": round 1's hand-written CUDA tower (csrc/deepfm_tower.cu, three row gathers);
        tower="mma": its tensor-core variant (csrc/deepfm_tower_mma.cu, rows gathered once, 3xTF32 mma.sync);
        tower="torch": torch autograd over library kernels (kept for A/B measurements and tests).
        row_source="table": the tile tower reads each sample's rows straight from the table records
        (b200_deepfm_rows_t) and step() launches no row pull; "pull": the rows of the unique ids are first
        pulled into bet_w / bet_d.  "auto" takes "table" where it applies: tile tower, one shard, direct
        exchange, tables not paired.
        model="deepfm" (DeepFMTower), "dcn" (DCNTower, the dac_ctr Deep & Cross Network: csrc/dcn_tower.cu) or
        "wide_deep" (WideDeepTower, the dac_ctr Wide & Deep model: DeepFM without the FM term, on the tile tower's
        kernel without it) or "xdeepfm" (XDeepFMTower, the model the dac_ctr training script runs: Wide & Deep plus
        a CIN, csrc/xdeepfm_cin.cu); the dedup, the rows, the push and the pipelines are the same for all four.
        The models other than "deepfm" run on tower="tile" or "torch" and at most 38 id groups, "xdeepfm" on at
        least 2, and raise ValueError otherwise (the fused and mma towers compute DeepFM only)."""
        assert tower in ("tile", "fused", "mma", "torch")
        if model not in TOWERS:
            raise ValueError("model must be one of %s, not %r" % (sorted(TOWERS), model))
        if model != "deepfm" and tower not in ("tile", "torch"):
            raise ValueError('model="%s" runs on tower="tile" or "torch", not %r' % (model, tower))
        if model != "deepfm" and len(group_rows) > DEEPFM_TILE_MAXG:
            raise ValueError('model="%s" holds at most %d id groups, not %d' % (model, DEEPFM_TILE_MAXG, len(group_rows)))
        if model == "xdeepfm" and len(group_rows) < 2:
            raise ValueError('model="xdeepfm" needs at least 2 id groups (its CIN crosses fields), not %d'
                             % len(group_rows))
        self.model = model
        if tower == "tile" and len(group_rows) > DEEPFM_TILE_MAXG:
            tower = "fused"  # the tile tower holds at most 38 id groups in its shared-memory row
        self.tower_kind = tower
        self.calls = tower_calls(group.lib, model, tower)
        # paired=True: the deep (dim 8) and wide (dim 1) tables of an id group share one record
        # per id, so one request per id serves both (ps_kernels.cuh "Paired tables")
        # (default: when rows live on peer GPUs -- remote reads are bounded by requests in flight)
        if paired is None:
            paired = False
        self.paired = bool(paired) and deep_dim == 8
        # exchange="owner": rank-per-GPU groups bucket ids by owner and move everything over NVLink in
        # contiguous runs, the owner serves / updates its own shard (csrc/ps_exchange.cuh);
        # exchange="direct": kernels dereference the peer shard row by row.  The exchange moves at most
        # MAX_SEGS / 2 id groups (b200ps_xchg_create).
        if exchange is None:
            exchange = "owner" if (group.n_shards > 1 and len(group.local_shards) == 1 and deep_dim == 8
                                   and len(group_rows) <= MAX_SEGS // 2) else "direct"
        assert exchange in ("owner", "direct")
        self.exchange = exchange
        if exchange == "owner":
            self.paired = False
        self.row_source = resolve_row_source(row_source, tower, group.n_shards, exchange, self.paired)
        self.group = group
        self.B = int(batch)
        self.G = len(group_rows)
        self.D = deep_dim
        self.lr = lr
        dev = group.device
        self.device = dev
        G, B, D = self.G, self.B, self.D
        self.wide_names = ["group_%d_wide/embeddings:0" % i for i in range(G)]
        self.deep_names = ["group_%d_deep/embeddings:0" % i for i in range(G)]
        if self.paired:
            ids_ab = [group.register_pair(d, w, r) for d, w, r in zip(self.deep_names, self.wide_names, group_rows)]
            self.deep_ids = [a for a, _ in ids_ab]
            self.wide_ids = [b for _, b in ids_ab]
        else:
            self.wide_ids = [group.register_table(n, 1, "zero", r) for n, r in zip(self.wide_names, group_rows)]
            self.deep_ids = [group.register_table(n, D, "zero", r) for n, r in zip(self.deep_names, group_rows)]
        torch.manual_seed(seed)
        self.tower = TOWERS[model](G, D).to(dev)
        n_flat = int(self.calls.param_count(G))
        self.flat_params = torch.zeros(n_flat, dtype=torch.float32, device=dev)
        self.flat_grads = torch.zeros(n_flat, dtype=torch.float32, device=dev)
        self.flat_views = flatten_tower(self.tower, self.flat_params)
        # named_parameters order != flat order: keep both
        names = {id(p): n for n, p in self.tower.named_parameters()}
        self.params = [(names[id(p)], p) for p, _ in flat_order(self.tower)]
        from elasticdl_b200.common.hash_utils import string_to_id

        self.dense_ids = []
        for n, p in self.params:
            self.dense_ids.append(group.register_dense(n, tuple(p.shape), string_to_id(n, group.n_shards)))
        group.commit()
        # explicit N(0, init_std) initial rows, seed 7 (SURVEY 8d): set through the PS (set_rows)
        if init_rows and init_std > 0:
            gen = torch.Generator(device=dev).manual_seed(seed)
            for names, dim in ((self.wide_names, 1), (self.deep_names, D)):
                for n, r in zip(names, group_rows):
                    ids = torch.arange(r, device=dev)
                    if len(group.local_shards) != group.n_shards:
                        # multi-process: every rank initialises the rows it owns
                        mine = torch.zeros(r, dtype=torch.bool, device=dev)
                        for s in group.local_shards:
                            mine |= (ids % group.n_shards) == s
                        vals = torch.randn((r, dim), generator=gen, device=dev) * init_std
                        ids, vals = ids[mine], vals[mine]
                    else:
                        vals = torch.randn((r, dim), generator=gen, device=dev) * init_std
                    if ids.numel():
                        group.set_rows([(n, ids, vals)])
        # first-writer-wins dense init (PushModel)
        for s in range(group.n_shards):
            if s in group.local_shards and group.try_init(s):
                mine = [(n, p.detach()) for (n, p) in self.params if string_to_id(n, group.n_shards) == s]
                if mine:
                    group.set_dense(mine)
                group.finish_init(s, 0)
        # persistent buffers
        f32 = dict(dtype=torch.float32, device=dev)
        import ctypes as _ctb

        self.bounds = (_ctb.c_int64 * G)(*[int(r) for r in group_rows])  # id ranges: dedup by direct address
        self.ws = torch.zeros(group.lib.b200ps_unique_bounded_workspace(G, B, self.bounds), dtype=torch.uint8, device=dev)
        self._predict_state = None  # predict() dedups into its own workspace / plan (lazy)
        # id transport of the packed batches (pack_batch / HostFeeder / captured graphs): "int32" or "narrow"
        # (1 / 2 / 4 bytes per id by table size -- 72 instead of 152 bytes of ids per dac_ctr sample)
        self.id_transport = id_transport
        self.widths = id_widths(group_rows) if id_transport == "narrow" else [4] * G
        self._c_widths = (_ctb.c_int32 * G)(*self.widths)
        self.bet_w = torch.zeros((G * B, 1), **f32)
        self.bet_d = torch.zeros((G * B, D), **f32)
        self.act_w = torch.empty((G * B, 1), **f32)
        self.act_d = torch.empty((G * B, D), **f32)
        self.gsum_w = torch.zeros((G * B, 1), **f32)
        self.gsum_d = torch.zeros((G * B, D), **f32)
        # b200_deepfm.h: backward state + W1^T (fused / mma) | the tile tower's
        self.scratch = torch.empty(max(B * 44 + 16 * (N_DENSE + D * G), self.calls.scratch(G, B)), **f32)
        self.loss_buf = torch.zeros(1, **f32)
        # the loss of every step also lands in a ring of pinned host memory, written by a 1-thread kernel at the end
        # of the step (b200_deepfm_publish_loss): loss_host(k) reads step k's value after a synchronize, no D2H copy
        self.LOSS_RING = 256
        self.loss_ring = torch.zeros(self.LOSS_RING, dtype=torch.float32).pin_memory()
        self.loss_cursor = torch.zeros(1, dtype=torch.int32, device=self.device)
        self.logits_buf = torch.empty(B, **f32)
        self.zero_versions = [0] * group.n_shards

        self.loss_fn = torch.nn.BCEWithLogitsLoss()
        # everything addressed through one (uniq, inv, n_unique) triple is a "plan"; the lookahead
        # pipeline (prepare / step_ahead) alternates between two of them
        self.plans = [self._make_plan()]
        self.cur = 0
        self.side = None
        self.aux = None  # second stream of the branched step (see step())
        self.graph = None
        self.graphs_ahead = None
        if self.exchange == "owner":
            group.xchg_create(G, B, self.deep_ids, self.wide_ids)
        self.steps = 0

    _PLAN_ATTRS = ("uniq", "inv", "n_unique", "pull_segs", "push_segs", "pull_pair", "push_pair", "tower_args",
                   "tower_rows", "pull_names", "push_names")

    def _make_plan(self):
        dev, G, B = self.device, self.G, self.B
        self.uniq = torch.empty(G * B, dtype=torch.int64, device=dev)
        self.inv = torch.empty(G * B, dtype=torch.int32, device=dev)
        self.n_unique = torch.empty(G, dtype=torch.int32, device=dev)
        self._build_segs()
        return {k: getattr(self, k) for k in self._PLAN_ATTRS}

    def _use(self, p):
        self.__dict__.update(self.plans[p])
        self.cur = p

    def _seg_items(self, ids_tab, rows, dim):
        B = self.B
        return [(ids_tab[t], B, self.uniq[t * B:(t + 1) * B], self.n_unique[t:t + 1], rows[t * B:(t + 1) * B])
                for t in range(self.G)]

    def _build_segs(self):
        g = self.group
        # all 2G tables in ONE flat launch when they fit (csrc/ps_flat.cuh), else one launch per family
        wide_pull, deep_pull = self._seg_items(self.wide_ids, self.bet_w, 1), self._seg_items(self.deep_ids, self.bet_d, self.D)
        wide_push, deep_push = self._seg_items(self.wide_ids, self.gsum_w, 1), self._seg_items(self.deep_ids, self.gsum_d, self.D)
        from elasticdl_b200 import _lib as _l0

        if 2 * self.G <= _l0.MAX_SEGS:
            self.pull_names, self.push_names = ("pull",), ("push",)
            self.pull_segs = [g.make_segs(deep_pull + wide_pull)]
            self.push_segs = [g.make_segs(deep_push + wide_push)]
        else:
            self.pull_names, self.push_names = ("pull_wide", "pull_deep"), ("push_wide", "push_deep")
            self.pull_segs = [g.make_segs(wide_pull), g.make_segs(deep_pull)]
            self.push_segs = [g.make_segs(wide_push), g.make_segs(deep_push)]
        self.pull_dense_segs = g.make_segs([(tid, 0, None, None, p) for tid, (_, p) in zip(self.dense_ids, self.params)])
        import ctypes as _ct
        from elasticdl_b200 import _lib as _l

        half, B = _l.MAX_SEGS // 2, self.B

        def pair_plan(rows_a, rows_b):
            items = self._seg_items(self.deep_ids, rows_a, self.D)
            plan = []
            for i in range(0, self.G, half):
                arr, n = g.make_segs(items[i:i + half])
                ptrs = (_ct.c_void_p * n)(*[rows_b[t * B:(t + 1) * B].data_ptr() for t in range(i, min(i + half, self.G))])
                plan.append((arr, ptrs, n))
            return plan

        self.pull_pair = pair_plan(self.bet_d, self.bet_w)
        self.push_pair = pair_plan(self.gsum_d, self.gsum_w)
        grad_views = [self.flat_grads[off:off + n] for off, n in self.flat_views]
        self.push_dense_segs = g.make_segs([(tid, 0, None, None, gv) for tid, gv in zip(self.dense_ids, grad_views)])
        from elasticdl_b200._lib import DeepFMArgs

        a = DeepFMArgs()
        a.G, a.B = self.G, self.B
        a.inv, a.n_unique = self.inv.data_ptr(), self.n_unique.data_ptr()
        a.bet_wide, a.bet_deep = self.bet_w.data_ptr(), self.bet_d.data_ptr()
        a.params, a.grads = self.flat_params.data_ptr(), self.flat_grads.data_ptr()
        a.gsum_wide, a.gsum_deep = self.gsum_w.data_ptr(), self.gsum_d.data_ptr()
        a.loss, a.logits, a.scratch = self.loss_buf.data_ptr(), self.logits_buf.data_ptr(), self.scratch.data_ptr()
        self.tower_args = a
        self.tower_rows = None
        if self.row_source == "table":
            self.tower_rows = self._table_rows()
            a.rows = _ct.pointer(self.tower_rows)

    def _table_rows(self):
        """b200_deepfm_rows_t of the current plan: its unique ids and the record slabs of the G deep and G wide
        tables (one shard)."""
        import ctypes as _ct
        from elasticdl_b200._lib import DeepFMRows

        g, r = self.group, DeepFMRows()
        r.uniq = self.uniq.data_ptr()
        for fam, tids, bases in (("deep", self.deep_ids, r.deep_base), ("wide", self.wide_ids, r.wide_base)):
            layout = set()
            for k, tid in enumerate(tids):
                base, stride, off, rows = _ct.POINTER(_ct.c_float)(), _ct.c_int64(), _ct.c_int64(), _ct.c_int64()
                check(g.lib.b200ps_table_rows_ptr(g._h, tid, 0, _ct.byref(base), _ct.byref(stride), _ct.byref(off),
                                                  _ct.byref(rows)))
                bases[k] = _ct.cast(base, _ct.c_void_p).value
                layout.add((stride.value, off.value))
            assert len(layout) == 1, layout  # one record layout per family: same dim, same optimizer
            (stride, off), = layout
            setattr(r, fam + "_stride", stride)
            setattr(r, fam + "_param_off", off)
        return r

    def step(self, ids, dense, labels, ev=None, after_tower=None):
        """ids int64 [G, B] (group-major), dense fp32 [B, 13], labels fp32 [B] -- all on the device.
        Returns the loss (device scalar).  ev: optional dict name -> list; CUDA-event pairs are
        recorded around the named PS kernels on the launching stream."""
        g, lib, h = self.group, self.group.lib, self.group._h
        G, B, D = self.G, self.B, self.D
        st = g._stream()

        def mark(name):
            if ev is None:
                return None
            e = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            ev.setdefault(name, []).append(e)
            e[0].record()
            return e

        def done(e):
            if e is not None:
                e[1].record()

        # Branches: the step has six launch-bound kernels (pull_dense, tower prologue, push_begin, push_dense,
        # push_end) that do not depend on the row kernels beside them.  With
        # `branch` they run on a second stream -- inside a captured graph these become parallel branches --
        # while the main stream carries unique -> pull -> tower -> push rows:
        #   aux:  pull_dense -> push_begin -> tower prologue  | joined before the tower
        #   aux:  push_dense                                   | beside the row push, joined before push_end
        branch = self.tower_kind == "tile" and ev is None
        main = torch.cuda.current_stream(self.device)
        if branch:
            if self.aux is None:
                self.aux = torch.cuda.Stream(device=self.device)
            a = self.tower_args
            a.dense, a.labels = dense.data_ptr(), labels.data_ptr()
        # (2) unique ids per group; wide and deep tables of a group share them
        if ids is not None:
            e = mark("unique")
            self._unique_into(ids)
            done(e)
        # (1) pull dense parameters straight into the tower's tensors
        if branch:
            self.aux.wait_stream(main)  # n_unique of this batch, parameters of the previous step
            with torch.cuda.stream(self.aux):
                arr, n = self.pull_dense_segs
                check(lib.b200ps_pull_dense(h, arr, n, g._stream()))
                self._tower_call(self.calls.prologue, a, g._stream())
                ev_prep = torch.cuda.Event()
                ev_prep.record(self.aux)  # the tower waits for this, not for push_begin behind it
                g.push_begin(self.lr, self.zero_versions)
                ev_begin = torch.cuda.Event()
                ev_begin.record(self.aux)
        else:
            arr, n = self.pull_dense_segs
            check(lib.b200ps_pull_dense(h, arr, n, st))
        # (3) pull the unique rows of all 76 tables (row_source "table": the tower reads them from the tables)
        if self.row_source == "pull":
            if self.exchange == "owner":
                e = mark("pull_exchange")
                check(lib.b200ps_xchg_pull(h, self.uniq.data_ptr(), self.n_unique.data_ptr(), self.bet_d.data_ptr(),
                                           self.bet_w.data_ptr(), st))
                done(e)
            elif self.paired:
                e = mark("pull_pair")
                for arr, ptrs, n in self.pull_pair:
                    check(lib.b200ps_pull_rows_pair(h, arr, ptrs, n, st))
                done(e)
            else:
                for name, (arr, n) in zip(self.pull_names, self.pull_segs):
                    e = mark(name)
                    check(lib.b200ps_pull_rows(h, arr, n, st))
                    done(e)
        if branch:
            main.wait_event(ev_prep)
            self._tower_call(self.calls.main, a, st)
            loss = self.loss_buf
            dense_segs = self.push_dense_segs
        elif self.calls.fwd_bwd is not None:
            # (4-6) gather + tower forward/backward + per-unique-id gradient sums: three launches
            e_t = mark("tower_fwd_bwd")
            a = self.tower_args
            a.dense, a.labels = dense.data_ptr(), labels.data_ptr()
            self._tower_call(self.calls.fwd_bwd, a, st)
            done(e_t)
            loss = self.loss_buf
            dense_segs = self.push_dense_segs
        else:
            loss, dense_segs = self._torch_tower(dense, labels, mark, done, st)
        if after_tower is not None:
            after_tower()  # lookahead pipeline: the next batch's dedup forks here (beside the push)
        # (7) push: one ApplyGradients per shard
        if branch:
            main.wait_event(ev_begin)  # this push's lr / Adam alpha / step (k_push_begin ran on the second stream)
            self.aux.wait_stream(main)
            with torch.cuda.stream(self.aux):
                arr, n = dense_segs
                check(lib.b200ps_push_dense(h, arr, n, g._stream()))
                self._publish_loss(loss, g._stream())
        else:
            g.push_begin(self.lr, self.zero_versions)
            arr, n = dense_segs
            check(lib.b200ps_push_dense(h, arr, n, st))
            self._publish_loss(loss, st)
        if self.exchange == "owner":
            e = mark("push_exchange")
            check(lib.b200ps_xchg_push(h, self.gsum_d.data_ptr(), self.gsum_w.data_ptr(), st))
            done(e)
        elif self.paired:
            e = mark("push_pair")
            for arr, ptrs, n in self.push_pair:
                check(lib.b200ps_push_rows_pair(h, arr, ptrs, n, st))
            done(e)
        else:
            for name, (arr, n) in zip(self.push_names, self.push_segs):
                e = mark(name)
                check(lib.b200ps_push_rows(h, arr, n, st))
                done(e)
        if branch:
            main.wait_stream(self.aux)
        g.push_end(sync=False)
        self.steps += 1
        return loss.detach().reshape(())

    def _tower_call(self, fn, args, st):
        """One tower entry point on `args` (DeepFMArgs); RuntimeError with its return code and
        b200_deepfm_last_error if it fails."""
        rc = fn(ctypes.byref(args), st)
        if rc:
            raise RuntimeError("%s failed (%d): %s" % (fn.__name__, rc, _tower_error(self.group.lib)))

    def _publish_loss(self, loss, st):
        if loss is not self.loss_buf:  # torch tower: its loss tensor is not persistent
            self.loss_buf.copy_(loss.detach().reshape(1))
        rc = self.group.lib.b200_deepfm_publish_loss(self.loss_buf.data_ptr(), self.loss_ring.data_ptr(), self.LOSS_RING,
                                                     self.loss_cursor.data_ptr(), st)
        if rc:
            raise RuntimeError("b200_deepfm_publish_loss failed (%d): %s" % (rc, _tower_error(self.group.lib)))

    def loss_host(self, step_index):
        """Loss of step `step_index` (0-based count of steps run by this engine) from the host ring; valid once
        the device has finished that step (synchronize / event) and for the last LOSS_RING steps."""
        return float(self.loss_ring[step_index % self.LOSS_RING])

    def _unique_into(self, ids):
        """tf.unique per id group into the current plan, on the current stream (the library's default grid:
        blocks_per_sm = 0)."""
        g = self.group
        if ids.dtype == torch.uint8:  # the id region of a packed batch with per-group widths
            check(g.lib.b200ps_unique_packed(g._h, ids.data_ptr(), self._c_widths, self.G, self.B, self.bounds,
                                             self.uniq.data_ptr(), self.inv.data_ptr(), self.n_unique.data_ptr(),
                                             self.ws.data_ptr(), self.ws.numel(), 0, g._stream()))
            return
        check(g.lib.b200ps_unique_bounded_ex(g._h, ids.data_ptr(), 1 if ids.dtype == torch.int32 else 0, self.G, self.B,
                                             self.bounds, self.uniq.data_ptr(), self.inv.data_ptr(),
                                             self.n_unique.data_ptr(), self.ws.data_ptr(), self.ws.numel(), 0,
                                             g._stream()))

    # ------------------------------------------------------------------ lookahead pipeline
    def _ensure_plans(self):
        if len(self.plans) == 1:
            cur = self.cur
            self.plans.append(self._make_plan())
            self._use(cur)
            self.side = torch.cuda.Stream(device=self.device)

    def prepare(self, ids):
        """Start the lookahead pipeline: deduplicate the FIRST batch's ids.  Afterwards every
        step_ahead(dense_i, labels_i, ids_{i+1}) trains on batch i while the ids of batch i+1 are
        deduplicated on a second stream (the dedup only depends on the input batch, like the
        reference's dataset.prefetch(1) work, elasticdl/python/worker/worker.py:334)."""
        self._ensure_plans()
        self._unique_into(ids)

    def step_ahead(self, dense, labels, next_ids, ev=None):
        """One training step on the prepared batch + the dedup of `next_ids` (int64 or int32 [G, B],
        device) overlapped on the side stream.  Same kernels, same results as step()."""
        if len(self.plans) != 2:
            raise RuntimeError("call prepare(first_ids) before step_ahead")
        main = torch.cuda.current_stream(self.device)
        p = self.cur

        def fork():
            # The dedup of the next batch runs beside the PUSH of this one: the push kernels are light
            # (48 registers, < 1 KB of shared memory) and share the SMs with the persistent dedup blocks,
            # whereas the tower's CTAs need the whole register file of an SM and would simply wait for
            # the dedup to finish (forking at the start of the step hid only a quarter of it).
            self.side.wait_stream(main)  # the other plan's buffers were last read by the previous step
            self._use(1 - p)
            with torch.cuda.stream(self.side):
                self._unique_into(next_ids)
            self._use(p)

        loss = self.step(None, dense, labels, ev=ev, after_tower=fork)
        main.wait_stream(self.side)  # join
        self._use(1 - p)
        return loss

    def capture_ahead(self):
        """Two CUDA graphs (one per plan parity) of step_ahead over two static PACKED batch buffers
        S[0], S[1] (pack_batch layout): graph p trains on the dense / labels of S[p] (its ids were
        deduplicated into plan p by the previous step) while it deduplicates the ids of S[1 - p]."""
        if self.tower_kind == "torch":
            raise RuntimeError("graph capture needs the fused tower (torch autograd allocates)")
        dev, G, B = self.device, self.G, self.B
        self._ensure_plans()
        self.s_packed = [torch.zeros(packed_nbytes(G, B, self.widths), dtype=torch.uint8, device=dev) for _ in range(2)]
        views = [packed_views(b, G, B, self.widths) for b in self.s_packed]
        torch.cuda.synchronize(dev)
        start, steps = self.cur, self.steps
        self.graphs_ahead = [None, None]
        for p in (start, 1 - start):
            assert self.cur == p
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                self.step_ahead(views[p][1], views[p][2], views[1 - p][0])
            self.graphs_ahead[p] = gr
        self._use(start)
        self.steps = steps  # capture does not execute
        return self.graphs_ahead

    def _fill(self, dst, batch):
        """dst: static packed buffer; batch: (packed,) or (ids, dense, labels) -- device or pinned host.  Separate
        ids are range-checked against the widths first (check_id_widths); a packed buffer is already narrowed."""
        if len(batch) == 1:
            dst.copy_(batch[0], non_blocking=True)
            return
        check_id_widths(batch[0], self.widths)
        views = packed_views(dst, self.G, self.B, self.widths)
        if views[0].dtype == torch.int32:  # an unpadded int32 [G, B] id region: copy into the views
            for d, src in zip(views, batch):
                d.copy_(src, non_blocking=True)
        else:  # separate tensors into a narrow or padded layout: pack on the device (compatibility path)
            ids, dense, labels = batch
            dst.copy_(pack_batch(ids.to(self.device), dense.to(self.device), labels.to(self.device), widths=self.widths),
                      non_blocking=True)

    def prepare_packed(self, *batch):
        """Lookahead through the captured graphs: load the FIRST batch and deduplicate its ids."""
        if self.graphs_ahead is None:
            self.capture_ahead()
        self._fill(self.s_packed[self.cur], batch)
        self._unique_into(packed_views(self.s_packed[self.cur], self.G, self.B, self.widths)[0])

    def step_ahead_graph(self, *next_batch):
        """step_ahead through the captured graphs: trains on the batch loaded by the previous call (or
        prepare_packed) while `next_batch` -- (packed,) or (ids, dense, labels) -- is loaded and its ids
        are deduplicated.  Inputs may be pinned-host or device tensors."""
        self._fill(self.s_packed[1 - self.cur], next_batch)
        self.graphs_ahead[self.cur].replay()
        self._use(1 - self.cur)
        self.steps += 1
        return self.loss_buf.reshape(())

    # ------------------------------------------------------------------ CUDA graph
    def capture(self):
        """Capture one whole step into a CUDA graph.  Every buffer the step touches is persistent, so
        the graph replays on new inputs copied into the static packed input buffer.  lr is baked in:
        re-capture to change it."""
        if self.tower_kind == "torch":
            raise RuntimeError("graph capture needs the fused tower (torch autograd allocates)")
        dev, G, B = self.device, self.G, self.B
        self.s_one = torch.zeros(packed_nbytes(G, B, self.widths), dtype=torch.uint8, device=dev)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.step(*packed_views(self.s_one, G, B, self.widths))
        self.steps -= 1  # capture does not execute
        return self.graph

    def step_graph(self, *batch):
        """Same step through the captured graph; batch = (packed,) or (ids, dense, labels), pinned-host
        or device tensors."""
        self._fill(self.s_one, batch)
        self.graph.replay()
        self.steps += 1
        return self.loss_buf.reshape(())

    def host_feeder(self, depth=2, lookahead=False):
        """Input pipeline for host-resident batches: H2D copies run on a side stream into
        `depth` staging slots and overlap the previous step's kernels (the reference prefetches
        one batch too: dataset.prefetch(1), elasticdl/python/worker/worker.py:334)."""
        return HostFeeder(self, depth, lookahead)

    def _torch_tower(self, dense, labels, mark, done, st):
        """Steps (4)-(6) with torch autograd over library kernels (A/B reference for the fused tower)."""
        g, lib, h = self.group, self.group.lib, self.group._h
        G, B, D = self.G, self.B, self.D
        check(lib.b200ps_gather_rows(h, self.bet_w.data_ptr(), self.inv.data_ptr(), G, B, 1, self.act_w.data_ptr(), st))
        check(lib.b200ps_gather_rows(h, self.bet_d.data_ptr(), self.inv.data_ptr(), G, B, D, self.act_d.data_ptr(), st))
        e_t = mark("tower_fwd_bwd")
        act_w = self.act_w.detach().requires_grad_(True)
        act_d = self.act_d.detach().requires_grad_(True)
        wide = act_w.view(G, B).t()
        deep = act_d.view(G, B, D).permute(1, 0, 2)
        logits = self.tower(dense, wide, deep)
        loss = self.loss_fn(logits, labels)
        if self.calls.regularized:
            loss = loss + self.tower.regularization()
        plist = [p for _, p in self.params]
        grads = torch.autograd.grad(loss, plist + [act_w, act_d])
        gw, gd = grads[-2].contiguous(), grads[-1].contiguous()
        done(e_t)
        check(lib.b200ps_segment_sum(h, gw.data_ptr(), self.inv.data_ptr(), G, B, 1, self.gsum_w.data_ptr(), st))
        e = mark("segment_sum_deep")
        check(lib.b200ps_segment_sum(h, gd.data_ptr(), self.inv.data_ptr(), G, B, D, self.gsum_d.data_ptr(), st))
        done(e)
        self._dense_grads = [gr.contiguous() for gr in grads[:-2]]
        return loss, g.make_segs([(tid, 0, None, None, gr) for tid, gr in zip(self.dense_ids, self._dense_grads)])

    def predict(self, ids, dense):
        """Forward only (logits) through the PS: unique -> pull -> fused tower forward.  Uses its own
        dedup workspace and (uniq, inv, n_unique) plan, so a prepared lookahead batch stays intact."""
        g, lib, h = self.group, self.group.lib, self.group._h
        st = g._stream()
        if self._predict_state is None:
            cur = self.cur
            ws = torch.zeros(lib.b200ps_unique_workspace(self.G, self.B), dtype=torch.uint8, device=self.device)
            plan = self._make_plan()
            # predict() pulls its rows: with no push after it, the pull is what marks rows as created on first
            # read (embedding_table.go:41-58)
            plan["tower_args"].rows = None
            self._use(cur)
            self._predict_state = (ws, plan)
        ws, plan = self._predict_state
        saved = {k: getattr(self, k) for k in self._PLAN_ATTRS}
        self.__dict__.update(plan)
        try:
            arr, n = self.pull_dense_segs
            check(lib.b200ps_pull_dense(h, arr, n, st))
            ids = ids.to(torch.int64)
            check(lib.b200ps_unique(h, ids.data_ptr(), self.G, self.B, self.uniq.data_ptr(), self.inv.data_ptr(),
                                    self.n_unique.data_ptr(), ws.data_ptr(), ws.numel(), st))
            for arr, n in self.pull_segs:
                check(lib.b200ps_pull_rows(h, arr, n, st))
            a = self.tower_args
            a.dense = dense.data_ptr()
            self._tower_call(self.calls.forward, a, st)
        finally:
            self.__dict__.update(saved)
        return self.logits_buf

    def evaluate(self, ids, dense, labels, metrics):
        """predict() on one batch, then metrics.update_evaluation_metrics({"logits": logits, "probs":
        sigmoid(logits)}, labels) (an EvaluationMetrics, e.g. of eval_metrics_fn()).  Pushes nothing.  Returns the
        logits [B] on the device (the buffer predict() returns: the next predict() or step overwrites it)."""
        logits = self.predict(ids, dense)
        metrics.update_evaluation_metrics({"logits": logits, "probs": torch.sigmoid(logits)}, labels)
        return logits

    def kernel_report(self, ev, uniq_per_step, opt_slots=2):
        """Average CUDA-event duration and algorithmic GB/s per named PS kernel.
        Algorithmic bytes (SURVEY.md 8d): pull U*(8+8D); push U*(8+4D+(1+S)*8D); segment_sum
        k*(4+4D)+U*4D; unique k*(8+4)+U*8 (ids in, inverse out, unique ids out)."""
        D, k = self.D, self.G * self.B
        out = {}
        for name, pairs in ev.items():
            ms = [a.elapsed_time(b) for a, b in pairs]
            U = sum(uniq_per_step) / max(len(uniq_per_step), 1)
            nbytes = {
                "pull_wide": U * (8 + 8 * 1), "pull_deep": U * (8 + 8 * D),
                "pull": U * (8 + 8 * 1) + U * (8 + 8 * D),
                "push": U * (8 + 4 * 1 + (1 + opt_slots) * 8 * 1) + U * (8 + 4 * D + (1 + opt_slots) * 8 * D),
                # tower: per (sample, group) one rank read + one deep row + one wide value gathered, the
                # embedding gradient scattered back (reduced per unique id), + the dense inputs / labels
                # (row_source "table": + the low word of the row's id); the same for DeepFM and DCN, whose cross
                # network reads the tile's rows a second time from shared memory only
                "tower_fwd_bwd": k * (4 + 4 * D + 4 + (4 if self.row_source == "table" else 0)) + U * (4 * D + 4)
                + self.B * 4 * (N_DENSE + 1),
                "pull_pair": U * (8 + 8 * D + 8 * 1), "pull_exchange": U * (8 + 8 * D + 8 * 1),
                "push_exchange": U * (8 + 4 * D + 4 * 1 + (1 + opt_slots) * 8 * (D + 1)),
                "push_pair": U * (8 + 4 * D + 4 * 1 + (1 + opt_slots) * 8 * (D + 1)),
                "push_wide": U * (8 + 4 * 1 + (1 + opt_slots) * 8 * 1),
                "push_deep": U * (8 + 4 * D + (1 + opt_slots) * 8 * D),
                "segment_sum_deep": k * (4 + 4 * D) + U * 4 * D,
                "unique": k * 12 + U * 8,
            }.get(name)
            avg = sum(ms) / len(ms)
            out[name] = {"ms": avg, "launches": len(ms)}
            if nbytes:
                out[name]["bytes"] = nbytes
                out[name]["gbs"] = nbytes / (avg * 1e-3) / 1e9
        return out

    @staticmethod
    def algorithmic_bytes(n_unique_total, opt_slots=2, deep_dim=DEEP_DIM):
        """SURVEY.md section 8d per-unit figures, fp32 rows, int64 ids:
        pull U*(8 + 4D + 4D); sparse push U*(8 + 4D + (1+S)*8D), for D in {1, deep_dim}."""
        pull = sum(n_unique_total * (8 + 8 * d) for d in (1, deep_dim))
        push = sum(n_unique_total * (8 + 4 * d + (1 + opt_slots) * 8 * d) for d in (1, deep_dim))
        return pull, push


class DeepFMLayersModel(torch.nn.Module):
    """The model a model_zoo job runs through the drop-in API (model_zoo/dac_ctr/deepfm_model.py:33-109):
    one elasticdl Embedding layer per feature group and family -- G deep layers (dim 8) and G wide layers
    (dim 1), each looked up with its own id tensor -- in front of DeepFMTower in eager torch.
    forward(features): features = {"dense": [B, 13] float32, "ids_0" .. "ids_{G-1}": [B] int64}.
    Carries `.optimizer` / `.loss` as ParameterServerTrainer expects (worker/ps_trainer.py)."""

    def __init__(self, group_rows=GROUP_ROWS, deep_dim=DEEP_DIM, lr=1e-3, initializer="zero"):
        super().__init__()
        from elasticdl_b200.layers import Embedding

        G = len(group_rows)
        self.deep = torch.nn.ModuleList(
            [Embedding(deep_dim, input_dim=r, embeddings_initializer=initializer, name="deep_%d" % g)
             for g, r in enumerate(group_rows)])
        self.wide = torch.nn.ModuleList(
            [Embedding(1, input_dim=r, embeddings_initializer=initializer, name="wide_%d" % g)
             for g, r in enumerate(group_rows)])
        self.tower = DeepFMTower(G, deep_dim)
        self.optimizer = torch.optim.Adam(self.tower.parameters(), lr=lr)
        bce = torch.nn.BCEWithLogitsLoss()
        self.loss = lambda labels, logits: bce(logits, labels)

    @staticmethod
    def features_of(ids, dense):
        """ids [G, B] int64 -> the per-feature dict (row views of the one array, as a dataset's
        feature columns are)."""
        f = {"dense": dense}
        for g in range(ids.shape[0]):
            f["ids_%d" % g] = ids[g]
        return f

    def forward(self, features):
        G = len(self.deep)
        deep = torch.stack([self.deep[g](features["ids_%d" % g]) for g in range(G)], 1)  # [B, G, D]
        wide = torch.cat([self.wide[g](features["ids_%d" % g]) for g in range(G)], 1)    # [B, G]
        return self.tower(features["dense"], wide, deep)
