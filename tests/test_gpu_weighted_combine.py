"""GPU tests of the weighted pooled lookup (Embedding's sparse_weights, EmbeddingBag's per_sample_weights): the
reference's literal vectors (feature_column_test.py:75-111, :172-270), random shapes against the float64 oracle's
bound (tests/weighted_oracle.py), unit weights against the unweighted kernels bit for bit, determinism, torch's own
F.embedding_bag, the refusals, and a model trained through ModelHandler and ParameterServerTrainer."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sparse_oracle as so
from tests import weighted_oracle as wo
from tests.test_gpu_sparse_combine import CASES, _random_case

pytestmark = pytest.mark.gpu
COMBINERS = ["sum", "mean", "sqrtn"]
ADAM = ("Adam", "learning_rate=0.01;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")


def _layer(dim, combiner, lookup, input_dim=None):
    from elasticdl_b200.layers import Embedding

    layer = Embedding(dim, input_dim=input_dim, combiner=combiner)
    layer.set_lookup_embedding_func(lookup)
    return layer


def _coo(ids, values):
    ids = torch.as_tensor(ids)
    idx = torch.stack([torch.arange(ids.shape[0]).repeat_interleave(ids.shape[1]),
                       torch.arange(ids.shape[1]).repeat(ids.shape[0])])
    return torch.sparse_coo_tensor(idx, torch.as_tensor(values).reshape(-1), tuple(ids.shape)).cuda()


def test_feature_column_weighted_output():
    one_hot = lambda name, ids: (torch.arange(8, device=ids.device)[None, :] == (ids[:, None] % 8)).float()
    layer = _layer(8, "sum", one_hot, input_dim=128)
    out = layer(_coo([[2, 6, 5], [3, 1, 1]], [[2, 6, 5], [3, 1, 1]]),
                _coo([[2, 6, 5], [3, 1, 1]], [[0.33, 5.0, 1.024], [2.048, 0.5, 1.0]]))
    want = torch.tensor([[0.0, 0.0, 0.33, 0.0, 0.0, 1.024, 5.0, 0.0],
                         [0.0, 1.5, 0.0, 2.048, 0.0, 0.0, 0.0, 0.0]], dtype=torch.float32)
    assert torch.equal(out.cpu(), want)


GRAD_IDS = [[1, 2], [10, 10], [6, 3], [10, 2]]
GRAD_W = [[0.3, 0.6], [0.1, 0.2], [0.8, 0.1], [0.9, 0.6]]


@pytest.mark.parametrize("combiner", COMBINERS)
def test_feature_column_weighted_gradients(combiner):
    """feature_column_test.py:172-270, summed per unique id (1, 2, 10, 6, 3) as our BET gradient is."""
    from tests.test_oracle_weighted_combine import GRAD_OCC

    fill = lambda name, ids: ids.float().unsqueeze(1).repeat(1, 8)
    layer = _layer(8, combiner, fill, input_dim=128)
    layer.set_tape(True)
    out = layer(_coo(GRAD_IDS, GRAD_IDS), _coo(GRAD_IDS, GRAD_W))
    bet, ids = layer.embedding_and_ids[0]
    assert ids.tolist() == [1, 2, 10, 6, 3]
    (g,) = torch.autograd.grad(out.sum(), [bet])
    _, idx = so.unique_first(np.array(GRAD_IDS).reshape(-1))
    want = np.zeros(5)
    np.add.at(want, idx, GRAD_OCC[combiner])
    np.testing.assert_allclose(g.cpu().numpy(), np.repeat(want[:, None], 8, axis=1), rtol=2e-6)


def _prep_pull(rows, cols, vals, B, L, table, vdtype=torch.int64):
    from elasticdl_b200 import ops

    sp = torch.sparse_coo_tensor(torch.tensor(np.stack([rows, cols])), torch.tensor(vals).to(vdtype), (B, L)).cuda()
    sp = sp.coalesce()
    assert torch.equal(sp.indices()[0].cpu(), torch.tensor(rows))  # row-major input: coalesce keeps the entry order
    ids, ws = ops.sparse_prep(sp.indices()[0], sp.values(), B, table.shape[1])
    uniq, inv, n = ops.unique(ids)
    u = uniq[: int(n.item())]
    return table[u % table.shape[0]].detach().clone(), inv, ws, sp.values().numel(), u


@pytest.mark.parametrize("B,mean_len,dim,long_row,vdtype", CASES + [(32768, 10, 3, 600, torch.int64)])
@pytest.mark.parametrize("bounded", [True, False])
def test_random_against_oracle(B, mean_len, dim, long_row, vdtype, bounded):
    from elasticdl_b200 import ops

    rng = np.random.default_rng(B + dim + long_row + 1)
    rows, cols, vals, L = _random_case(rng, B, mean_len, long_row)
    n_rows = 1000 if bounded else 1 << 40  # hashed: ids anywhere in int64, looked up modulo the table
    if not bounded:
        vals = np.where(vals >= 0, vals * 1_000_003 % n_rows, vals)
    table = torch.randn(1000, dim, device="cuda")
    tab = table.double().cpu().numpy()
    w = rng.uniform(0.25, 2.0, rows.size).astype(np.float32)
    wt = torch.tensor(w, device="cuda")
    bet0, inv, ws, nnz, uniq = _prep_pull(rows, cols, vals, B, L, table, vdtype)
    for combiner in COMBINERS:
        bet = bet0.clone().requires_grad_(True)
        wl = wt.clone().requires_grad_(combiner == "sum")
        out = ops.SparseCombine.apply(bet, inv, ws, B, nnz, combiner, dim, wl)
        want, ouniq, obet = wo.lookup_weighted(rows, vals, w, B, lambda u: tab[u % 1000], combiner)
        np.testing.assert_array_equal(uniq.cpu().numpy(), ouniq)
        err = np.abs(out.detach().double().cpu().numpy() - want)
        bd = wo.bound_weighted(rows, vals, w, B, np.abs(obet), combiner)
        assert (err <= bd).all(), (combiner, float((err - bd).max()))
        G = torch.randn(B, dim, device="cuda")
        Gd = G.double().cpu().numpy()
        grads = torch.autograd.grad(out, [bet, wl] if combiner == "sum" else [bet], G)
        gw = wo.grad_bet_weighted(rows, vals, w, B, len(ouniq), Gd, combiner)
        gb = wo.grad_bound_weighted(rows, vals, w, B, len(ouniq), np.abs(Gd), combiner)
        gerr = np.abs(grads[0].double().cpu().numpy() - gw)
        assert (gerr <= gb).all(), (combiner, float((gerr - gb).max()))
        if combiner == "sum":
            ww = wo.grad_weights(rows, vals, B, obet, Gd)
            wb = wo.grad_weights_bound(rows, vals, B, np.abs(obet), np.abs(Gd))
            werr = np.abs(grads[1].double().cpu().numpy() - ww)
            assert (werr <= wb).all(), float((werr - wb).max())
            again = torch.autograd.grad(ops.SparseCombine.apply(bet, inv, ws, B, nnz, combiner, dim, wl), [wl], G)
            assert torch.equal(again[0], grads[1])  # no atomics: the same bits
        assert torch.equal(ops.SparseCombine.apply(bet, inv, ws, B, nnz, combiner, dim, wl), out)


@pytest.mark.parametrize("dim", [1, 3, 8, 64])
@pytest.mark.parametrize("combiner", COMBINERS)
def test_unit_weights_give_the_unweighted_bits(dim, combiner):
    """Forward on any input; the BET gradient on distinct ids, where each unique row gets one addend and the segment
    sum's atomics cannot reorder anything.  Rows of 1, 300 and 700 entries: one, two and three combine pieces."""
    from elasticdl_b200 import ops

    rng = np.random.default_rng(dim)
    lens = np.array([1, 300, 0, 5, 700, 2, 0, 40])
    B = lens.size
    rows = np.repeat(np.arange(B), lens)
    cols = np.concatenate([np.arange(n) for n in lens])
    table = torch.randn(5000, dim, device="cuda")
    for vals in (rng.integers(0, 60, rows.size), rng.permutation(5000)[: rows.size]):
        bet0, inv, ws, nnz, _ = _prep_pull(rows, cols, vals, B, int(lens.max()), table)
        ones = torch.ones(nnz, device="cuda")
        G = torch.randn(B, dim, device="cuda")
        bet = bet0.clone().requires_grad_(True)
        out = ops.SparseCombine.apply(bet, inv, ws, B, nnz, combiner, dim)
        (g,) = torch.autograd.grad(out, [bet], G)
        bet_w = bet0.clone().requires_grad_(True)
        out_w = ops.SparseCombine.apply(bet_w, inv, ws, B, nnz, combiner, dim, ones)
        (g_w,) = torch.autograd.grad(out_w, [bet_w], G)
        assert torch.equal(out, out_w)
        if len(set(vals.tolist())) == vals.size:
            assert torch.equal(g, g_w)
        else:  # the same addends, summed by atomics in whatever order the warps arrive
            assert torch.allclose(g, g_w, rtol=1e-5, atol=1e-4)


def test_empty_rows_pruned_weights_and_zero_sums():
    """DESIGN.md §4, Q14: a weight goes with its pruned id, an empty row gives 0, weights are not pruned by sign, and
    a row whose weights sum to 0 divides by zero."""
    from elasticdl_b200 import ops

    rows = np.array([0, 0, 1, 2, 2, 3, 3])
    cols = np.array([0, 1, 0, 0, 1, 0, 1])
    vals = np.array([4, -1, -2, 5, 6, 7, 8])
    w = torch.tensor([2.0, 100.0, 7.0, -1.0, 3.0, 0.0, 0.0], device="cuda")
    fill = torch.arange(10, device="cuda").float().unsqueeze(1).repeat(1, 2)
    bet, inv, ws, nnz, uniq = _prep_pull(rows, cols, vals, 4, 2, fill)
    out = ops.SparseCombine.apply(bet, inv, ws, 4, nnz, "mean", 2, w).cpu()
    assert uniq.tolist() == [4, 0, 5, 6, 7, 8]
    assert out[0].tolist() == [4.0, 4.0] and out[1].tolist() == [0.0, 0.0] and out[2].tolist() == [6.5, 6.5]
    assert torch.isnan(out[3]).all()
    wl = w.clone().requires_grad_(True)
    betl = bet.clone().requires_grad_(True)
    out = ops.SparseCombine.apply(betl, inv, ws, 4, nnz, "sum", 2, wl)
    gb, gw = torch.autograd.grad(out, [betl, wl], torch.ones(4, 2, device="cuda"))
    assert gw.tolist() == [8.0, 0.0, 0.0, 10.0, 12.0, 14.0, 16.0]  # the pruned entries get 0
    assert gb[:, 0].tolist() == [2.0, 0.0, -1.0, 3.0, 0.0, 0.0]  # the fill id 0 of the empty row gets nothing


def _bag_layer(dim, n, mode, group, table, **kw):
    from elasticdl_b200.layers.embedding_bag import EmbeddingBag

    layer = EmbeddingBag(dim, input_dim=n, mode=mode, **kw)
    layer.set_ps_group(group)
    layer.set_lookup_embedding_func(lambda name, ids: table[ids])
    layer.set_tape(True)
    return layer


@pytest.mark.parametrize("form", ["2d", "offsets", "offsets_last"])
@pytest.mark.parametrize("pad", [None, 2])
@pytest.mark.parametrize("vdtype", [torch.int64, torch.int32])
def test_embedding_bag_against_torch(form, pad, vdtype):
    from elasticdl_b200.ps import PSGroup

    group = PSGroup(1, *ADAM, device=0)
    gen = torch.Generator().manual_seed(3)
    B, N, dim = 3000, 300, 8
    table = torch.randn(N, dim, generator=gen).cuda()
    if form == "2d":
        x = torch.randint(0, N, (B, 6), generator=gen)
        if pad is not None:
            x[torch.rand(B, 6, generator=gen) < 0.3] = pad
        ids, offsets, offs = x, None, None
    else:
        lens = torch.randint(0, 9, (B,), generator=gen)
        lens[B // 2] = 600  # a bag of three combine pieces
        ids = torch.randint(0, N, (int(lens.sum()),), generator=gen)
        if pad is not None:
            ids[torch.rand(ids.numel(), generator=gen) < 0.3] = pad
        offsets = torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)])
        offs = offsets if form == "offsets_last" else offsets[:-1]
    psw = torch.rand(tuple(ids.shape), generator=gen).cuda() * 2 - 0.5
    layer = _bag_layer(dim, N, "sum", group, table, padding_idx=pad, include_last_offset=form == "offsets_last")
    w_ours = psw.clone().requires_grad_(True)
    out = layer(ids.to(vdtype).cuda(), None if offs is None else offs.cuda(), per_sample_weights=w_ours)
    group.check()
    bet, uniq = layer.embedding_and_ids[0]
    G = torch.randn(B, dim, generator=gen).cuda()
    g_bet, g_w = torch.autograd.grad(out, [bet, w_ours], G)
    t_table = table.clone().requires_grad_(True)
    w_t = psw.clone().requires_grad_(True)
    want = F.embedding_bag(ids.cuda(), t_table, None if offs is None else offs.cuda(), mode="sum",
                           per_sample_weights=w_t, include_last_offset=form == "offsets_last", padding_idx=pad)
    want.backward(G)
    assert torch.allclose(out, want, rtol=1e-5, atol=1e-5)
    dense = torch.zeros_like(table).index_add_(0, uniq, g_bet)
    assert torch.allclose(dense, t_table.grad, rtol=1e-5, atol=1e-5)
    assert torch.allclose(g_w, w_t.grad, rtol=1e-5, atol=1e-5)
    if pad is not None:
        assert (g_w[ids.cuda() == pad] == 0).all()
    group.close()


def test_refusals():
    from elasticdl_b200 import _lib, ops
    from elasticdl_b200.layers.embedding_bag import EmbeddingBag
    from elasticdl_b200.ps import PSGroup

    group = PSGroup(1, *ADAM, device=0)
    table = torch.randn(50, 4, device="cuda")
    x = torch.tensor([[1, 2], [3, 4]], device="cuda")
    with pytest.raises(NotImplementedError, match="mode='sum'"):
        _bag_layer(4, 50, "mean", group, table)(x, per_sample_weights=torch.ones(2, 2, device="cuda"))
    with pytest.raises(ValueError):
        EmbeddingBag(4, input_dim=50, mode="max")
    with pytest.raises(ValueError, match="same shape"):
        _bag_layer(4, 50, "sum", group, table)(x, per_sample_weights=torch.ones(4, device="cuda"))
    lookup = lambda name, ids: table[ids]
    ids = _coo([[1, 2], [3, 4]], [[1, 2], [3, 4]])
    with pytest.raises(ValueError, match="entries"):  # another shape
        _layer(4, "sum", lookup)(ids, _coo([[1, 2, 3], [3, 4, 5]], [[1.0, 1.0, 1.0], [1.0, 1.0, 1.0]]))
    wide = torch.sparse_coo_tensor(torch.tensor([[0, 0, 1, 1], [0, 1, 0, 1]]), torch.tensor([1, 2, 3, 4]), (2, 3))
    moved = torch.sparse_coo_tensor(torch.tensor([[0, 0, 1, 1], [0, 2, 0, 1]]), torch.ones(4), (2, 3))
    with pytest.raises(ValueError, match="indices"):  # same shape and count, one index differs
        _layer(4, "sum", lookup)(wide.cuda(), moved.cuda())
    with pytest.raises(ValueError, match="sparse ids"):
        _layer(4, "sum", lookup)(x, ids)
    sp = _coo([[1, 2], [3, 4]], [[1, 2], [3, 4]]).coalesce()
    idsf, ws = ops.sparse_prep(sp.indices()[0], sp.values(), 2, 4)
    uniq, inv, n = ops.unique(idsf)
    bet = table[uniq[: int(n.item())]]
    for combiner in ("mean", "sqrtn"):
        with pytest.raises(ValueError, match="sum combiner"):
            ops.SparseCombine.apply(bet, inv, ws, 2, 4, combiner, 4, torch.ones(4, device="cuda", requires_grad=True))
    with pytest.raises(ValueError, match="weights for"):
        ops.SparseCombine.apply(bet, inv, ws, 2, 4, "sum", 4, torch.ones(3, device="cuda"))
    lib = _lib.lib()
    gw = torch.empty(4, device="cuda")
    g = torch.empty(int(n.item()), 4, device="cuda")
    rc = lib.b200ps_sparse_combine_weighted_grad(None, g.data_ptr(), inv.data_ptr(), gw.data_ptr(), bet.data_ptr(),
                                                 ws.data_ptr(), ws.numel(), 2, 4, 4, 1, int(n.item()), g.data_ptr(),
                                                 gw.data_ptr(), ops._stream(g.device))
    assert rc == _lib.EINVAL and b"sum combiner" in lib.b200ps_last_error()
    rc = lib.b200ps_sparse_combine_weighted(None, bet.data_ptr(), inv.data_ptr(), gw.data_ptr(), ws.data_ptr(),
                                            ws.numel() - 4, 2, 4, 4, 0, g.data_ptr(), ops._stream(g.device))
    assert rc == _lib.EINVAL and b"workspace smaller" in lib.b200ps_last_error()
    group.close()



# ------------------------------------------------------------------ training through ModelHandler and the trainer
B = 256
PAD = 3


class WeightedBags(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.big = torch.nn.EmbeddingBag(70000, 8, mode="sum")  # 2.24 MB: a PS table
        self.small = torch.nn.EmbeddingBag(500, 8, mode="sum", include_last_offset=True, padding_idx=PAD)  # kept
        self.fc = torch.nn.Linear(16, 1)

    def forward(self, f):
        a = self.big(f["tags"], per_sample_weights=f["tag_w"])
        b = self.small(f["flat"], f["offs"], per_sample_weights=f["flat_w"])
        return self.fc(torch.cat([a, b], 1)).squeeze(1)


def _batch(gen, step):
    lo = 1000 * (step % 3)
    lens = torch.bincount(torch.randint(0, B, (2 * B,), generator=gen), minlength=B)  # some bags empty
    flat = torch.randint(0, 200, (2 * B,), generator=gen)
    flat[torch.rand(flat.numel(), generator=gen) < 0.2] = PAD
    return ({"tags": torch.randint(lo, lo + 2000, (B, 4), generator=gen).cuda(),
             "tag_w": torch.rand(B, 4, generator=gen).cuda() * 2,
             "flat": flat.cuda(), "flat_w": torch.rand(2 * B, generator=gen).cuda() - 0.3,
             "offs": torch.cat([torch.zeros(1, dtype=torch.int64), lens.cumsum(0)]).cuda()},
            (torch.rand(B, generator=gen) < 0.3).float().cuda())


def _trainer(mode):
    from elasticdl_b200.common.model_handler import ParameterServerModelHandler
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    torch.manual_seed(0)
    handler = ParameterServerModelHandler()
    model = handler.get_model_to_train(WeightedBags()).cuda()
    model.optimizer = torch.optim.SGD(model.parameters(), lr=0.01)
    model.loss = lambda labels, out: F.binary_cross_entropy_with_logits(out, labels)
    group = PSGroup(1, *ADAM, device=0)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
        get_model_steps=1, batched_embedding_lookups=mode != "eager", cuda_graph=mode == "graphed",
        cuda_graph_warmup=2))
    return handler, model, group, trainer


def _keras_adam(w, g, m, v, rows, step, lr=0.01):
    """The PS's Adam (kernel_api.cc:40-77) on the rows a push carries."""
    m[rows] = 0.9 * m[rows] + 0.1 * g[rows]
    v[rows] = 0.999 * v[rows] + 0.001 * g[rows] ** 2
    alpha = lr * np.sqrt(1 - 0.999 ** step) / (1 - 0.9 ** step)
    w[rows] -= alpha * m[rows] / (v[rows].sqrt() + 1e-7)


def test_weighted_bags_train_eager_batched_graphed_against_float64_and_export():
    steps = 5
    runs = {mode: _trainer(mode) for mode in ("eager", "batched", "graphed")}
    _, model0, _, _ = runs["eager"]
    d = torch.float64
    W = {"big": torch.zeros(70000, 8, dtype=d),  # the PS zero-initialises swapped tables (Q6)
         "small": model0.small.weight.detach().cpu().to(d).clone(),
         "fc.w": model0.fc.weight.detach().cpu().to(d).clone(), "fc.b": model0.fc.bias.detach().cpu().to(d).clone()}
    mom = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in W.items()}
    gen = torch.Generator().manual_seed(5)
    for step in range(1, steps + 1):
        f, labels = _batch(gen, step)
        losses = {}
        for mode, (_, _, _, trainer) in runs.items():
            accepted, version, loss = trainer.train_minibatch(f, labels)
            assert accepted and version == step
            losses[mode] = float(loss)
        P = {k: v.clone().requires_grad_(True) for k, v in W.items()}
        fc = {k: v.cpu() for k, v in f.items()}
        a = F.embedding_bag(fc["tags"], P["big"], mode="sum", per_sample_weights=fc["tag_w"].to(d))
        b = F.embedding_bag(fc["flat"], P["small"], fc["offs"], mode="sum", per_sample_weights=fc["flat_w"].to(d),
                            include_last_offset=True, padding_idx=PAD)
        out = F.linear(torch.cat([a, b], 1), P["fc.w"], P["fc.b"]).squeeze(1)
        ref = F.binary_cross_entropy_with_logits(out, labels.cpu().to(d))
        ref.backward()
        for mode, loss in losses.items():
            assert abs(loss - float(ref)) < 1e-5, (mode, step, loss, float(ref))
        kept = fc["flat"][fc["flat"] != PAD]
        lens = torch.tensor([int((fc["flat"][fc["offs"][i]:fc["offs"][i + 1]] != PAD).sum()) for i in range(B)])
        small_rows = torch.cat([kept, torch.zeros(int((lens == 0).any()), dtype=torch.int64)]).unique()
        with torch.no_grad():
            for k, rows in (("big", fc["tags"].unique()), ("small", small_rows), ("fc.w", slice(None)),
                            ("fc.b", slice(None))):
                _keras_adam(W[k], P[k].grad, *mom[k], rows, step)
    graphed = runs["graphed"][3]
    assert isinstance(graphed._graph_state, dict) and graphed.graph_fallback_reason is None, \
        graphed.graph_fallback_reason
    tag_ids = torch.arange(0, 3000)
    states = {}
    for mode, (_, _, group, _) in runs.items():
        dense = group.pull_dense(["small.weight", "fc.weight", "fc.bias"])
        big = group.pull_rows([("big/embeddings:0", tag_ids.cuda())])[0]
        states[mode] = [big.cpu(), dense["small.weight"].cpu(), dense["fc.weight"].cpu(), dense["fc.bias"].cpu()]
        want = [W["big"][:3000], W["small"], W["fc.w"], W["fc.b"]]
        for got, w in zip(states[mode], want):
            assert torch.allclose(got.double(), w, rtol=1e-4, atol=2e-5), mode
    for mode in ("batched", "graphed"):
        for a, b in zip(states[mode], states["eager"]):
            assert torch.allclose(a, b, rtol=1e-5, atol=1e-6), mode
    # the exported torch model computes what the trained model computes, per_sample_weights included
    handler, model, group, trainer = runs["eager"]
    f, labels = _batch(gen, 9)
    trainer._get_model()
    trainer.evaluate_minibatch(f, labels)
    trained = trainer.get_evaluation_result()["output"][-1]
    exported = handler.get_model_to_export(model, group=group)
    assert type(exported.big) is torch.nn.EmbeddingBag and type(exported.small) is torch.nn.EmbeddingBag
    with torch.no_grad():
        out = exported(f).cpu().numpy()
    assert np.allclose(out, trained, rtol=1e-5, atol=1e-6)
    for _, _, group, _ in runs.values():
        group.close()
