"""GPU tests of the pooled lookup of sparse input (Embedding with a combiner on a sparse COO input): the
reference's literal vectors (layer_test.py:188-215 forward, :294-370 BET gradients), random shapes against the
float64 oracle's bound (oracle/sparse_oracle.py), determinism, refusals, and PS training against local training."""
import numpy as np
import pytest
import torch

from oracle import sparse_oracle as so

pytestmark = pytest.mark.gpu
COMBINERS = ["sum", "mean", "sqrtn"]
ADAM = ("Adam", "learning_rate=0.01;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")

# layer_test.py:191-193
IDX = [[0, 1, 1, 2, 3, 3, 3], [0, 1, 2, 1, 1, 3, 5]]
VAL = [1, 1, 3, 2, 0, 2, 6]
FWD = {"sum": [1.0, 4.0, 2.0, 8.0], "mean": [1.0, 2.0, 2.0, 8.0 / 3.0],
       "sqrtn": [1.0, 4.0 / np.sqrt(2.0), 2.0, 8.0 / np.sqrt(3.0)]}
GRADS = {"sum": [1, 1, 5, 3, 3], "mean": [0.5, 0.5, 3.0, 1.0, 1.0],
         "sqrtn": [1 / np.sqrt(2.0), 1 / np.sqrt(2.0), 2 + 3 / np.sqrt(3.0), 3 / np.sqrt(3.0), 3 / np.sqrt(3.0)]}


def fake_lookup(dim):
    def fn(name, ids):  # layer_test.py:71-101 mock_worker.lookup_embedding
        return ids.to(torch.float32).unsqueeze(1).repeat(1, dim)
    return fn


def table_lookup(table):
    def fn(name, ids):
        return table[ids % table.shape[0]]
    return fn


def _layer(dim, combiner, input_dim=None, lookup=None):
    from elasticdl_b200.layers import Embedding

    layer = Embedding(dim, input_dim=input_dim, combiner=combiner)
    layer.set_lookup_embedding_func(lookup or fake_lookup(dim))
    return layer


@pytest.mark.parametrize("combiner", COMBINERS)
def test_layer_test_py_vectors(combiner):
    sp = torch.sparse_coo_tensor(torch.tensor(IDX), torch.tensor(VAL), (4, 6)).cuda()
    layer = _layer(8, combiner, input_dim=16)
    out = layer(sp)
    want = torch.tensor(FWD[combiner], dtype=torch.float64).unsqueeze(1).repeat(1, 8)
    assert out.shape == (4, 8)
    if combiner == "sum":
        assert torch.equal(out.cpu().double(), want)
    else:
        np.testing.assert_allclose(out.cpu().numpy(), want.numpy(), atol=5e-6)
    mult = torch.arange(4, dtype=torch.float32, device="cuda").unsqueeze(1).repeat(1, 8)  # layer_test.py:303-305
    layer.set_tape(True)
    for _ in range(2):  # two calls record two entries
        out = layer(sp)
        bet, ids = layer.embedding_and_ids[-1]
        (g,) = torch.autograd.grad((out * mult).sum(), [bet])
        assert ids.tolist() == [1, 3, 2, 0, 6]
        if combiner == "sum":
            assert torch.equal(g[:, 0].cpu().double(), torch.tensor(GRADS["sum"], dtype=torch.float64))
        else:
            np.testing.assert_allclose(g[:, 0].cpu().numpy(), GRADS[combiner], atol=5e-6)
        assert torch.equal(g, g[:, :1].expand_as(g))
    assert len(layer.embedding_and_ids) == 2


def _random_case(rng, B, mean_len, long_row=0, neg=0.05, empty=0.02, all_neg=0.01, id_range=1000):
    lens = rng.poisson(mean_len, B).astype(np.int64)
    lens[rng.random(B) < empty] = 0
    if long_row:
        lens[rng.integers(0, B)] = long_row
    rows = np.repeat(np.arange(B), lens)
    vals = rng.integers(0, id_range, rows.size)
    vals[rng.random(rows.size) < neg] = -rng.integers(1, 5, 1)
    allneg = np.isin(rows, np.nonzero(rng.random(B) < all_neg)[0])
    vals[allneg] = -1
    cols = np.concatenate([np.arange(n) for n in lens]) if rows.size else np.zeros(0, np.int64)
    return rows, cols, vals, int(max(lens.max() if B else 1, 1))


CASES = [  # (B, mean ids per row, dim, long row, value dtype)
    (1, 5, 8, 0, torch.int64),
    (1, 0, 4, 6000, torch.int32),
    (257, 10, 1, 5000, torch.int64),
    (4096, 10, 13, 0, torch.int32),
    (4096, 3, 64, 7000, torch.int64),
    (70000, 4, 8, 0, torch.int64),
    (20000, 30, 4, 5000, torch.int32),  # nnz = 6e5 in 586 prep tiles of 1024 entries
    # nnz = 2.5e6 in 2442 tiles: past the 132 * 16 = 2112 blocks the prep's count and scatter get without a group (a
    # second pass of their tile loops) and past the scan's 1024-tile chunk (its carry across chunks)
    (90000, 28, 1, 0, torch.int32),
]


@pytest.mark.parametrize("B,mean_len,dim,long_row,vdtype", CASES)
@pytest.mark.parametrize("bounded", [True, False])
def test_random_against_oracle(B, mean_len, dim, long_row, vdtype, bounded):
    rng = np.random.default_rng(B + dim + long_row)
    rows, cols, vals, L = _random_case(rng, B, mean_len, long_row)
    rows_t = torch.tensor(rows, dtype=torch.int64)
    table = torch.randn(1000, dim, device="cuda")
    for combiner in COMBINERS:
        sp = torch.sparse_coo_tensor(torch.stack([rows_t, torch.tensor(cols)]), torch.tensor(vals).to(vdtype),
                                     (B, L)).cuda()
        layer = _layer(dim, combiner, input_dim=1000 if bounded else None, lookup=table_lookup(table))
        layer.set_tape(True)
        out = layer(sp)
        bet, ids = layer.embedding_and_ids[0]
        tab = table.double().cpu().numpy()
        want, uniq, obet = so.lookup(rows, vals, B, lambda u: tab[u % 1000], combiner)
        np.testing.assert_array_equal(ids.cpu().numpy(), uniq)
        bd = so.bound(rows, vals, B, np.abs(obet), combiner)
        err = np.abs(out.detach().double().cpu().numpy() - want)
        assert (err <= bd).all(), (combiner, float((err - bd).max()))
        G = torch.randn(B, dim, device="cuda")
        (g,) = torch.autograd.grad((out * G).sum(), [bet])
        gw = so.grad_bet(rows, vals, B, len(uniq), G.double().cpu().numpy(), combiner)
        gb = so.grad_bound(rows, vals, B, len(uniq), np.abs(G.double().cpu().numpy()), combiner)
        gerr = np.abs(g.detach().double().cpu().numpy() - gw)
        assert (gerr <= gb).all(), (combiner, float((gerr - gb).max()))
        again = layer(sp)
        assert torch.equal(out, again)  # every summation order is fixed


def test_nnz_zero():
    for combiner in COMBINERS:
        sp = torch.sparse_coo_tensor(torch.zeros(2, 0, dtype=torch.int64), torch.zeros(0, dtype=torch.int64),
                                     (5, 3)).cuda()
        layer = _layer(4, combiner)
        layer.set_tape(True)
        out = layer(sp)
        bet, ids = layer.embedding_and_ids[0]
        assert ids.tolist() == [0] and bet.shape == (1, 4)
        assert out.shape == (5, 4) and (out == 0).all()
        (g,) = torch.autograd.grad(out.sum(), [bet])
        assert (g == 0).all()


def test_row_outside_batch_raises_and_next_call_is_correct():
    # coalesced on the CPU, which keeps row 7 (CUDA's coalesce re-derives rows modulo the size), then moved
    idx = torch.tensor([[0, 1, 7], [0, 0, 0]])
    bad = torch.sparse_coo_tensor(idx, torch.tensor([1, 2, 3]), (3, 2), check_invariants=False).coalesce().cuda()
    assert bad.is_coalesced() and bad.indices()[0].tolist() == [0, 1, 7]
    layer = _layer(4, "sum")
    with pytest.raises(ValueError, match="row index"):
        layer(bad)
    good = torch.sparse_coo_tensor(torch.tensor([[0, 1, 2], [0, 0, 0]]), torch.tensor([1, 2, 3]), (3, 2)).cuda()
    assert layer(good)[:, 0].tolist() == [1.0, 2.0, 3.0]


def test_id_past_input_dim_raises():
    sp = torch.sparse_coo_tensor(torch.tensor([[0, 1], [0, 0]]), torch.tensor([1, 50]), (2, 1)).cuda()
    with pytest.raises(ValueError):
        _layer(4, "mean", input_dim=10)(sp)


def _prep_and_pull(rows, cols, vals, B, L, table):
    from elasticdl_b200 import ops

    sp = torch.sparse_coo_tensor(torch.tensor(np.stack([rows, cols])), torch.tensor(vals), (B, L)).coalesce().cuda()
    ids, ws = ops.sparse_prep(sp.indices()[0], sp.values(), B, table.shape[1])
    uniq, inv, n = ops.unique(ids)
    return table[uniq[: int(n.item())] % table.shape[0]], inv, ws, sp.values().numel()


@pytest.mark.parametrize("combiner", COMBINERS)
def test_combine_and_grad_twice_on_one_workspace(combiner):
    """The combine may run again after one prep (e.g. after a re-pull): rows longer than one 256-entry piece go through
    the arrival counter, which the finishing piece resets."""
    from elasticdl_b200 import ops

    rng = np.random.default_rng(5)
    B, dim = 6, 8
    lens = np.array([1000, 3, 0, 257, 1, 600])
    rows = np.repeat(np.arange(B), lens)
    cols = np.concatenate([np.arange(n) for n in lens])
    vals = rng.integers(0, 500, rows.size)
    table = torch.randn(500, dim, device="cuda")
    bet, inv, ws, nnz = _prep_and_pull(rows, cols, vals, B, int(lens.max()), table)
    bet.requires_grad_(True)
    G = torch.randn(B, dim, device="cuda")
    outs, grads = [], []
    for _ in range(3):
        poison = torch.full((B, dim), float("nan"), device="cuda")  # the next output block starts as NaN
        del poison
        out = ops.SparseCombine.apply(bet, inv, ws, B, nnz, combiner, dim)
        (g,) = torch.autograd.grad(out, [bet], G)
        outs.append(out.detach())
        grads.append(g)
    want, _, obet = so.lookup(rows, vals, B, lambda u: table.double().cpu().numpy()[u], combiner)
    assert (np.abs(outs[0].double().cpu().numpy() - want) <= so.bound(rows, vals, B, np.abs(obet), combiner)).all()
    for o, g in zip(outs[1:], grads[1:]):
        assert torch.equal(o, outs[0])
        assert torch.allclose(g, grads[0], rtol=1e-6, atol=1e-6)


def test_lookup_of_another_width_raises():
    table = torch.randn(50, 5, device="cuda")
    sp = torch.sparse_coo_tensor(torch.tensor([[0, 1], [0, 0]]), torch.tensor([1, 2]), (2, 1)).cuda()
    with pytest.raises(ValueError, match="n_unique, 4"):
        _layer(4, "mean", lookup=table_lookup(table))(sp)


def test_combine_refuses_a_small_workspace():
    from elasticdl_b200 import _lib, ops

    B, dim = 4, 8
    lens = np.array([300, 1, 0, 2])
    rows = np.repeat(np.arange(B), lens)
    cols = np.concatenate([np.arange(n) for n in lens])
    bet, inv, ws, nnz = _prep_and_pull(rows, cols, np.arange(rows.size) % 40, B, 300, torch.randn(40, dim, device="cuda"))
    lib = _lib.lib()
    need = lib.b200ps_sparse_workspace(B, nnz, dim)
    assert need == ws.numel()
    wider = lib.b200ps_sparse_workspace(B, nnz, 2 * dim)
    assert wider > need  # the partial sums of rows past one piece are sized by dim
    out = torch.empty(B, 2 * dim, device="cuda")
    g = torch.empty(bet.shape[0], 2 * dim, device="cuda")
    stream = ops._stream(bet.device)
    rc = lib.b200ps_sparse_combine(None, bet.data_ptr(), inv.data_ptr(), ws.data_ptr(), ws.numel(), B, nnz, 2 * dim, 1,
                                   out.data_ptr(), stream)
    assert rc == _lib.EINVAL and b"workspace smaller" in lib.b200ps_last_error()
    rc = lib.b200ps_sparse_combine_grad(None, out.data_ptr(), inv.data_ptr(), ws.data_ptr(), ws.numel(), B, nnz,
                                        2 * dim, 1, bet.shape[0], g.data_ptr(), stream)
    assert rc == _lib.EINVAL and b"workspace smaller" in lib.b200ps_last_error()


class SparseDenseModel(torch.nn.Module):
    """One multi-hot feature pooled by mean over a hashed table and one dense-id feature."""

    def __init__(self, dim=4):
        super().__init__()
        from elasticdl_b200.layers import Embedding

        self.tags = Embedding(dim, combiner="mean", embeddings_initializer="zero", name="sp_tags")
        self.item = Embedding(dim, input_dim=40, embeddings_initializer="zero", name="sp_item")
        self.fc = torch.nn.Linear(3 * dim, 1)
        self.optimizer = torch.optim.Adam(self.fc.parameters(), lr=0.01)
        self.loss = lambda labels, out: ((out.squeeze(1) - labels) ** 2).mean()

    def forward(self, features):
        t = self.tags(features["tags"])
        i = self.item(features["item"]).reshape(features["item"].shape[0], -1)
        return self.fc(torch.cat([t, i], 1))


def test_trainer_sparse_and_dense_layers_equal_local_training():
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    torch.manual_seed(0)
    dim, B = 4, 16
    model = SparseDenseModel(dim).cuda()
    group = PSGroup(1, *ADAM, device=0)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client)
    tag_ids = torch.arange(0, 1000, 37)
    tag0 = torch.randn(len(tag_ids), dim, device="cuda") * 0.1
    item0 = torch.randn(40, dim, device="cuda") * 0.1
    group.set_rows([("sp_tags/embeddings:0", tag_ids, tag0), ("sp_item/embeddings:0", torch.arange(40), item0)])
    tags = torch.zeros(1000, dim, device="cuda")
    tags[tag_ids.cuda()] = tag0
    tags.requires_grad_(True)
    items = item0.clone().requires_grad_(True)
    fc = torch.nn.Linear(3 * dim, 1).cuda()
    fc.load_state_dict(model.fc.state_dict())
    opt = torch.optim.Adam(list(fc.parameters()), lr=0.01, eps=1e-7)
    moments = {id(t): (torch.zeros_like(t), torch.zeros_like(t)) for t in (tags, items)}

    def sparse_adam(t, touched, step):  # the PS's Adam on the rows a push carries (kernel_api.cc:40-77)
        m, v = moments[id(t)]
        g = t.grad[touched]
        m[touched] = 0.9 * m[touched] + 0.1 * g
        v[touched] = 0.999 * v[touched] + 0.001 * g * g
        alpha = 0.01 * np.sqrt(1 - 0.999 ** step) / (1 - 0.9 ** step)
        with torch.no_grad():
            t[touched] -= alpha * m[touched] / (v[touched].sqrt() + 1e-7)

    gen = torch.Generator().manual_seed(2)
    for step in range(1, 4):
        lens = torch.randint(0, 5, (B,), generator=gen)
        rows = torch.repeat_interleave(torch.arange(B), lens)
        cols = torch.cat([torch.arange(int(n)) for n in lens])
        vals = tag_ids[torch.randint(0, len(tag_ids), (rows.numel(),), generator=gen)]
        vals[torch.rand(rows.numel(), generator=gen) < 0.1] = -1
        sp = torch.sparse_coo_tensor(torch.stack([rows, cols]), vals, (B, 5)).cuda()
        item = torch.randint(0, 40, (B, 2), generator=gen).cuda()
        labels = torch.randn(B, generator=gen).cuda()
        accepted, version, loss = trainer.train_minibatch({"tags": sp, "item": item}, labels)
        assert accepted and version == step
        # local twin: the same pooling written with torch ops on a dense table
        keep = vals >= 0
        r, v = rows[keep].cuda(), vals[keep].cuda()
        cnt = torch.bincount(r, minlength=B)
        empty = cnt == 0
        pooled = torch.zeros(B, dim, device="cuda").index_add(0, r, tags[v])
        pooled = pooled + empty.float().unsqueeze(1) * tags[0]  # the fill id 0 of an empty row (zero gradient)
        pooled = torch.where(empty.unsqueeze(1), torch.zeros_like(pooled), pooled / cnt.clamp(min=1).unsqueeze(1))
        out = fc(torch.cat([pooled, items[item].reshape(B, -1)], 1))
        l2 = ((out.squeeze(1) - labels) ** 2).mean()
        opt.zero_grad()
        tags.grad = items.grad = None
        l2.backward()
        opt.step()
        touched = torch.unique(torch.cat([v, torch.zeros(int(empty.any()), dtype=torch.int64, device="cuda")]))
        sparse_adam(tags, touched, step)
        sparse_adam(items, torch.unique(item), step)
        assert abs(float(loss) - float(l2.detach())) < 1e-5
    # Adam divides by sqrt(v): a gradient entry near zero turns its last-bit differences (summation order, the
    # twin's float32 moments) into a step difference of up to ~1e-5 of lr = 0.01
    got = client.pull_embedding_vectors("sp_tags/embeddings:0", tag_ids.cuda())
    assert torch.allclose(got, tags.detach()[tag_ids.cuda()], rtol=1e-4, atol=2e-5)
    got = client.pull_embedding_vectors("sp_item/embeddings:0", torch.arange(40).cuda())
    assert torch.allclose(got, items.detach(), rtol=1e-4, atol=2e-5)
    group.close()
