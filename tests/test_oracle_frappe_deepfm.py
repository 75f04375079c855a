"""The float64 frappe DeepFM oracle (oracle/frappe_oracle.py) on the CPU: against torch float64 autograd of an
independently written layered model on batches with pads, its mutations, the parameter layout, and the synthetic
frappe batches."""
import pytest
import torch

from elasticdl_b200.workloads import frappe as FR
from oracle import frappe_oracle as O


def _batch(B, seed, pad_fraction=0.3):
    gen = torch.Generator().manual_seed(seed)
    ids, labels = FR.synthetic_frappe_batch(B, seed, "cpu", pad_fraction=pad_fraction)
    uniq, inv, U = O.dedup(ids)
    E = (torch.rand((FR.INPUT_DIM, 64), generator=gen, dtype=torch.float64) * 2 - 1) * 0.5
    W = (torch.rand((FR.INPUT_DIM, 1), generator=gen, dtype=torch.float64) * 2 - 1) * 0.5
    flat = O.random_params(gen, "cpu", dtype=torch.float64)
    return ids, labels.double(), uniq, inv, U, E[uniq], W[uniq], flat


def _layered(ids, labels, rows_deep, rows_wide, inv, flat):
    """The model as Keras runs it, written as plain torch layers: lookup, ApplyMask, FM, Flatten, two Dense."""
    B = ids.shape[0]
    p = O.unflatten(flat)
    leaves = [rows_deep.clone().requires_grad_(True), rows_wide.clone().requires_grad_(True)]
    leaves += [p[n].clone().requires_grad_(True) for n, _ in O.DENSE_PARAMS]
    Eu, Wu, K, b, w2, b2 = leaves
    mask = (ids != 0).double().unsqueeze(-1)
    emb = torch.nn.functional.embedding(inv.view(B, 10), Eu) * mask
    bias = torch.nn.functional.embedding(inv.view(B, 10), Wu) * mask
    first = torch.sum(bias, dim=(1, 2))
    sum_sq = torch.square(torch.sum(emb, dim=1))
    sq_sum = torch.sum(torch.square(emb), dim=1)
    second = torch.sum(0.5 * (sum_sq - sq_sum), dim=1)
    flat_x = torch.flatten(emb, start_dim=1)
    deep = torch.nn.functional.linear(torch.nn.functional.linear(flat_x, K.t(), b), w2.t(), b2)[:, 0]
    z = first + second + deep
    loss = torch.nn.functional.binary_cross_entropy_with_logits(z, labels)
    return z, loss, torch.autograd.grad(loss, leaves)


@pytest.mark.parametrize("B", [1, 2, 7, 64, 130])
def test_oracle_matches_layered_autograd(B):
    ids, labels, uniq, inv, U, rd, rw, flat = _batch(B, seed=B)
    ids[0, :3] = 0  # pads in every batch
    uniq, inv, U = O.dedup(ids)
    gen = torch.Generator().manual_seed(B + 1)
    rd = (torch.rand((U, 64), generator=gen, dtype=torch.float64) * 2 - 1) * 0.5
    rw = (torch.rand((U, 1), generator=gen, dtype=torch.float64) * 2 - 1) * 0.5
    ref = O.frappe_reference(ids, inv, U, rd, rw, labels, flat)
    z, loss, g = _layered(ids, labels, rd, rw, inv, flat)
    torch.testing.assert_close(ref["logits"], z.detach(), rtol=1e-12, atol=1e-13)
    torch.testing.assert_close(ref["loss"], loss.detach(), rtol=1e-12, atol=1e-14)
    dense = torch.cat([g[2].reshape(-1), g[3], g[4].reshape(-1), g[5].reshape(-1)])
    torch.testing.assert_close(ref["grads"], dense, rtol=1e-10, atol=1e-14)
    torch.testing.assert_close(ref["gsum_deep"], g[0], rtol=1e-10, atol=1e-14)
    torch.testing.assert_close(ref["gsum_wide"], g[1], rtol=1e-10, atol=1e-14)
    pad = ref["row_id"] == 0
    assert bool(pad.any()) and bool((ref["gsum_deep"][pad] == 0).all()) and bool((ref["gsum_wide"][pad] == 0).all())
    assert torch.equal(ref["row_id"], uniq)
    for fam in O.FAMILIES:  # the magnitude pass bounds every value
        assert bool((ref["M"][fam] >= ref[fam].abs() * (1 - 1e-12)).all()), fam


def test_collapsed_form_equals_layers():
    """The kernel's algebra: deep = x . (K w2) + (b . w2 + b2), and a row's gradient per occurrence is
    m g (S - e + v_f)."""
    B = 33
    ids, labels, uniq, inv, U, rd, rw, flat = _batch(B, seed=3)
    ref = O.frappe_reference(ids, inv, U, rd, rw, labels, flat)
    p = O.unflatten(flat)
    v = p["dense/kernel:0"] @ p["dense_1/kernel:0"][:, 0]
    c = p["dense/bias:0"] @ p["dense_1/kernel:0"][:, 0] + p["dense_1/bias:0"][0]
    m = (ids != 0).double().unsqueeze(-1)
    e = m * rd[inv.view(B, 10)]
    S = e.sum(1)
    z = (m * rw[inv.view(B, 10)]).sum((1, 2)) + 0.5 * (S * S - (e * e).sum(1)).sum(1) + e.reshape(B, 640) @ v + c
    torch.testing.assert_close(z, ref["logits"], rtol=1e-12, atol=1e-13)
    g = (torch.sigmoid(z) - labels) / B
    per = m * g.view(B, 1, 1) * (S.unsqueeze(1) - e + v.view(1, 10, 64))
    gd = torch.zeros((U, 64), dtype=torch.float64).index_add_(0, inv, per.reshape(-1, 64))
    torch.testing.assert_close(gd, ref["gsum_deep"], rtol=1e-10, atol=1e-14)


@pytest.mark.parametrize("B", [16, 64])
def test_every_mutation_is_caught(B):
    ids, labels, uniq, inv, U, rd, rw, flat = _batch(B, seed=11 + B, pad_fraction=0.5)
    inputs = (ids, inv, U, rd, rw, labels, flat)
    ref = O.frappe_reference(*inputs)
    # the reference passes its own check with float32 rounding of every output
    f32 = {k: ref[k].float() for k in O.FAMILIES}
    assert not O.caught_by(f32, ref)
    muts = O.mutations(ref, inputs)
    assert set(muts) == {"mask_dropped", "pad_row_gradient", "flatten_d_major", "fm_sign", "c_missing", "wide_twice",
                         "drop_one_sample"}
    for name, mut in muts.items():
        assert O.caught_by(mut, ref), name


def test_parameter_names_and_layout():
    assert FR.DENSE_PARAMS == O.DENSE_PARAMS
    assert [FR.OFFSETS[n] for n in FR.DENSE_NAMES] == [0, 40960, 41024, 41088] == [O.OFFSETS[n] for n in FR.DENSE_NAMES]
    assert FR.N_PARAMS == O.N_PARAMS == 41089
    assert (FR.DEEP_NAME, FR.WIDE_NAME) == ("embedding/embeddings:0", "embedding_1/embeddings:0")
    flat = torch.arange(FR.N_PARAMS, dtype=torch.float32)
    assert float(FR.flat_views(flat)["dense/kernel:0"][1, 0]) == 64  # [in, out] row-major
    init = FR.flat_views(FR.initial_dense(5, "cpu"))
    assert float(init["dense/bias:0"].abs().max()) == 0 and float(init["dense_1/bias:0"].abs().max()) == 0
    assert 0 < float(init["dense/kernel:0"].abs().max()) <= (6.0 / 704) ** 0.5
    # the drop-in twin registers the same dense parameter names
    model = FR.FrappeDeepFM(0.1)
    assert [n for n, _ in model.named_parameters()] == FR.DENSE_NAMES
    assert (model.deep.embedding_weight_name, model.wide.embedding_weight_name) == (FR.DEEP_NAME, FR.WIDE_NAME)


def test_twin_tower_equals_oracle():
    B = 20
    ids, labels, uniq, inv, U, rd, rw, flat = _batch(B, seed=8)
    ref = O.frappe_reference(ids, inv, U, rd, rw, labels, flat)
    model = FR.FrappeDeepFM(0.1).double()
    model.load_mlp(flat)
    z = model.tower(rd[inv.view(B, 10)], rw[inv.view(B, 10)], ids != 0)
    torch.testing.assert_close(z.detach(), ref["logits"], rtol=1e-12, atol=1e-13)


def test_synthetic_batches():
    ids, labels = FR.synthetic_frappe_batch(20000, 4, "cpu", pad_fraction=0.3)
    assert ids.dtype == torch.int64 and ids.shape == (20000, 10) and labels.shape == (20000,)
    assert int(ids.min()) >= 0 and int(ids.max()) <= 5382
    real = ids != 0
    for f in range(10):  # field f's ids are its own contiguous 1-based range
        col = ids[:, f][real[:, f]]
        lo, hi = FR.FIELD_START[f], FR.FIELD_START[f] + FR.FIELD_SIZES[f]
        assert int(col.min()) >= lo and int(col.max()) < hi, f
    assert FR.FIELD_START[0] == 1 and FR.FIELD_START[-1] + FR.FIELD_SIZES[-1] == 5383
    # pads only on the left: once a sample has a real id, every later field is real
    assert bool((real[:, 1:] >= real[:, :-1]).all())
    frac = float((~real).any(1).double().mean())
    assert 0.27 < frac < 0.33
    assert 0.30 < float(labels.mean()) < 0.37
    # Zipf within a field: the first id of a field is drawn most often
    item = ids[:, 1][real[:, 1]]
    assert int((item == FR.FIELD_START[1]).sum()) > 10 * int((item == FR.FIELD_START[1] + 100).sum())
    none, _ = FR.synthetic_frappe_batch(100, 4, "cpu")
    assert bool((none != 0).all())


def test_teacher_is_learnable_by_the_oracle():
    """The GPU sanity run's task, calibrated here: 200 SGD 0.1 steps of batch 64 (float64 oracle gradients, the
    PS's plain SGD update) on synthetic batches labelled by a fixed random teacher reach a held-out accuracy well
    above the reference's 0.65 threshold (worker_ps_interaction_test.py:333-343)."""
    ref_ids, _ = FR.synthetic_frappe_batch(8192, 12345, "cpu", pad_fraction=0.1)
    teacher = O.make_teacher(0, ref_ids)
    g = torch.Generator().manual_seed(1)
    E = (torch.rand((FR.INPUT_DIM, 64), generator=g, dtype=torch.float64) * 2 - 1) * 0.05
    W = (torch.rand((FR.INPUT_DIM, 1), generator=g, dtype=torch.float64) * 2 - 1) * 0.05
    flat = FR.initial_dense(0, "cpu").double()
    for step in range(200):
        ids, _ = FR.synthetic_frappe_batch(64, 100 + step, "cpu", pad_fraction=0.1)
        y = O.teacher_labels(teacher, ids).double()
        uniq, inv, U = O.dedup(ids)
        r = O.frappe_reference(ids, inv, U, E[uniq], W[uniq], y, flat)
        flat -= 0.1 * r["grads"]
        E[uniq] -= 0.1 * r["gsum_deep"]
        W[uniq] -= 0.1 * r["gsum_wide"]
    ids, _ = FR.synthetic_frappe_batch(4096, 7, "cpu", pad_fraction=0.1)
    y = O.teacher_labels(teacher, ids).double()
    assert 0.45 < float(y.mean()) < 0.55
    uniq, inv, U = O.dedup(ids)
    z = O.frappe_reference(ids, inv, U, E[uniq], W[uniq], y, flat)["logits"]
    acc = float(((z > 0).double() == y).double().mean())
    assert acc > 0.75, acc  # 0.79 with these seeds
