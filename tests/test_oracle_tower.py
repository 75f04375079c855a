"""CPU tests of the float64 DeepFM tower reference (oracle/tower_oracle.py) and of the comparator the GPU
tower tests use: the reference equals float64 autograd through workloads.deepfm.DeepFMTower, an honest fp32
evaluation passes the bound, and five classic tiled-reduction faults fail it at the benchmark shape."""
import numpy as np
import pytest
import torch

from oracle import ps_oracle as O
from oracle import tower_oracle as T

CPU = torch.device("cpu")


def _inputs(G, B, seed, ids=None, rows_std=0.3):
    gen = torch.Generator(device=CPU).manual_seed(seed)
    if ids is None:  # heavy duplication: a handful of ids per group
        ids = torch.randint(0, max(2, B // 3), (G, B), generator=gen)
    inv, n_unique, uniq = T.first_occurrence_inverse(ids)
    bet_wide = torch.full((G, B), float("nan"))
    bet_deep = torch.full((G, B, T.D), float("nan"))
    for g in range(G):
        u = int(n_unique[g])
        bet_wide[g, :u] = torch.randn(u, generator=gen) * rows_std
        bet_deep[g, :u] = torch.randn((u, T.D), generator=gen) * rows_std
    dense = torch.randn((B, T.ND), generator=gen)
    labels = (torch.rand(B, generator=gen) < 0.3).float()
    params = T.random_params(G, gen, CPU)
    return inv, n_unique, bet_wide, bet_deep, dense, labels, params


def _autograd(inputs, dtype):
    """Per-occurrence rows through DeepFMTower + BCEWithLogitsLoss, torch autograd in `dtype`."""
    from elasticdl_b200.workloads.deepfm import DeepFMTower, flatten_tower

    inv, n_unique, bet_wide, bet_deep, dense, labels, params = inputs
    G, B = inv.shape
    tower = DeepFMTower(G).to(dtype)
    flat = torch.zeros(T.layout(G)["total"], dtype=dtype)
    flatten_tower(tower, flat)
    with torch.no_grad():
        flat.copy_(params.to(dtype))
    il = inv.long()
    wide = torch.gather(bet_wide, 1, il).to(dtype).t().contiguous().requires_grad_(True)  # [B, G]
    deep = torch.gather(bet_deep, 1, il.unsqueeze(2).expand(G, B, T.D)).to(dtype).permute(1, 0, 2).contiguous()
    deep.requires_grad_(True)
    logits = tower(dense.to(dtype), wide, deep)
    loss = torch.nn.BCEWithLogitsLoss()(logits, labels.to(dtype))
    order = [tower.dense_linear.weight, tower.dnn[0].weight, tower.dnn[0].bias, tower.dnn[1].weight,
             tower.dnn[1].bias, tower.dnn_logit.weight]
    grads = torch.autograd.grad(loss, order + [wide, deep])
    flat_g = T.flatten(tuple(g_.reshape(-1) for g_ in grads[:6]), G)
    gw = torch.zeros((G, B), dtype=dtype).scatter_add_(1, il, grads[6].t())
    gd = torch.zeros((G, B, T.D), dtype=dtype).scatter_add_(1, il.unsqueeze(2).expand(G, B, T.D),
                                                             grads[7].permute(1, 0, 2))
    return {"logits": logits.detach(), "loss": loss.detach(), "grads": flat_g, "gsum_wide": gw, "gsum_deep": gd}


def test_first_occurrence_inverse_matches_oracle_unique():
    gen = torch.Generator().manual_seed(3)
    ids = torch.randint(0, 40, (3, 257), generator=gen) * 1000003
    ids[1] = 7  # one id only
    ids[2] = torch.randperm(257, generator=gen)  # all distinct
    inv, n_unique, uniq = T.first_occurrence_inverse(ids)
    for g in range(3):
        u_ref, inv_ref = O.unique_first_occurrence(ids[g].numpy())
        assert int(n_unique[g]) == len(u_ref)
        assert np.array_equal(uniq[g, :len(u_ref)].numpy(), u_ref)
        assert (uniq[g, len(u_ref):] == -1).all()
        assert np.array_equal(inv[g].numpy(), inv_ref)
    inv1, n1, u1 = T.first_occurrence_inverse(ids[0])
    assert torch.equal(inv1, inv[0]) and int(n1) == int(n_unique[0]) and torch.equal(u1, uniq[0])


@pytest.mark.parametrize("G", [1, 5, 38])
@pytest.mark.parametrize("B", [1, 45, 200])
def test_reference_equals_float64_autograd(G, B):
    """Hand-written forward / backward == autograd through DeepFMTower in float64, with duplicated ids: the
    per-unique-id sums equal autograd's per-occurrence gradients summed by inv."""
    inputs = _inputs(G, B, seed=G * 1000 + B)
    ref = T.tower_reference(*inputs)
    want = _autograd(inputs, torch.float64)
    assert int(inputs[1].min()) < B or B == 1  # duplicates present
    for k, w in want.items():
        got = ref[k]
        scale = float(w.abs().max()) if w.numel() else 0.0
        assert torch.allclose(got, w, rtol=1e-12, atol=1e-12 * scale), (k, float((got - w).abs().max()), scale)
    # gsum rows past n_unique are zero in the reference; the padding floats of the flat gradient too
    for g in range(G):
        u = int(inputs[1][g])
        assert (ref["gsum_wide"][g, u:] == 0).all() and (ref["gsum_deep"][g, u:] == 0).all()
    assert (ref["grads"][T.ND:T.WD_PAD] == 0).all()


def test_magnitudes_bound_the_values():
    """|value| <= M everywhere (M sums the absolute values of what makes up the value)."""
    inputs = _inputs(7, 300, seed=11)
    ref = T.tower_reference(*inputs)
    for k in ("logits", "grads", "gsum_wide", "gsum_deep", "h1", "h2"):
        assert (ref[k].abs() <= ref["M"][k] * (1 + 1e-12)).all(), k
    assert abs(float(ref["loss"])) <= float(ref["M"]["loss"])


def _benchmark_batch(B=32768, seed=5):
    """The benchmark's shape: a conditioned Zipf synthetic_batch over the 38 dac_ctr groups (row counts capped
    at 5000 so that the table draws stay small on the host; the id statistics of the batch are what matters)."""
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, synthetic_batch

    rows = [min(r, 5000) for r in GROUP_ROWS]
    G = len(rows)
    ids, dense, labels = synthetic_batch(B, seed, CPU, "zipf", group_rows=rows)
    inv, n_unique, _ = T.first_occurrence_inverse(ids)
    gen = torch.Generator().manual_seed(seed + 1)
    live = torch.arange(B).unsqueeze(0) < n_unique.unsqueeze(1)
    bet_wide = torch.where(live, torch.randn((G, B), generator=gen) * 0.2, torch.tensor(float("nan")))
    bet_deep = torch.where(live.unsqueeze(2), torch.randn((G, B, T.D), generator=gen) * 0.2, torch.tensor(float("nan")))
    params = T.random_params(G, gen, CPU)
    for _ in range(30):
        ref = T.tower_reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params)
        near = T.near_relu_kink(ref)
        if not bool(near.any()):
            break
        dense[near] = torch.randn((int(near.sum()), T.ND), generator=gen)
    else:
        raise AssertionError("conditioning did not converge")
    return (inv, n_unique, bet_wide, bet_deep, dense, labels, params), ref


@pytest.fixture(scope="module")
def bench_case():
    return _benchmark_batch()


def test_fp32_autograd_passes_the_bound(bench_case):
    """An honest fp32 evaluation of the same batch (torch autograd, library GEMMs, different summation
    orders) lies inside the bound everywhere: the tolerance is not tighter than fp32 arithmetic."""
    inputs, ref = bench_case
    got = _autograd(inputs, torch.float32)
    rs = T.check(got, ref, label="fp32 autograd")
    assert all(r <= 1.0 for r in rs.values()), rs


# Which output families reject each fault at B = 32768, G = 38.  A fault that one family cannot see at this
# size (one sample in a sum over 32768 samples is below sqrt(B) rounding) is caught by another:
#   drop_one_sample:         the sample's rare ids put it alone in some per-id rows (gsum); its 1/B share of
#                            the loss and of the parameter gradients is inside the bound
#   last_sample_x32:         31 extra copies of the sample in its own id rows (gsum); in the parameter
#                            gradients they sit near the bound
#   tile_missing_from_grads: 32 samples' share of the parameter gradients (only the gradients change)
#   id_row_missing:          the row itself
#   loss_not_divided_by_B:   the loss
EXPECTED_CATCH = {
    "drop_one_sample": {"gsum_wide", "gsum_deep"},
    "last_sample_x32": {"gsum_wide", "gsum_deep"},
    "tile_missing_from_grads": {"grads"},
    "id_row_missing": {"gsum_wide", "gsum_deep"},
    "loss_not_divided_by_B": {"loss"},
}


def test_mutations_are_rejected_at_the_benchmark_shape(bench_case):
    inputs, ref = bench_case
    assert T.check({k: ref[k] for k in T.FAMILIES}, ref) is not None  # the reference itself passes
    muts = T.mutations(ref, inputs)
    assert set(muts) == set(EXPECTED_CATCH)
    for name, got in muts.items():
        caught = T.caught_by(got, ref)
        assert caught, name
        assert EXPECTED_CATCH[name] <= caught, (name, caught)


def test_conditioning_keeps_preactivations_off_the_kink(bench_case):
    _, ref = bench_case
    assert not bool(T.near_relu_kink(ref).any())
