"""CPU tests of the float64 DCN tower reference (oracle/dcn_oracle.py) and of its comparator: the hand-written
reference (the literal cross-layer recursion) equals float64 autograd through workloads.deepfm.DCNTower, the
closed form the CUDA tower computes equals the recursion, an honest fp32 evaluation passes the bound, the classic
tiled-reduction faults fail it, and the engine refuses what model="dcn" does not run."""
import pytest
import torch

from oracle import dcn_oracle as R

CPU = torch.device("cpu")


def _inputs(G, B, seed, rows_std=0.3):
    gen = torch.Generator(device=CPU).manual_seed(seed)
    ids = torch.randint(0, max(2, B // 3), (G, B), generator=gen)  # heavy duplication
    inv, n_unique, _ = R.first_occurrence_inverse(ids)
    bet_wide = torch.full((G, B), float("nan"))
    bet_deep = torch.full((G, B, R.D), float("nan"))
    for g in range(G):
        u = int(n_unique[g])
        bet_wide[g, :u] = torch.randn(u, generator=gen) * rows_std
        bet_deep[g, :u] = torch.randn((u, R.D), generator=gen) * rows_std
    dense = torch.randn((B, R.ND), generator=gen)
    labels = (torch.rand(B, generator=gen) < 0.3).float()
    params = R.random_params(G, gen, CPU)
    return inv, n_unique, bet_wide, bet_deep, dense, labels, params


def _autograd(inputs, dtype):
    """Per-occurrence rows through DCNTower + BCEWithLogitsLoss + its l2 term, torch autograd in `dtype`."""
    from elasticdl_b200.workloads.deepfm import DCNTower, flat_order, flatten_tower

    inv, n_unique, bet_wide, bet_deep, dense, labels, params = inputs
    G, B = inv.shape
    tower = DCNTower(G).to(dtype)
    flat = torch.zeros(R.layout(G)["total"], dtype=dtype)
    flatten_tower(tower, flat)
    with torch.no_grad():
        flat.copy_(params.to(dtype))
    il = inv.long()
    wide = torch.gather(bet_wide, 1, il).to(dtype).t().contiguous().requires_grad_(True)
    deep = torch.gather(bet_deep, 1, il.unsqueeze(2).expand(G, B, R.D)).to(dtype).permute(1, 0, 2).contiguous()
    deep.requires_grad_(True)
    logits = tower(dense.to(dtype), wide, deep)
    loss = torch.nn.BCEWithLogitsLoss()(logits, labels.to(dtype)) + tower.regularization()
    order = [p for p, _ in flat_order(tower)]
    grads = torch.autograd.grad(loss, order + [wide, deep])
    flat_g = R.flatten(tuple(g_.reshape(-1) for g_ in grads[:-2]), G)
    gw = torch.zeros((G, B), dtype=dtype).scatter_add_(1, il, grads[-2].t())
    gd = torch.zeros((G, B, R.D), dtype=dtype).scatter_add_(1, il.unsqueeze(2).expand(G, B, R.D),
                                                             grads[-1].permute(1, 0, 2))
    return {"logits": logits.detach(), "loss": loss.detach(), "grads": flat_g, "gsum_wide": gw, "gsum_deep": gd}


def test_flat_layout_matches_the_header():
    """flatten_tower(DCNTower) lays the parameters out as include/b200_deepfm.h documents (dcn_oracle.layout)."""
    from elasticdl_b200.workloads.deepfm import DCNTower, flat_order, flatten_tower

    for G in (1, 5, 38):
        tower = DCNTower(G)
        n = R.layout(G)["total"]
        flat = torch.zeros(n)
        views = flatten_tower(tower, flat)
        o = R.layout(G)
        assert [off for off, _ in views] == [o[k] for k in ("wd", "w1", "b1", "w2", "b2", "wout", "cw", "cb")]
        assert views[-1][0] + views[-1][1] == n
        assert [p.shape for p, _ in flat_order(tower)][-3:] == [(1, 4 + o["in"]), (2, o["in"]), (2, o["in"])]


@pytest.mark.parametrize("G", [1, 5, 38])
@pytest.mark.parametrize("B", [1, 45, 200])
def test_reference_equals_float64_autograd(G, B):
    """Hand-written forward / backward == autograd through DCNTower in float64 (loss with its l2 term, logits,
    every parameter gradient, the per-unique-id row sums), with duplicated ids."""
    inputs = _inputs(G, B, seed=G * 1000 + B)
    ref = R.dcn_reference(*inputs)
    want = _autograd(inputs, torch.float64)
    for k, w in want.items():
        got = ref[k]
        scale = float(w.abs().max()) if w.numel() else 0.0
        assert torch.allclose(got, w, rtol=1e-12, atol=1e-12 * scale), (k, float((got - w).abs().max()), scale)
    for g in range(G):
        u = int(inputs[1][g])
        assert (ref["gsum_wide"][g, u:] == 0).all() and (ref["gsum_deep"][g, u:] == 0).all()
    assert (ref["grads"][R.ND:R.WD_PAD] == 0).all()


@pytest.mark.parametrize("G", [1, 5, 38])
def test_closed_form_equals_the_recursion(G):
    """((1 + a)(1 + c) + beta) e + gamma == w_out_cross . x_2 of the layer recursion, for nonzero biases."""
    inputs = _inputs(G, 300, seed=7 + G)
    ref = R.dcn_reference(*inputs)
    _, _, _, _, _, wout, cw, cb = (t.double() for t in R.unflatten(inputs[6], G))
    wc = wout[R.H2:]
    x0 = torch.cat([inputs[4].double(), torch.gather(inputs[3], 1, inputs[0].long().unsqueeze(2).expand(
        G, 300, R.D)).double().permute(1, 0, 2).reshape(300, -1)], 1)
    assert float(cb.abs().min()) > 0
    want = ref["x2"] @ wc
    got = R.closed_form(x0, cw, cb, wc)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12 * float(want.abs().max()))
    # x_2 itself: x0 ((1 + a)(1 + c) + beta) + b0 + b1
    a, c = x0 @ cw[0], x0 @ cw[1]
    K = (1 + a) * (1 + c) + cb[0] @ cw[1]
    assert torch.allclose(ref["x2"], x0 * K.unsqueeze(1) + cb[0] + cb[1], rtol=1e-12, atol=1e-12)


def test_magnitudes_bound_the_values():
    inputs = _inputs(7, 300, seed=11)
    ref = R.dcn_reference(*inputs)
    for k in ("logits", "grads", "gsum_wide", "gsum_deep", "h1", "h2"):
        assert (ref[k].abs() <= ref["M"][k] * (1 + 1e-12)).all(), k
    assert abs(float(ref["loss"])) <= float(ref["M"]["loss"])


def _benchmark_batch(B=32768, seed=5):
    """A conditioned Zipf batch over the 38 dac_ctr groups (row counts capped at 5000 on the host)."""
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, synthetic_batch

    rows = [min(r, 5000) for r in GROUP_ROWS]
    G = len(rows)
    ids, dense, labels = synthetic_batch(B, seed, CPU, "zipf", group_rows=rows)
    inv, n_unique, _ = R.first_occurrence_inverse(ids)
    gen = torch.Generator().manual_seed(seed + 1)
    live = torch.arange(B).unsqueeze(0) < n_unique.unsqueeze(1)
    bet_wide = torch.where(live, torch.randn((G, B), generator=gen) * 0.2, torch.tensor(float("nan")))
    bet_deep = torch.where(live.unsqueeze(2), torch.randn((G, B, R.D), generator=gen) * 0.2, torch.tensor(float("nan")))
    params = R.random_params(G, gen, CPU)
    for _ in range(30):
        ref = R.dcn_reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params)
        near = R.near_relu_kink(ref)
        if not bool(near.any()):
            break
        dense[near] = torch.randn((int(near.sum()), R.ND), generator=gen)
    else:
        raise AssertionError("conditioning did not converge")
    return (inv, n_unique, bet_wide, bet_deep, dense, labels, params), ref


@pytest.fixture(scope="module")
def bench_case():
    return _benchmark_batch()


def test_fp32_autograd_passes_the_bound(bench_case):
    """An honest fp32 evaluation (torch autograd through the recursion, library GEMMs) lies inside the bound."""
    inputs, ref = bench_case
    rs = R.check(_autograd(inputs, torch.float32), ref, label="fp32 autograd")
    assert all(r <= 1.0 for r in rs.values()), rs


def test_mutations_are_rejected_at_the_benchmark_shape(bench_case):
    inputs, ref = bench_case
    R.check({k: ref[k] for k in R.FAMILIES}, ref)
    expected = {"drop_one_sample": {"gsum_wide", "gsum_deep"}, "last_sample_x32": {"gsum_wide", "gsum_deep"},
                "tile_missing_from_grads": {"grads"}, "id_row_missing": {"gsum_wide", "gsum_deep"},
                "loss_not_divided_by_B": {"loss"}}
    muts = R.mutations(ref, inputs)
    assert set(muts) == set(expected)
    for name, got in muts.items():
        caught = R.caught_by(got, ref)
        assert expected[name] <= caught, (name, caught)


@pytest.mark.parametrize("tower", ["fused", "mma"])
def test_engine_refuses_dcn_on_other_towers(tower):
    """model="dcn" runs on the tile tower (or torch): the other CUDA towers compute DeepFM only, and the engine
    raises before it touches the parameter server rather than fall back."""
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    with pytest.raises(ValueError, match="dcn"):
        DeepFMPSEngine(None, 64, group_rows=[10, 20], tower=tower, model="dcn")


def test_engine_refuses_dcn_past_38_groups_and_unknown_models():
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    for tower in ("tile", "torch"):
        with pytest.raises(ValueError, match="38"):
            DeepFMPSEngine(None, 64, group_rows=[10] * 39, tower=tower, model="dcn")
    with pytest.raises(ValueError, match="model"):
        DeepFMPSEngine(None, 64, group_rows=[10], model="xdeepfm")
