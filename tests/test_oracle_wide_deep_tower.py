"""CPU tests of the float64 Wide & Deep reference (oracle/wide_deep_oracle.py) and of its comparator: the
hand-written reference equals float64 autograd through workloads.deepfm.WideDeepTower, DeepFM (oracle/tower_oracle.py)
minus Wide & Deep is the FM term and its row gradient alone, an honest fp32 evaluation passes the bound, the classic
tiled-reduction faults fail it, and the engine refuses what model="wide_deep" does not run."""
import pytest
import torch

from oracle import tower_oracle as T
from oracle import wide_deep_oracle as W

CPU = torch.device("cpu")


def _inputs(G, B, seed, ids=None, rows_std=0.3):
    gen = torch.Generator(device=CPU).manual_seed(seed)
    if ids is None:  # heavy duplication
        ids = torch.randint(0, max(2, B // 3), (G, B), generator=gen)
    inv, n_unique, _ = T.first_occurrence_inverse(ids)
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
    """Per-occurrence rows through WideDeepTower + BCEWithLogitsLoss, torch autograd in `dtype`."""
    from elasticdl_b200.workloads.deepfm import WideDeepTower, flat_order, flatten_tower

    inv, n_unique, bet_wide, bet_deep, dense, labels, params = inputs
    G, B = inv.shape
    tower = WideDeepTower(G).to(dtype)
    flat = torch.zeros(T.layout(G)["total"], dtype=dtype)
    flatten_tower(tower, flat)
    with torch.no_grad():
        flat.copy_(params.to(dtype))
    il = inv.long()
    wide = torch.gather(bet_wide, 1, il).to(dtype).t().contiguous().requires_grad_(True)
    deep = torch.gather(bet_deep, 1, il.unsqueeze(2).expand(G, B, T.D)).to(dtype).permute(1, 0, 2).contiguous()
    deep.requires_grad_(True)
    logits = tower(dense.to(dtype), wide, deep)
    loss = torch.nn.BCEWithLogitsLoss()(logits, labels.to(dtype))
    order = [p for p, _ in flat_order(tower)]
    grads = torch.autograd.grad(loss, order + [wide, deep])
    flat_g = T.flatten(tuple(g_.reshape(-1) for g_ in grads[:-2]), G)
    gw = torch.zeros((G, B), dtype=dtype).scatter_add_(1, il, grads[-2].t())
    gd = torch.zeros((G, B, T.D), dtype=dtype).scatter_add_(1, il.unsqueeze(2).expand(G, B, T.D),
                                                             grads[-1].permute(1, 0, 2))
    return {"logits": logits.detach(), "loss": loss.detach(), "grads": flat_g, "gsum_wide": gw, "gsum_deep": gd}


def test_flat_layout_is_deepfms():
    """WideDeepTower has DeepFMTower's parameters under the same names: flatten_tower lays them out as
    include/b200_deepfm.h documents for DeepFM, b200_deepfm_param_count's size."""
    from elasticdl_b200.workloads.deepfm import DeepFMTower, WideDeepTower, flat_order, flatten_tower

    for G in (1, 5, 38):
        o = T.layout(G)
        views = flatten_tower(WideDeepTower(G), torch.zeros(o["total"]))
        assert [off for off, _ in views] == [o[k] for k in ("wd", "w1", "b1", "w2", "b2", "w3")]
        assert views[-1][0] + views[-1][1] == o["total"]
        assert views == flatten_tower(DeepFMTower(G), torch.zeros(o["total"]))
        assert [n for n, _ in WideDeepTower(G).named_parameters()] == [n for n, _ in DeepFMTower(G).named_parameters()]
        assert [p.shape for p, _ in flat_order(WideDeepTower(G))] == [p.shape for p, _ in flat_order(DeepFMTower(G))]


@pytest.mark.parametrize("G", [1, 5, 38])
@pytest.mark.parametrize("B", [1, 45, 200])
def test_reference_equals_float64_autograd(G, B):
    """wide_deep_reference == autograd through WideDeepTower in float64 (loss, logits, every parameter
    gradient, the per-unique-id row sums), with duplicated ids."""
    inputs = _inputs(G, B, seed=G * 1000 + B)
    ref = W.wide_deep_reference(*inputs)
    want = _autograd(inputs, torch.float64)
    for k, w in want.items():
        got = ref[k]
        scale = float(w.abs().max()) if w.numel() else 0.0
        assert torch.allclose(got, w, rtol=1e-12, atol=1e-12 * scale), (k, float((got - w).abs().max()), scale)
    for g in range(G):
        u = int(inputs[1][g])
        assert (ref["gsum_wide"][g, u:] == 0).all() and (ref["gsum_deep"][g, u:] == 0).all()
    assert (ref["grads"][T.ND:T.WD_PAD] == 0).all()


@pytest.mark.parametrize("G", [1, 5, 38])
def test_fm_minus_wide_deep_is_the_fm_term_alone(G):
    """Every id distinct, so gsum rows are per-sample rows and gsum_wide[g, b] is the sample's dz.  DeepFM's logit
    minus Wide & Deep's is the FM term 0.5 (|s|^2 - sum |e|^2); a deep row's gradient, once Wide & Deep's is scaled
    to DeepFM's dz (the DNN part is linear in dz and both share the ReLU masks), differs by dz (s - e) alone; and
    the logit's magnitude by the FM term's."""
    B = 300
    ids = torch.stack([torch.randperm(B, generator=torch.Generator().manual_seed(g)) for g in range(G)])
    inputs = _inputs(G, B, seed=50 + G, ids=ids)
    fm, wd = T.tower_reference(*inputs), W.wide_deep_reference(*inputs)
    inv = inputs[0].long()
    deep = torch.gather(inputs[3], 1, inv.unsqueeze(2).expand(G, B, T.D)).double()  # [G, B, 8] per sample
    s = deep.sum(0)
    fm_term = 0.5 * ((s * s).sum(1) - (deep * deep).sum((0, 2)))
    assert torch.allclose(fm["logits"] - wd["logits"], fm_term, rtol=0, atol=1e-12)
    assert torch.equal(fm["h1"], wd["h1"]) and torch.equal(fm["h2"], wd["h2"])
    # per-sample rows in sample order
    per_sample = {k: torch.gather(r["gsum_deep"], 1, inv.unsqueeze(2).expand(G, B, T.D)) for k, r in
                  (("fm", fm), ("wd", wd))}
    dz_fm = torch.gather(fm["gsum_wide"], 1, inv)[0]
    dz_wd = torch.gather(wd["gsum_wide"], 1, inv)[0]
    assert bool((dz_wd != 0).all())
    scaled = per_sample["wd"] * (dz_fm / dz_wd).view(1, B, 1)
    want = dz_fm.view(1, B, 1) * (s.unsqueeze(0) - deep)
    assert torch.allclose(per_sample["fm"] - scaled, want, rtol=0, atol=1e-12 * float(per_sample["fm"].abs().max()))
    Ms = deep.abs().sum(0)
    M_fm = 0.5 * ((Ms * Ms).sum(1) + (deep * deep).sum((0, 2)))
    assert torch.allclose(fm["M"]["logits"] - wd["M"]["logits"], M_fm, rtol=1e-12, atol=1e-12)


def test_magnitudes_bound_the_values():
    inputs = _inputs(7, 300, seed=11)
    ref = W.wide_deep_reference(*inputs)
    for k in ("logits", "grads", "gsum_wide", "gsum_deep", "h1", "h2"):
        assert (ref[k].abs() <= ref["M"][k] * (1 + 1e-12)).all(), k
    assert abs(float(ref["loss"])) <= float(ref["M"]["loss"])


def _benchmark_batch(B=32768, seed=5):
    """A conditioned Zipf batch over the 38 dac_ctr groups (row counts capped at 5000 on the host)."""
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
        ref = W.wide_deep_reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params)
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
    """An honest fp32 evaluation (torch autograd through WideDeepTower, library GEMMs) lies inside the bound."""
    inputs, ref = bench_case
    rs = T.check(_autograd(inputs, torch.float32), ref, label="fp32 autograd")
    assert all(r <= 1.0 for r in rs.values()), rs


def test_mutations_are_rejected_at_the_benchmark_shape(bench_case):
    """The same faults are caught in the same families as DeepFM's (test_oracle_tower.EXPECTED_CATCH) with the
    FM term's share gone from every bound."""
    inputs, ref = bench_case
    T.check({k: ref[k] for k in T.FAMILIES}, ref)
    expected = {"drop_one_sample": {"gsum_wide", "gsum_deep"}, "last_sample_x32": {"gsum_wide", "gsum_deep"},
                "tile_missing_from_grads": {"grads"}, "id_row_missing": {"gsum_wide", "gsum_deep"},
                "loss_not_divided_by_B": {"loss"}}
    muts = W.mutations(ref, inputs)
    assert set(muts) == set(expected)
    for name, got in muts.items():
        caught = T.caught_by(got, ref)
        assert expected[name] <= caught, (name, caught)


@pytest.mark.parametrize("tower", ["fused", "mma"])
def test_engine_refuses_wide_deep_on_other_towers(tower):
    """model="wide_deep" runs on the tile tower (or torch): the fused and mma towers compute DeepFM only, and the
    engine raises before it touches the parameter server rather than train DeepFM."""
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    with pytest.raises(ValueError, match="wide_deep"):
        DeepFMPSEngine(None, 64, group_rows=[10, 20], tower=tower, model="wide_deep")


def test_engine_refuses_wide_deep_past_38_groups():
    """39 groups are refused on the tile and torch towers alike: the tile tower's fall-back to the fused tower past
    38 groups would train DeepFM instead."""
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    for tower in ("tile", "torch"):
        with pytest.raises(ValueError, match="38"):
            DeepFMPSEngine(None, 64, group_rows=[10] * 39, tower=tower, model="wide_deep")
