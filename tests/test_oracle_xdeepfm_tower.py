"""CPU tests of the float64 xDeepFM reference (oracle/xdeepfm_oracle.py) and of its comparator: the hand-written
reference (deepctr's literal CIN) equals float64 autograd through workloads.deepfm.XDeepFMTower, the flat layout
round-trips, the mask override acts only inside its window, an honest evaluation passes the bound and every
mutation is caught at the benchmarked size, and the engine refuses what model="xdeepfm" does not run."""
import pytest
import torch

from oracle import xdeepfm_oracle as X

CPU = torch.device("cpu")


def _inputs(G, B, seed, ids=None, rows_std=0.4):
    gen = torch.Generator(device=CPU).manual_seed(seed)
    if ids is None:  # heavy duplication
        ids = torch.randint(0, max(2, B // 3), (G, B), generator=gen)
    inv, n_unique, _ = X.first_occurrence_inverse(ids)
    bet_wide = torch.full((G, B), float("nan"))
    bet_deep = torch.full((G, B, X.D), float("nan"))
    for g in range(G):
        u = int(n_unique[g])
        bet_wide[g, :u] = torch.randn(u, generator=gen) * rows_std
        bet_deep[g, :u] = torch.randn((u, X.D), generator=gen) * rows_std
    dense = torch.randn((B, X.ND), generator=gen)
    labels = (torch.rand(B, generator=gen) < 0.3).float()
    params = X.random_params(G, gen, CPU)
    return inv, n_unique, bet_wide, bet_deep, dense, labels, params


def _autograd(inputs, dtype):
    """Per-occurrence rows through XDeepFMTower + BCEWithLogitsLoss + regularization(), torch autograd in `dtype`."""
    from elasticdl_b200.workloads.deepfm import XDeepFMTower, flat_order, flatten_tower

    inv, n_unique, bet_wide, bet_deep, dense, labels, params = inputs
    G, B = inv.shape
    tower = XDeepFMTower(G).to(dtype)
    flat = torch.zeros(X.layout(G)["total"], dtype=dtype)
    flatten_tower(tower, flat)
    with torch.no_grad():
        flat.copy_(params.to(dtype))
    il = inv.long()
    wide = torch.gather(bet_wide, 1, il).to(dtype).t().contiguous().requires_grad_(True)
    deep = torch.gather(bet_deep, 1, il.unsqueeze(2).expand(G, B, X.D)).to(dtype).permute(1, 0, 2).contiguous()
    deep.requires_grad_(True)
    logits = tower(dense.to(dtype), wide, deep)
    loss = torch.nn.BCEWithLogitsLoss()(logits, labels.to(dtype)) + tower.regularization()
    order = [p for p, _ in flat_order(tower)]
    grads = torch.autograd.grad(loss, order + [wide, deep])
    flat_g = X.flatten(tuple(g_.reshape(-1) for g_ in grads[:-2]), G)
    gw = torch.zeros((G, B), dtype=dtype).scatter_add_(1, il, grads[-2].t())
    gd = torch.zeros((G, B, X.D), dtype=dtype).scatter_add_(1, il.unsqueeze(2).expand(G, B, X.D),
                                                             grads[-1].permute(1, 0, 2))
    return {"logits": logits.detach(), "loss": loss.detach(), "grads": flat_g, "gsum_wide": gw, "gsum_deep": gd}


def test_flat_layout_round_trips():
    """flat_order / flatten_tower lay XDeepFMTower out as include/b200_deepfm.h documents: Wide & Deep's parameters
    at Wide & Deep's offsets under the same names, then the CIN's; 501,753 floats at G = 38 (496,577 of the CIN)."""
    from elasticdl_b200.workloads.deepfm import WideDeepTower, XDeepFMTower, flat_order, flatten_tower

    for G in (2, 5, 38):
        o = X.layout(G)
        tower = XDeepFMTower(G)
        flat = torch.randn(o["total"])
        views = flatten_tower(tower, torch.zeros(o["total"]))
        assert [off for off, _ in views] == [o[k] for k in ("wd", "w1", "b1", "w2", "b2", "w3", "cin_w0", "cin_b0",
                                                              "cin_w1", "cin_b1", "wex", "bex")]
        assert views[-1][0] + views[-1][1] == o["total"]
        assert views[:6] == flatten_tower(WideDeepTower(G), torch.zeros(X.layout(G)["cin_w0"]))
        names = [n for n, _ in tower.named_parameters()]
        assert [n for n in names if not n.startswith(("cin_", "exfm."))] == \
            [n for n, _ in WideDeepTower(G).named_parameters()]
        flatten_tower(tower, flat)
        parts = X.unflatten(flat, G)
        assert torch.equal(X.flatten(parts, G)[X.WD_PAD:], flat[X.WD_PAD:])
        for p, q in zip([p for p, _ in flat_order(tower)], parts):
            assert torch.equal(p.detach().reshape(-1), q.reshape(-1))
    o = X.layout(38)
    assert o["total"] == 501753 and o["total"] - o["cin_w0"] == 496577


def test_initialization():
    """Filters glorot-uniform over (K, 128), biases zero, exfm glorot-uniform over (192, 1) with a zero bias."""
    from elasticdl_b200.workloads.deepfm import XDeepFMTower

    torch.manual_seed(3)
    t = XDeepFMTower(38)
    for w, k in ((t.cin_w0, 38 * 38), (t.cin_w1, 64 * 38)):
        lim = (6.0 / (k + 128)) ** 0.5
        m = float(w.detach().abs().max())
        assert w.shape == (128, k) and 0.9 * lim < m <= lim
    assert float(t.exfm.weight.detach().abs().max()) <= (6.0 / 193) ** 0.5
    assert not t.cin_b0.any() and not t.cin_b1.any() and not t.exfm.bias.any()


@pytest.mark.parametrize("G", [2, 3, 5])
@pytest.mark.parametrize("B", [1, 45])
def test_reference_equals_float64_autograd(G, B):
    """xdeepfm_reference == autograd through XDeepFMTower in float64 (loss with the L2 term, logits, every parameter
    gradient, the per-unique-id row sums), with duplicated ids, in several chunks."""
    inputs = _inputs(G, B, seed=G * 1000 + B)
    ref = X.xdeepfm_reference(*inputs, chunk=16)
    want = _autograd(inputs, torch.float64)
    for k, w in want.items():
        got = ref[k]
        scale = float(w.abs().max()) if w.numel() else 0.0
        assert torch.allclose(got, w, rtol=1e-11, atol=1e-11 * scale), (k, float((got - w).abs().max()), scale)
    assert float(ref["cin"].std() if B > 1 else 1.0) > 0
    assert (ref["grads"][X.ND:X.WD_PAD] == 0).all()


def test_magnitudes_bound_the_values():
    inputs = _inputs(5, 200, seed=11)
    ref = X.xdeepfm_reference(*inputs, chunk=64)
    for k in ("logits", "grads", "gsum_wide", "gsum_deep", "h1", "h2", "pre0", "pre1"):
        assert (ref[k].abs() <= ref["M"][k] * (1 + 1e-12)).all(), k
    assert abs(float(ref["loss"])) <= float(ref["M"]["loss"])


def test_mask_override_acts_only_near_kinks():
    """Flipped masks change the outputs only where a pre-activation lies inside the tau window."""
    inputs = _inputs(3, 64, seed=5)
    ref = X.xdeepfm_reference(*inputs)
    m0, m1 = ~(ref["pre0"] > 0), ~(ref["pre1"] > 0)
    same = X.xdeepfm_reference(*inputs, mask_override=(m0, m1, 0.0))
    for k in X.KEYS:
        assert torch.equal(same[k], ref[k]), k
    flipped = X.xdeepfm_reference(*inputs, mask_override=(m0, m1, 1.0))
    assert not torch.equal(flipped["logits"], ref["logits"])


def test_decode_masks_reads_the_kernel_layout():
    """Word 4 (h / 16) + 2 ((h / 8) % 2) + d % 2, bit 4 (h % 8) + d / 2, layer 1 in words 32..63."""
    m = torch.zeros((1, 2, 128, 8), dtype=torch.bool)
    m[0, 0, 21, 5] = True
    m[0, 1, 127, 0] = True
    words = torch.zeros((1, 64), dtype=torch.int64)
    words[0, 4 * 1 + 2 * 0 + 1] = 1 << (4 * 5 + 2)
    words[0, 32 + 4 * 7 + 2 * 1 + 0] = 1 << (4 * 7 + 0)
    m0, m1 = X.decode_masks(words)
    assert torch.equal(m0, m[:, 0]) and torch.equal(m1, m[:, 1])


def _benchmark_batch(B=32768, seed=5):
    """A conditioned Zipf batch over the 38 dac_ctr groups (row counts capped at 5000 on the host)."""
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, synthetic_batch

    rows = [min(r, 5000) for r in GROUP_ROWS]
    G = len(rows)
    ids, dense, labels = synthetic_batch(B, seed, CPU, "zipf", group_rows=rows)
    inv, n_unique, _ = X.first_occurrence_inverse(ids)
    gen = torch.Generator().manual_seed(seed + 1)
    live = torch.arange(B).unsqueeze(0) < n_unique.unsqueeze(1)
    bet_wide = torch.where(live, torch.randn((G, B), generator=gen) * 0.2, torch.tensor(float("nan")))
    bet_deep = torch.where(live.unsqueeze(2), torch.randn((G, B, X.D), generator=gen) * 0.4,
                           torch.tensor(float("nan")))
    params = X.random_params(G, gen, CPU)
    inputs = (inv, n_unique, bet_wide, bet_deep, dense, labels, params)
    ref = X.xdeepfm_reference(*inputs)
    mo = (ref["pre0"] > 0, ref["pre1"] > 0, 1e-4)  # the float64 masks stand in for a kernel's
    return inputs, X.xdeepfm_reference(*inputs, mask_override=mo), mo


@pytest.fixture(scope="module")
def bench_case():
    return _benchmark_batch()


def test_mutations_are_rejected_at_the_benchmark_shape(bench_case):
    """B = 32768, G = 38: the reference passes its own bound, the CIN logit moves the logit (its spread is a fair
    share of the whole logit's), and each fault but UNCAUGHT_AT_MAXG's is caught in the families EXPECTED_CATCH
    names."""
    inputs, ref, mo = bench_case
    X.check({k: ref[k] for k in X.KEYS}, ref)
    assert float(ref["cin"].std()) > 0.3 * float(ref["logits"].std())
    muts = X.mutations(ref, inputs, mask_override=mo)
    assert set(muts) == set(X.EXPECTED_CATCH)
    for name, got in muts.items():
        if name in X.UNCAUGHT_AT_MAXG:
            continue
        caught = X.caught_by(got, ref)
        assert X.EXPECTED_CATCH[name] <= caught, (name, caught)


@pytest.mark.parametrize("tower", ["fused", "mma"])
def test_engine_refuses_xdeepfm_on_other_towers(tower):
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    with pytest.raises(ValueError, match="xdeepfm"):
        DeepFMPSEngine(None, 64, group_rows=[10, 20], tower=tower, model="xdeepfm")


@pytest.mark.parametrize("tower", ["tile", "torch"])
def test_engine_refuses_xdeepfm_outside_2_to_38_groups(tower):
    """One group (the reference builds a different model without a CIN) and 39 (the tile tower's limit) are refused
    before the parameter server is touched (group=None would fail on first use)."""
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine

    with pytest.raises(ValueError, match="model"):
        DeepFMPSEngine(None, 64, group_rows=[10], tower=tower, model="xdeepfm")
    with pytest.raises(ValueError, match="38"):
        DeepFMPSEngine(None, 64, group_rows=[10] * 39, tower=tower, model="xdeepfm")
