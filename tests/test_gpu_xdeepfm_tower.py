"""The xDeepFM tile tower (csrc/xdeepfm_cin.cu + the Wide & Deep tile kernel's CIN instance, include/b200_deepfm.h
b200_deepfm_xdeepfm_*) against the float64 reference of oracle/xdeepfm_oracle.py.

Kernel level, through the C ABI (no PS), every output and the scratch buffer poisoned with NaN before each call:
G in {2, 3, 5, 13, 38} (K of layer 0 not a multiple of 8), batches at the tile edge, past one wave of CTAs and at
32768, both row sources, prologue + main against one call, forward-only logits, the mutations and the refusals.
Batches are conditioned as in test_gpu_wide_deep_tower.py for the DNN's kinks; the CIN's kinks cannot be moved (its
units depend on the shared deep rows only), so the kernel's own mask bits must equal pre > 0 wherever the float64
pre-activation lies outside tau * M of 0, and inside that window the reference takes the kernel's bits.

Engine level: DeepFMPSEngine(model="xdeepfm") for three Adam steps at B = 32768 on bench.py's Zipf batches through
the graphed lookahead feed on narrow packed ids, every step's dedup, loss, gradients and push checked; predict();
graphed against eager steps; and tower="torch" against "tile" over the same batches."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import ps_oracle as O
from oracle import xdeepfm_oracle as X
from tests.test_gpu_tower_reference import NAN, Buffers, _batch, _ids, _n_sm

pytestmark = pytest.mark.gpu
TAU = 1e-4
WORST = {}


def _dev():
    return torch.device("cuda", 0)


def _lib():
    from elasticdl_b200 import _lib

    return _lib.lib()


def mask_offset(G, B):
    """include/b200_deepfm.h scratch layout (csrc/xdeepfm.cuh CinScratch): the float offset of the mask words."""
    hp0 = -(-G // 8) * 8
    k0, k1 = G * hp0, 64 * G
    k0b = -(-k0 // 16) * 16
    bp = -(-B // 4) * 4
    o_wf0 = 320 * 16 + 16 + 2 * bp + 16
    return o_wf0 + 128 * (k0 + k1 + k0b + k1) + 192 * B


def kernel_masks(scratch, G, B):
    o = mask_offset(G, B)
    return X.decode_masks(scratch[o:o + 64 * B].view(torch.int32).view(B, 64))


class XBuffers(Buffers):
    def __init__(self, G, B):
        super().__init__(G, B)
        self.params = torch.empty(X.layout(G)["total"], dtype=torch.float32, device=_dev())
        self.grads = torch.empty_like(self.params)
        self.scratch = torch.empty(int(_lib().b200_deepfm_xdeepfm_scratch_floats(G, B)), dtype=torch.float32,
                                   device=_dev())


# Value regimes: Wide & Deep's (test_gpu_wide_deep_tower.py) and the CIN's own.  dead_cin: b_0 = -100 kills every
# layer-0 channel, so X_1 = 0 and layer 1 sees pre1 = b_1 < 0 (dead too), and b_ex = 0: the CIN adds nothing and
# the tower is Wide & Deep.  half_dead_cin: b_0[:64] = -100 kills X_1 only, the direct half of layer 0 lives and
# layer 1's live channels see pre1 = b_1 > 0.  strong_cin: filters 3 times the initializer's and deep rows of
# scale 1 make the CIN logit dominate, with the Wide & Deep DNN's first layer small (w1_gain 0.1).
REGIMES = ("base", "large_logit", "dead_l1", "soft", "dead_cin", "half_dead_cin", "strong_cin")


def make_inputs(G, B, pattern="zipf", seed=0, regime="base"):
    """Device inputs of one batch in the kernel's layout, conditioned on the DNN's kinks; rows past n_unique[g] and
    the parameters' padding are NaN.  Returns (inputs, float64 reference without a mask override)."""
    dev = _dev()
    gen = torch.Generator(device=dev).manual_seed(5000 + seed)
    ids = _ids(pattern, G, B, seed, gen)
    inv, n_unique, _ = X.first_occurrence_inverse(ids)
    sw = 0.5 * (5.0 / max(G, 5)) ** 0.5
    sd = 1.0 if regime == "strong_cin" else 0.5
    live = torch.arange(B, device=dev).unsqueeze(0) < n_unique.unsqueeze(1).long()
    bet_wide = torch.where(live, torch.randn((G, B), generator=gen, device=dev) * sw, NAN).contiguous()
    bet_deep = torch.where(live.unsqueeze(2), torch.randn((G, B, X.D), generator=gen, device=dev) * sd, NAN)
    bet_deep = bet_deep.contiguous()
    dense = torch.randn((B, X.ND), generator=gen, device=dev)
    if regime == "soft":
        labels = torch.rand(B, generator=gen, device=dev)
    else:
        labels = (torch.rand(B, generator=gen, device=dev) < 0.25).float()
    kw = {}
    if regime == "large_logit":
        kw["wd_std"] = 6.0
    if regime == "dead_l1":
        kw.update(b1=-100.0, b2=[0.5, -0.5, 0.7, 0.3])
    if regime == "strong_cin":
        kw.update(cin_gain=3.0, w1_gain=0.1)
    params = X.random_params(G, gen, dev, pad=NAN, **kw)
    o = X.layout(G)
    if regime == "dead_cin":
        params[o["cin_b0"]:o["cin_w1"]] = -100.0
        params[o["cin_b1"]:o["wex"]] = -0.05 - 0.1 * torch.rand(X.CIN_H, generator=gen, device=dev)
        params[o["bex"]] = 0.0
    if regime == "half_dead_cin":
        params[o["cin_b0"]:o["cin_b0"] + X.HALF] = -100.0
    for _ in range(40):
        ref = X.xdeepfm_reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params, chunk=4096)
        near = X.near_relu_kink(ref, TAU)
        if not bool(near.any()):
            break
        dense[near] = torch.randn((int(near.sum()), X.ND), generator=gen, device=dev)
    else:
        raise AssertionError("conditioning did not converge")
    if regime == "large_logit" and B >= 1000:
        assert float(ref["logits"].abs().max()) > 50
    return (inv, n_unique, bet_wide, bet_deep, dense, labels, params), ref


def reference_with_kernel_masks(inputs, ref, scratch, label):
    """The kernel's mask bits equal pre > 0 outside the tau window; the reference with them inside it."""
    G, B = inputs[0].shape
    km = kernel_masks(scratch, G, B)
    near = X.near_cin_kink(ref, TAU)
    for k in (0, 1):
        bad = (km[k] != (ref["pre%d" % k] > 0)) & ~near[k]
        assert not bool(bad.any()), "%s: layer %d mask bits wrong at %s" % (label, k, bad.nonzero()[:4].tolist())
    ref = X.xdeepfm_reference(*inputs, mask_override=(km[0], km[1], TAU), chunk=4096)
    ref["kernel_masks"] = km
    return ref


def _call(kind, a):
    L = _lib()
    st = torch.cuda.current_stream().cuda_stream
    p = ctypes.byref(a)
    if kind == "split":
        rc = L.b200_deepfm_xdeepfm_tile_prologue(p, st)
        return rc or L.b200_deepfm_xdeepfm_tile_main(p, st)
    return {"tile": L.b200_deepfm_xdeepfm_fwd_bwd_tile, "forward": L.b200_deepfm_xdeepfm_forward_tile}[kind](p, st)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nxDeepFM tile tower, largest err / bound per output family (%s, %d SMs):" % (
            torch.cuda.get_device_name(0), _n_sm()))
        for (kind, fam), r in sorted(WORST.items()):
            print("  %-19s %-10s %.4f" % (kind, fam, r))


def _outputs(buf):
    return {"logits": buf.logits, "loss": buf.loss, "grads": buf.grads, "gsum_wide": buf.gsum_wide,
            "gsum_deep": buf.gsum_deep}


def run_and_check(kind, G, B, pattern="zipf", seed=0, table_rows=False, regime="base"):
    buf = XBuffers(G, B)
    backward = kind != "forward"
    inputs, ref = make_inputs(G, B, pattern, seed, regime)
    buf.load(inputs)
    a = buf.args(backward)
    group = None
    if table_rows:
        from tests.test_gpu_tower_table_rows import ADAM, _rows_struct, _table_state

        group, uniq = _table_state(ADAM, inputs, seed)
        rows = _rows_struct(group, G, uniq)
        buf.bet_wide.fill_(NAN)
        buf.bet_deep.fill_(NAN)
        a.rows = ctypes.pointer(rows)
    try:
        before = _lib().b200_deepfm_xdeepfm_launch_count()
        rc = _call(kind, a)
        assert rc == 0, (kind, rc, _lib().b200_deepfm_last_error())
        torch.cuda.synchronize()
        assert _lib().b200_deepfm_xdeepfm_launch_count() - before == (6 if backward else 4)
    finally:
        if group is not None:
            group.close()
    label = "xdeepfm %s G=%d B=%d %s/%s%s:" % (kind, G, B, pattern, regime, " table" if table_rows else "")
    if not backward:  # the forward stores no masks: its logits must equal the training call's (the same code)
        return inputs, ref, {f: v.clone() for f, v in _outputs(buf).items()}
    ref = reference_with_kernel_masks(inputs, ref, buf.scratch, label)
    fams = X.FAMILIES
    rs = X.check({f: v for f, v in _outputs(buf).items() if f in fams}, ref, families=fams, label=label,
                 n_sm=_n_sm())
    for fam, r in rs.items():
        key = kind if regime == "base" else "%s/%s" % (kind, regime)
        WORST[(key, fam)] = max(WORST.get((key, fam), 0.0), r)
    if backward:
        dead = torch.arange(B, device=_dev()).unsqueeze(0) >= inputs[1].unsqueeze(1).long()
        assert torch.isnan(buf.gsum_wide[dead]).all() and torch.isnan(buf.gsum_deep[dead]).all(), label
    return inputs, ref, {f: v.clone() for f, v in _outputs(buf).items()}


@pytest.mark.parametrize("B", ["1", "31", "33", "tile_wave2", "32768"])
@pytest.mark.parametrize("G", [2, 3, 5, 13, 38])
def test_xdeepfm_tower_shapes(G, B):
    run_and_check("tile", G, _batch(B), seed=G)


@pytest.mark.parametrize("pattern", ["equal", "distinct", "lanes", "straddle"])
def test_xdeepfm_tower_id_patterns(pattern):
    run_and_check("tile", 38, _batch("tile_wave2"), pattern=pattern, seed=11)


@pytest.mark.parametrize("B", ["33", "32768"])
@pytest.mark.parametrize("G", [5, 38])
def test_xdeepfm_tower_table_rows(G, B):
    """Rows straight from the table records (NaN in bet_*)."""
    run_and_check("tile", G, _batch(B), seed=41, table_rows=True)


@pytest.mark.parametrize("B", ["33", "32768"])
def test_xdeepfm_split_prologue_main_equals_one_call(B):
    Bn = _batch(B)
    split = run_and_check("split", 38, Bn, seed=3)
    one = run_and_check("tile", 38, Bn, seed=3)
    assert torch.equal(split[2]["logits"], one[2]["logits"])


@pytest.mark.parametrize("B", ["33", "tile_wave2", "32768"])
@pytest.mark.parametrize("G", [5, 38])
def test_xdeepfm_forward_only(G, B):
    """Forward-only logits equal bit for bit to the training call's, which are checked against the reference."""
    Bn = _batch(B)
    fwd = run_and_check("forward", G, Bn, seed=31)
    one = run_and_check("tile", G, Bn, seed=31)
    assert torch.equal(fwd[2]["logits"], one[2]["logits"])


@pytest.mark.parametrize("B", ["1000", "32768"])
@pytest.mark.parametrize("regime", REGIMES)
def test_xdeepfm_tower_value_regimes(regime, B):
    """Every regime within the bound, with the kernel's mask bits equal to pre > 0 outside the tau window; the
    regimes' exact outputs besides.  dead_l1: Wide & Deep's hidden-layer gradients are 0.  dead_cin: the CIN filter
    gradients are exactly the prologue's fp32 L2 term 2e-5f W, its bias and w_ex gradients 0, and the logits and
    row sums are Wide & Deep's within Wide & Deep's (tighter) bound.  half_dead_cin: dW_1 is exactly its L2 term
    (Z_1 = X0 X_1 = 0).  strong_cin: the CIN logit dominates."""
    from oracle import wide_deep_oracle as WD

    G, Bn = 38, _batch(B)
    inputs, ref, got = run_and_check("tile", G, Bn, seed=21, regime=regime)
    label = "xdeepfm G=%d B=%d %s" % (G, Bn, regime)
    o = X.layout(G)
    p, g = inputs[6], got["grads"]

    def l2(a, b):
        return p[o[a]:o[b]] * torch.tensor(2e-5, dtype=torch.float32, device=p.device)

    if regime == "dead_l1":
        assert (g[o["w1"]:o["w2"] + X.H2 * X.H1] == 0).all(), label
    if regime in ("dead_cin", "half_dead_cin"):
        assert not ref["pre0"][:, :X.HALF].gt(0).any()
        assert torch.equal(g[o["cin_w1"]:o["cin_b1"]], l2("cin_w1", "cin_b1")), label
    if regime == "half_dead_cin":
        assert ref["pre0"][:, X.HALF:].gt(0).any() and ref["pre1"].gt(0).any()
    if regime == "dead_cin":
        assert not ref["pre0"].gt(0).any() and not ref["pre1"].gt(0).any()
        assert torch.equal(g[o["cin_w0"]:o["cin_b0"]], l2("cin_w0", "cin_b0")), label
        for a, b in (("cin_b0", "cin_w1"), ("cin_b1", "wex"), ("wex", "bex")):
            assert (g[o[a]:o[b]] == 0).all(), (label, a)
        wd = WD.wide_deep_reference(*inputs[:6], p[:o["cin_w0"]])
        fams = ("logits", "gsum_wide", "gsum_deep")
        rs = WD.check({f: got[f] for f in fams}, wd, families=fams, label=label + " vs Wide & Deep", n_sm=_n_sm())
        for fam, r in rs.items():
            WORST[("tile/dead_cin vs W&D", fam)] = max(WORST.get(("tile/dead_cin vs W&D", fam), 0.0), r)
    if regime == "strong_cin":
        assert float(ref["cin"].std()) > 3 * float((ref["logits"] - ref["cin"]).std()), label


def test_xdeepfm_cin_logit_is_not_hidden():
    """At the benchmarked shape the CIN logit's spread is a fair share of the whole logit's, so that an error in it
    is not hidden under the rest of the logit's bound."""
    _, ref, _ = run_and_check("tile", 38, 32768, seed=77)
    assert float(ref["cin"].std()) > 0.3 * float(ref["logits"].std())


@pytest.mark.parametrize("B", ["33", "32768"])
@pytest.mark.parametrize("G", [2, 38])
def test_xdeepfm_mutations_are_caught(G, B):
    """Each fault of xdeepfm_oracle.mutations lies outside the bound the kernel passes, in the families it is
    expected in (at 38 groups, all but UNCAUGHT_AT_MAXG's)."""
    Bn = _batch(B)
    inputs, ref, _ = run_and_check("tile", G, Bn, seed=G + 100)
    for name, got in X.mutations(ref, inputs).items():
        if G == 38 and name in X.UNCAUGHT_AT_MAXG:
            continue
        caught = X.caught_by(got, ref, n_sm=_n_sm())
        assert X.EXPECTED_CATCH[name] <= caught, (name, G, Bn, caught)


@pytest.mark.parametrize("G", [2, 38])
def test_xdeepfm_prologue_writes_the_l2_term(G):
    """The prologue alone leaves the CIN filters' gradients at 2e-5 W (every other CIN gradient 0) and the loss at
    1e-5 (|W_0|^2 + |W_1|^2), to fp32 rounding."""
    buf = XBuffers(G, 64)
    inputs, _ = make_inputs(G, 64, seed=G + 7)
    buf.load(inputs)
    assert _lib().b200_deepfm_xdeepfm_tile_prologue(ctypes.byref(buf.args(True)),
                                                    torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    o = X.layout(G)
    p = buf.params.double()
    want = torch.zeros(o["total"] - o["cin_w0"], dtype=torch.float64, device=_dev())
    for a_, b_ in (("cin_w0", "cin_b0"), ("cin_w1", "cin_b1")):
        want[o[a_] - o["cin_w0"]:o[b_] - o["cin_w0"]] = 2e-5 * p[o[a_]:o[b_]]
    assert torch.allclose(buf.grads[o["cin_w0"]:].double(), want, rtol=2 ** -22, atol=0)
    reg = 1e-5 * ((p[o["cin_w0"]:o["cin_b0"]] ** 2).sum() + (p[o["cin_w1"]:o["cin_b1"]] ** 2).sum())
    assert abs(float(buf.loss) - float(reg)) <= 1e-5 * float(reg)


def test_xdeepfm_refusals():
    """G = 1 and G = 39, a row source on the forward-only entry and a null scratch are refused (-1) by every entry
    point without a launch, with a message; the outputs stay NaN."""
    from elasticdl_b200._lib import DeepFMRows

    L = _lib()
    for G, msg in ((1, b"the xDeepFM tile tower needs at least 2 id groups"),
                   (39, b"the xDeepFM tile tower holds at most 38 id groups")):
        buf = Buffers(G, 64)  # DeepFM-sized buffers: nothing may be read or written
        buf.load(_wd_inputs(G))
        for kind in ("tile", "split", "forward"):
            before = L.b200_deepfm_xdeepfm_launch_count(), L.b200_deepfm_tile_launch_count()
            assert _call(kind, buf.args(kind != "forward")) == -1, (G, kind)
            assert L.b200_deepfm_last_error() == msg, (G, kind, L.b200_deepfm_last_error())
            assert (L.b200_deepfm_xdeepfm_launch_count(), L.b200_deepfm_tile_launch_count()) == before
        torch.cuda.synchronize()
        assert torch.isnan(buf.logits).all() and torch.isnan(buf.grads).all()
    buf = XBuffers(5, 64)
    buf.load(make_inputs(5, 64, seed=5)[0])
    a = buf.args(False)
    rows = DeepFMRows()
    a.rows = ctypes.pointer(rows)
    before = L.b200_deepfm_xdeepfm_launch_count()
    assert _call("forward", a) == -1
    assert L.b200_deepfm_last_error() == b"the forward-only xDeepFM tile tower reads pulled rows only"
    a = buf.args(True)
    a.scratch = None
    assert _call("tile", a) == -1 and L.b200_deepfm_last_error() == b"null input"
    assert L.b200_deepfm_xdeepfm_launch_count() == before
    torch.cuda.synchronize()
    assert torch.isnan(buf.logits).all()


def _wd_inputs(G):
    from tests.test_gpu_wide_deep_tower import make_inputs as wd_make_inputs

    return wd_make_inputs(G, 64, seed=G)[0]


# ---------------------------------------------------------------------------------------------------- engine level

def _ps_reference(group, eng, ids, dense, labels, mask_override=None):
    G, B, dev = eng.G, eng.B, eng.device
    inv, n_unique, uniq = X.first_occurrence_inverse(ids)
    bet_w = torch.full((G, B), NAN, device=dev)
    bet_d = torch.full((G, B, X.D), NAN, device=dev)
    for g in range(G):
        u = int(n_unique[g])
        touched = uniq[g, :u].cpu()
        bet_w[g, :u] = group.pull_rows([(eng.wide_names[g], touched)])[0].reshape(u).to(dev)
        bet_d[g, :u] = group.pull_rows([(eng.deep_names[g], touched)])[0].reshape(u, X.D).to(dev)
    d = group.pull_dense([n for n, _ in eng.params])
    params = torch.zeros(X.layout(G)["total"], dtype=torch.float32, device=dev)
    for (name, _), (off, n) in zip(eng.params, eng.flat_views):
        params[off:off + n] = torch.as_tensor(d[name]).reshape(-1).to(dev)
    inputs = (inv, n_unique, bet_w, bet_d, dense, labels, params)
    return inputs, X.xdeepfm_reference(*inputs, mask_override=mask_override, chunk=4096)


def _condition(group, eng, ids, dense, labels, seed):
    gen = torch.Generator(device=_dev()).manual_seed(seed)
    for _ in range(40):
        inputs, ref = _ps_reference(group, eng, ids, dense, labels)
        near = X.near_relu_kink(ref)
        if not bool(near.any()):
            return inputs, ref
        dense[near] = torch.randn((int(near.sum()), X.ND), generator=gen, device=_dev())
    raise AssertionError("conditioning did not converge")


def test_xdeepfm_engine_matches_references_over_adam_steps():
    """bench.py's configuration with model="xdeepfm": B = 32768, the 38 dac_ctr groups at full size, its batches
    (seeds 1234 + p), three Adam steps through the graphed lookahead feed on narrow packed ids, each step's dedup,
    loss, gradients and Adam push checked against the oracles; then predict()."""
    from bench import ADAM_ARGS
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, DeepFMPSEngine, XDeepFMTower, pack_batch, packed_views, \
        synthetic_batch
    from tests.test_gpu_engine_bench_path import BETA1, BETA2, EPS, FULL_SCAN_ROWS, LR, SAMPLE_ROWS, _check_dedup, \
        _dense, _oracle_dedup, _plan_dedup, _pre_state, _rows, _tables

    B, rows = 32768, GROUP_ROWS
    batches = [list(synthetic_batch(B, 1234 + p, _dev(), "zipf")) for p in range(4)]
    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    try:
        eng = DeepFMPSEngine(group, B, id_transport="narrow", model="xdeepfm")
        assert eng.tower_kind == "tile" and eng.row_source == "table" and isinstance(eng.tower, XDeepFMTower)
        G, D = eng.G, eng.D
        rng = np.random.RandomState(11)
        sample = [np.arange(r) if r <= FULL_SCAN_ROWS else np.sort(rng.choice(r, SAMPLE_ROWS, replace=False))
                  for r in rows]
        src = [pack_batch(*b, widths=eng.widths) for b in batches]
        for t in range(1, 4):
            ids, dense, labels = batches[t - 1]
            inputs, ref = _condition(group, eng, ids, dense, labels, seed=t)
            if t == 1:
                src[0] = pack_batch(ids, dense, labels, widths=eng.widths)
                eng.prepare_packed(src[0])
                torch.cuda.synchronize()
            else:
                packed_views(eng.s_packed[eng.cur], G, B, eng.widths)[1].copy_(dense)
            dedup = _oracle_dedup(ids)
            pre = _pre_state(group, eng, dedup, sample)
            p = eng.cur
            eng.step_ahead_graph(src[t])
            torch.cuda.synchronize()
            group.check()
            what = "xdeepfm engine step %d" % t
            _check_dedup(_plan_dedup(eng.plans[p], G, B), dedup, what + " dedup")
            ref = reference_with_kernel_masks(inputs, ref, eng.scratch, what)
            got = {"loss": eng.loss_buf, "logits": eng.logits_buf, "grads": eng.flat_grads,
                   "gsum_wide": eng.gsum_w.view(G, B), "gsum_deep": eng.gsum_d.view(G, B, D)}
            X.check({k: v for k, v in got.items() if k != "logits"}, ref, families=("loss", "grads", "gsum_wide",
                                                                                     "gsum_deep"),
                    label=what, n_sm=_n_sm())
            tabs, dense0, snap0 = pre
            gsum = {"wide": eng.gsum_w.view(G, B, 1).cpu().numpy(), "deep": eng.gsum_d.view(G, B, D).cpu().numpy()}
            for name, g, fam in _tables(eng):
                u = dedup[g][0]
                (p0, m0, v0), _ = tabs[name]
                want = [x.copy() for x in (p0, m0, v0)]
                O.np_adam(gsum[fam][g, :len(u)].copy(), *want, LR, t, BETA1, BETA2, EPS)
                for kind, a_, b_ in zip(("param", "m", "v"), _rows(group, name, u), want):
                    assert np.array_equal(a_, b_), "%s: %s %s != oracle Adam" % (what, name, kind)
            flat_g = eng.flat_grads.cpu().numpy()
            dense1 = _dense(group, eng)
            for (name, _), (off, n) in zip(eng.params, eng.flat_views):
                want = [x.copy() for x in dense0[name]]
                O.np_adam(flat_g[off:off + n].copy(), *want, LR, t, BETA1, BETA2, EPS)
                for kind, a_, b_ in zip(("param", "m", "v"), dense1[name], want):
                    assert np.array_equal(a_, b_), "%s: dense %s %s != oracle Adam" % (what, name, kind)
            assert group.snapshot() == [(t, t, True)] and eng.steps == t, what
        ids, dense, labels = batches[3]
        _, ref = _ps_reference(group, eng, ids, dense, labels)
        logits = eng.predict(ids, dense)
        torch.cuda.synchronize()
        X.check({"logits": logits}, ref, families=("logits",), label="xdeepfm predict", n_sm=_n_sm())
    finally:
        group.close()


def _trajectory(mode, tower, batches, rows, B):
    from bench import ADAM_ARGS
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, pack_batch

    group = PSGroup(1, "Adam", ADAM_ARGS, device=0)
    try:
        eng = DeepFMPSEngine(group, B, group_rows=rows, id_transport="narrow", model="xdeepfm", tower=tower)
        losses = []
        if mode == "ahead":
            eng.prepare_packed(pack_batch(*batches[0], widths=eng.widths))
            for t in range(len(batches) - 1):
                eng.step_ahead_graph(pack_batch(*batches[t + 1], widths=eng.widths))
                losses.append(float(eng.loss_buf))
        else:
            for t in range(len(batches) - 1):
                losses.append(float(eng.step(*batches[t])))
        torch.cuda.synchronize()
        group.check()
        dense = group.pull_dense([n for n, _ in eng.params])
        return losses, [dense[n].cpu() for n, _ in eng.params]
    finally:
        group.close()


def test_xdeepfm_engine_graph_equals_eager_and_torch_tower():
    """The captured lookahead graph and eager step() of the tile tower from the same seed and batches agree up to the
    order of fp32 atomic adds (losses rtol 1e-5, parameters atol 2e-4 after the Adam steps); tower="torch" follows
    the same loss trajectory within 1e-3."""
    from elasticdl_b200.workloads.deepfm import synthetic_batch

    rows, B = [5, 10, 1460, 582, 100000, 1000000], 4096
    batches = [synthetic_batch(B, 70 + p, _dev(), "zipf", group_rows=rows) for p in range(5)]
    l_e, d_e = _trajectory("eager", "tile", batches, rows, B)
    l_a, d_a = _trajectory("ahead", "tile", batches, rows, B)
    l_t, _ = _trajectory("eager", "torch", batches, rows, B)
    assert np.allclose(l_e, l_a, rtol=1e-5), (l_e, l_a)
    for a_, b_ in zip(d_e, d_a):
        assert torch.allclose(a_, b_, rtol=0, atol=2e-4), float((a_ - b_).abs().max())
    assert np.allclose(l_e, l_t, rtol=1e-3), (l_e, l_t)
