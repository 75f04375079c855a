"""Kernel-level tests of the three DeepFM towers (csrc/deepfm_tower2.cu "tile", csrc/deepfm_tower.cu "fused",
csrc/deepfm_tower_mma.cu "mma") against the float64 reference of oracle/tower_oracle.py, through the C ABI
of include/b200_deepfm.h (no PS): at the wave edges of the device (a CTA that runs a second tile / chunk),
at id patterns that stress the warp-level id dedup, in value regimes where each term of the model matters,
with every output buffer poisoned with NaN before each call.

Conditioning: a ReLU whose float64 pre-activation lies within rounding of 0 may switch the other way in
fp32, and then the backward differs by far more than rounding.  Every batch is therefore redrawn until no
sample has a layer-1 or layer-2 pre-activation within tau * M of 0 (tau = 1e-4, M from the magnitude pass):
the offending samples get a new dense row.  Without this the tests would fail at random.

Tolerance: |got - ref| <= 8 * sqrt(n) * 2^-24 * M elementwise, for every tower (tower_oracle.chain_lengths)."""
import ctypes

import pytest
import torch

from oracle import tower_oracle as T

pytestmark = pytest.mark.gpu
NAN = float("nan")
TAU = 1e-4
WORST = {}  # (tower, family) -> largest err / bound seen in this module


def _dev():
    return torch.device("cuda", 0)


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


# batch sizes by name: the wave edges are derived from the SM count of the device
def _batch(name):
    n = _n_sm()
    return {"1": 1, "31": 31, "32": 32, "33": 33, "1000": 1000,
            "tile_wave2": 2 * n * 32 + 1,      # tile tower: one CTA's second tile holds one live sample
            "32768": 32768,
            "fused_b_wave2": 4 * n * 32 + 5,   # fused k_tower_b: second grid-stride iteration
            "fused_a_wave2": 8 * n * 128 + 1,  # fused k_tower_a: second grid-stride iteration
            "262144": 262144}[name]


SHAPES_B = ["1", "31", "32", "33", "1000", "tile_wave2", "32768", "fused_b_wave2", "fused_a_wave2"]


def _group_rows(G):
    """Row counts of G groups: the dac_ctr tables, categorical ones first (so that G = 1 is a Zipf table)."""
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS

    return [GROUP_ROWS[(12 + g) % len(GROUP_ROWS)] for g in range(G)]


def _ids(pattern, G, B, seed, gen):
    dev = _dev()
    b = torch.arange(B, device=dev)
    if pattern == "zipf":
        from elasticdl_b200.workloads.deepfm import synthetic_batch

        return synthetic_batch(B, seed, dev, "zipf", group_rows=_group_rows(G))[0]
    if pattern == "equal":  # n_unique = 1: every CTA adds into one row, the dedup tree runs all 5 rounds
        return torch.zeros((G, B), dtype=torch.int64, device=dev)
    if pattern == "distinct":
        return torch.stack([torch.randperm(B, generator=gen, device=dev) for _ in range(G)])
    if pattern == "lanes":  # inside each warp of 32 samples, k distinct ids interleaved: multiplicity ~32 / k
        out = []
        for g in range(G):
            mult = torch.tensor([2, 3, 5, 7, 32], device=dev)[(b // 32 + g) % 5]
            k = (32 + mult - 1) // mult
            out.append((b // 32) * 32 + (b % 32) % k)
        return torch.stack(out)
    if pattern == "straddle":  # runs of 48 across tile (and CTA) boundaries / one id in every tile
        return torch.stack([(b + 16 + 5 * g) // 48 if g % 2 == 0 else b % 61 for g in range(G)])
    raise ValueError(pattern)


def make_inputs(G, B, pattern="zipf", regime="base", seed=0):
    """Device inputs of one batch in the kernel's layout, conditioned (module docstring).  Rows at or past
    n_unique[g] and the padding floats of the parameters are NaN: the towers must never read them."""
    dev = _dev()
    gen = torch.Generator(device=dev).manual_seed(1000 + seed)
    ids = _ids(pattern, G, B, seed, gen)
    inv, n_unique, _ = T.first_occurrence_inverse(ids)
    scale = (5.0 / max(G, 5)) ** 0.5  # FM, wide and linear terms all O(1) at any G
    sw = sd = 0.5 * scale
    live = torch.arange(B, device=dev).unsqueeze(0) < n_unique.unsqueeze(1).long()
    bet_wide = torch.where(live, torch.randn((G, B), generator=gen, device=dev) * sw, NAN).contiguous()
    bet_deep = torch.where(live.unsqueeze(2), torch.randn((G, B, T.D), generator=gen, device=dev) * sd, NAN).contiguous()
    dense = torch.randn((B, T.ND), generator=gen, device=dev)
    if regime == "soft":
        labels = torch.rand(B, generator=gen, device=dev)
    else:
        labels = (torch.rand(B, generator=gen, device=dev) < 0.25).float()
    kw = {}
    if regime == "large_logit":
        kw["wd_std"] = 6.0  # |z| up to ~80: expf(-|z|) underflows
    if regime == "dead_l1":
        kw.update(b1=-100.0, b2=[0.5, -0.5, 0.7, 0.3])
    params = T.random_params(G, gen, dev, pad=NAN, **kw)
    for _ in range(40):
        ref = T.tower_reference(inv, n_unique, bet_wide, bet_deep, dense, labels, params)
        near = T.near_relu_kink(ref, TAU)
        if not bool(near.any()):
            break
        dense[near] = torch.randn((int(near.sum()), T.ND), generator=gen, device=dev)
    else:
        raise AssertionError("conditioning did not converge")
    if regime == "large_logit" and B >= 1000:
        assert float(ref["logits"].abs().max()) > 50
    return (inv, n_unique, bet_wide, bet_deep, dense, labels, params), ref


class Buffers:
    """The output and scratch buffers of one shape, reused by every call (re-armed tile counter, re-zeroing)."""

    def __init__(self, G, B):
        dev, f32 = _dev(), torch.float32
        self.G, self.B = G, B
        self.inv = torch.empty((G, B), dtype=torch.int32, device=dev)
        self.n_unique = torch.empty(G, dtype=torch.int32, device=dev)
        self.bet_wide = torch.empty((G, B), dtype=f32, device=dev)
        self.bet_deep = torch.empty((G, B, T.D), dtype=f32, device=dev)
        self.dense = torch.empty((B, T.ND), dtype=f32, device=dev)
        self.labels = torch.empty(B, dtype=f32, device=dev)
        self.params = torch.empty(T.layout(G)["total"], dtype=f32, device=dev)
        self.grads = torch.empty_like(self.params)
        self.gsum_wide = torch.empty((G, B), dtype=f32, device=dev)
        self.gsum_deep = torch.empty((G, B, T.D), dtype=f32, device=dev)
        self.loss = torch.empty(1, dtype=f32, device=dev)
        self.logits = torch.empty(B, dtype=f32, device=dev)
        self.scratch = torch.empty(max(B * 44 + 16 * (T.ND + T.D * G), 320 * 16 + 16), dtype=f32, device=dev)

    def load(self, inputs):
        for dst, src in zip((self.inv, self.n_unique, self.bet_wide, self.bet_deep, self.dense, self.labels,
                             self.params), inputs):
            dst.copy_(src)
        for t in (self.grads, self.gsum_wide, self.gsum_deep, self.loss, self.logits, self.scratch):
            t.fill_(NAN)

    def args(self, backward=True):
        from elasticdl_b200._lib import DeepFMArgs

        a = DeepFMArgs()
        a.G, a.B = self.G, self.B
        a.inv, a.n_unique = self.inv.data_ptr(), self.n_unique.data_ptr()
        a.bet_wide, a.bet_deep = self.bet_wide.data_ptr(), self.bet_deep.data_ptr()
        a.dense, a.labels, a.params = self.dense.data_ptr(), self.labels.data_ptr(), self.params.data_ptr()
        a.logits, a.scratch = self.logits.data_ptr(), self.scratch.data_ptr()
        if backward:
            a.grads, a.gsum_wide, a.gsum_deep = self.grads.data_ptr(), self.gsum_wide.data_ptr(), self.gsum_deep.data_ptr()
            a.loss = self.loss.data_ptr()
        return a


def _call(tower, a):
    from elasticdl_b200 import _lib

    L = _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    p = ctypes.byref(a)
    if tower == "split":  # the engine's branched step: prologue, then the main kernel
        rc = L.b200_deepfm_tile_prologue(p, st)
        return rc or L.b200_deepfm_tile_main(p, st)
    fn = {"tile": L.b200_deepfm_fwd_bwd_tile, "fused": L.b200_deepfm_fwd_bwd, "mma": L.b200_deepfm_fwd_bwd_mma,
          "forward_tile": L.b200_deepfm_forward_tile, "forward": L.b200_deepfm_forward}[tower]
    return fn(p, st)


def _record(tower, rs):
    for fam, r in rs.items():
        WORST[(tower, fam)] = max(WORST.get((tower, fam), 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nlargest err / bound per tower and output family (%s, %d SMs):" % (
            torch.cuda.get_device_name(0), _n_sm()))
        for (tower, fam), r in sorted(WORST.items()):
            print("  %-13s %-10s %.4f" % (tower, fam, r))


def run_and_check(tower, G, B, pattern="zipf", regime="base", seed=0, calls=2):
    """`calls` calls of one tower on the same buffers, each with a new batch, every output poisoned before."""
    buf = Buffers(G, B)
    backward = not tower.startswith("forward")
    for k in range(calls):
        inputs, ref = make_inputs(G, B, pattern, regime, seed=seed * 7 + k)
        buf.load(inputs)
        rc = _call(tower, buf.args(backward))
        assert rc == 0, (tower, rc)
        torch.cuda.synchronize()
        label = "%s G=%d B=%d %s/%s call %d:" % (tower, G, B, pattern, regime, k)
        if not backward:
            rs = T.check({"logits": buf.logits}, ref, families=("logits",), label=label, n_sm=_n_sm())
            _record(tower, rs)
            continue
        got = {"logits": buf.logits, "loss": buf.loss, "grads": buf.grads, "gsum_wide": buf.gsum_wide,
               "gsum_deep": buf.gsum_deep}
        rs = T.check(got, ref, label=label, n_sm=_n_sm())  # also fails on a NaN left in any overwritten output
        _record(tower, rs)
        # rows at or past n_unique[g] belong to nobody: the tower must not write them
        dead = torch.arange(B, device=_dev()).unsqueeze(0) >= inputs[1].unsqueeze(1).long()
        assert torch.isnan(buf.gsum_wide[dead]).all(), label
        assert torch.isnan(buf.gsum_deep[dead]).all(), label
        if regime == "dead_l1":  # no live hidden unit: dW1, db1 and dW2 (= dh2 a1, a1 = 0) are exactly 0
            o = T.layout(G)
            assert (buf.grads[o["w1"]:o["w2"] + T.H2 * T.H1] == 0).all(), label
    return buf


@pytest.mark.parametrize("B", SHAPES_B)
@pytest.mark.parametrize("G", [1, 5, 33, 38, 39, 46])
@pytest.mark.parametrize("tower", ["tile", "fused", "mma"])
def test_tower_shapes(tower, G, B):
    if tower == "tile" and G > 38:
        pytest.skip("the tile tower holds at most 38 id groups (see test_group_limits_and_their_messages)")
    run_and_check(tower, G, _batch(B), seed=G)


@pytest.mark.parametrize("B", SHAPES_B + ["262144"])
def test_tile_split_prologue_main(B):
    run_and_check("split", 38, _batch(B), seed=3)


def test_tile_tower_largest_batch():
    run_and_check("tile", 38, _batch("262144"), seed=4)


@pytest.mark.parametrize("B", ["33", "tile_wave2", "32768"])
@pytest.mark.parametrize("pattern", ["equal", "distinct", "zipf", "lanes", "straddle"])
@pytest.mark.parametrize("tower", ["tile", "fused", "mma"])
def test_tower_id_patterns(tower, pattern, B):
    G = 38 if tower == "tile" else 46
    run_and_check(tower, G, _batch(B), pattern=pattern, seed=11)


@pytest.mark.parametrize("B", ["1000", "32768"])
@pytest.mark.parametrize("regime", ["base", "large_logit", "dead_l1", "soft"])
@pytest.mark.parametrize("tower", ["tile", "fused", "mma"])
def test_tower_value_regimes(tower, regime, B):
    run_and_check(tower, 38, _batch(B), regime=regime, seed=21)


@pytest.mark.parametrize("B", SHAPES_B)
@pytest.mark.parametrize("G", [5, 38])
@pytest.mark.parametrize("tower", ["forward_tile", "forward"])
def test_forward_only(tower, G, B):
    run_and_check(tower, G, _batch(B), seed=31)


def test_group_limits_and_their_messages():
    """G = 39 on the tile tower and G = 47 on the fused / mma towers are refused (-1) without a launch, and
    b200_deepfm_last_error names the limit of the tower that refused."""
    from elasticdl_b200 import _lib

    L = _lib.lib()
    for tower, G, count, limit in (("tile", 39, L.b200_deepfm_tile_launch_count, b"38"),
                                   ("split", 39, L.b200_deepfm_tile_launch_count, b"38"),
                                   ("forward_tile", 39, L.b200_deepfm_tile_launch_count, b"38"),
                                   ("fused", 47, L.b200_deepfm_launch_count, b"46"),
                                   ("forward", 47, L.b200_deepfm_launch_count, b"46"),
                                   ("mma", 47, L.b200_deepfm_mma_launch_count, b"46")):
        buf = Buffers(G, 64)
        buf.load(make_inputs(G, 64, seed=G)[0])
        before = count()
        assert _call(tower, buf.args(not tower.startswith("forward"))) == -1, tower
        assert limit in L.b200_deepfm_last_error(), (tower, L.b200_deepfm_last_error())
        assert count() == before, tower
        torch.cuda.synchronize()
        assert torch.isnan(buf.logits).all() and torch.isnan(buf.grads).all(), tower


@pytest.mark.parametrize("B", SHAPES_B + ["262144"])
@pytest.mark.parametrize("G", [1, 5, 33, 38, 39, 46])
def test_mutations_are_caught(G, B):
    """The comparator rejects each classic tiled-reduction fault (tower_oracle.mutations) at every shape the
    towers are tested at -- with one exception.  A single 32-sample tile missing from the parameter gradients
    (and from nothing else) is a 32 / B share of each sum; past about 40 000 samples that share is smaller
    than fp32 rounding of the batch sum allows the bound to be, so it is only required up to B = 32768.  The
    towers' real per-CTA fault -- every later tile of a CTA dropped -- removes far more."""
    Bn = _batch(B)
    if B == "262144" and G != 38:
        pytest.skip("B = 262144 is run on the tile tower at G = 38 only")
    inputs, ref = make_inputs(G, Bn, "zipf", seed=G + 100)
    for name, got in T.mutations(ref, inputs).items():
        if name == "loss_not_divided_by_B" and Bn == 1:
            continue  # the same number
        if name == "tile_missing_from_grads" and Bn > 32768:
            continue
        caught = T.caught_by(got, ref, n_sm=_n_sm())
        assert caught, (name, G, Bn, {f: v[0] for f, v in T.ratios(got, ref, n_sm=_n_sm()).items()})
