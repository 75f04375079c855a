"""The tensor-core towers keep fp32-grade products: the xDeepFM CIN (csrc/xdeepfm_cin.cu) and the mma DeepFM tower
(csrc/deepfm_tower_mma.cu) run their contractions as 3xTF32 (csrc/mma_tf32.cuh), and each contraction is checked
on its own with oracle/tf32.py's statistic

    r = ||got - ref||_2 / ||emu1x - ref||_2        over the elements the contraction feeds,

emu1x being the float64 reference with that one contraction on a single TF32 product (the same inputs, the
kernel's ReLU masks).  A 3xTF32 kernel sits at fp32 rounding noise, far under R_MAX = 1/4; a kernel on one
product sits near 1.  The per-element bound cannot tell them apart at the benchmarked 38 groups
(test_oracle_tensor_core_precision.py), so both are applied.  One limit: in the mma tower's data and weight
passes at B = 32768, a lost lo of A (dH1, a per-sample operand whose rounding averages out over the hot rows'
thousands of samples) moves r to only 0.10 - 0.15, under R_MAX; there the per-element bound catches it.

Inputs are those of the tower modules (test_gpu_xdeepfm_tower.py, test_gpu_tower_reference.py), every output
poisoned with NaN before the call.  The xDeepFM tower runs its strong_cin regime (the CIN logit dominates and the
Wide & Deep DNN is small), so that fp32 noise of the other terms does not swamp a contraction's yardstick."""
import pytest
import torch

from oracle import tf32
from oracle import tower_oracle as T
from oracle import xdeepfm_oracle as X
from tests import test_gpu_tower_reference as R
from tests import test_gpu_xdeepfm_tower as XT

pytestmark = pytest.mark.gpu
WORST = {}  # (tower, check, B) -> largest r
# The CIN weight pass's mask rows (A = the exact 0/1 mask, two products) reduce dz Z over every (sample, dim) of a
# CTA's batch slice, 8 x 32 per tile: at B = 32768 about 2000 tiles, in terms of mostly one sign where samples share
# their hot rows.  The tensor cores' fp32 accumulation (which truncates instead of rounding to nearest) then grows
# with the chain while the 1xTF32 yardstick, an operand rounding of random sign, does not: a correct kernel measured
# r = 0.33 there on an H100 (0.11 at B = 33).  Past one tile per CTA that check takes R_MAX_LONG_MASK = 1/2, which
# still lies halfway to the r of a kernel that drops the mask rows' lo product (1.04 at B = 32768 on the same
# H100); every other check, and this one on short batches, takes R_MAX = 1/4.
R_MAX_LONG_MASK = 0.5


def _record(tower, check, B, r):
    WORST[(tower, check, B)] = max(WORST.get((tower, check, B), 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nlargest ||got - ref|| / ||1xTF32 - ref|| per tower and contraction (%s, %d SMs; threshold %.2f):" % (
            torch.cuda.get_device_name(0), R._n_sm(), tf32.R_MAX))
        for (tower, check, B), r in sorted(WORST.items()):
            print("  %-8s %-12s B=%-6d %.5f" % (tower, check, B, r))


@pytest.mark.parametrize("B", ["33", "32768"])
@pytest.mark.parametrize("G", [5, 38])
def test_xdeepfm_cin_contractions_are_3xtf32(G, B):
    """The CIN's forward (logits), data pass (gsum_deep) and weight pass (the filter gradients: W_0's X_1
    channels, whose A operand dC_0 takes three products, and the mask-A rows) each within R_MAX of exact, as
    well as within the per-element bound (run_and_check)."""
    Bn = R._batch(B)
    inputs, ref, got = XT.run_and_check("tile", G, Bn, seed=G + 60, regime="strong_cin")
    km = ref["kernel_masks"]
    bad = []
    for check in X.PRECISION_CHECKS:
        fam, sel = X.precision_selection(ref, check)
        emu = X.xdeepfm_reference(*inputs, mask_override=(km[0], km[1], 1.0), magnitudes=False, chunk=4096,
                                  contraction={X.CONTRACTION_OF[check]: "1x"})
        r = tf32.ratio(got[fam], ref[fam], emu[fam], sel)
        _record("cin", check, Bn, r)
        if not r <= (R_MAX_LONG_MASK if check == "weight_mask" and Bn > 32 * R._n_sm() else tf32.R_MAX):
            bad.append((check, r))
    assert not bad, ("xdeepfm G=%d B=%d" % (G, Bn), bad)


@pytest.mark.parametrize("B", ["33", "32768"])
@pytest.mark.parametrize("G", [5, 38])
def test_mma_tower_contractions_are_3xtf32(G, B):
    """The mma tower's forward H = X W1^T (logits), data pass dX = dH1 W1 (gsum_deep) and weight pass
    dW1 = dH1^T X (dW1 and db1) each within R_MAX of exact, and every output within the per-element bound."""
    Bn = R._batch(B)
    inputs, ref = R.make_inputs(G, Bn, seed=G + 60)
    buf = R.Buffers(G, Bn)
    buf.load(inputs)  # poisons every output
    assert R._call("mma", buf.args(True)) == 0
    torch.cuda.synchronize()
    got = {"logits": buf.logits, "loss": buf.loss, "grads": buf.grads, "gsum_wide": buf.gsum_wide,
           "gsum_deep": buf.gsum_deep}
    label = "mma G=%d B=%d:" % (G, Bn)
    T.check(got, ref, label=label, n_sm=R._n_sm())
    masks = (ref["h1"] > 0, ref["h2"] > 0)  # conditioned: no unit within rounding of its kink
    bad = []
    for check in T.PRECISION_CHECKS:
        fam, sel = T.precision_selection(ref, check)
        emu = T.tower_reference(*inputs, contraction={check: "1x"}, dnn_masks=masks)
        r = tf32.ratio(got[fam], ref[fam], emu[fam], sel)
        _record("mma", check, Bn, r)
        if not r <= tf32.R_MAX:
            bad.append((check, r))
    assert not bad, (label, bad)
