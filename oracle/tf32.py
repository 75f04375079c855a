"""TF32 tensor-core contractions emulated in float64 -- TEST INFRASTRUCTURE.

csrc/mma_tf32.cuh runs an fp32 contraction on tensor cores as 3xTF32: each fp32 operand x is split into
hi = tf32(x) and lo = tf32(x - hi) (cvt.rna: round to nearest, ties away from zero, 10 explicit mantissa bits) and
a product is lo*hi + hi*lo + hi*hi, which leaves out only lo*lo (about 2^-22 of the product).  One product, hi*hi,
is a 1xTF32 kernel: every operand carries a relative error up to 2^-11.

`contract` evaluates a contraction the way a kernel with a given set of products would, in float64 (so that the
only error is the one the products leave), and `ratio` turns a kernel's output into the statistic

    r = ||got - ref||_2 / ||emu1x - ref||_2

over the elements one contraction feeds, where emu1x is the float64 reference with that contraction in "1x".  The
yardstick is the error a 1xTF32 kernel makes on the same inputs, so r needs no magnitude model: 3xTF32 sits at
fp32 accumulation noise (a few 2^-12 or less), one product gives about 1 and a dropped lo term about 0.5-0.7.
Device agnostic: every function takes and returns torch tensors on any device.
"""
import torch

MODES = ("fp32", "3x", "1x", "2x_no_a_lo", "2x_no_b_lo")
CONTRACTIONS = ("forward", "data", "weight")
R_MAX = 0.25  # a kernel's r above this lost a product


def round_tf32(x):
    """x rounded to fp32, then to TF32 as cvt.rna.tf32.f32 does (nearest, ties away from zero; the low 13 mantissa
    bits 0).  Returns float64.  Non-finite values pass through."""
    f = x.to(torch.float32).contiguous()
    b = f.view(torch.int32)
    r = ((b + 0x1000) & ~0x1FFF).view(torch.float32)
    return torch.where(torch.isfinite(f), r, f).to(torch.float64)


def split(x):
    """(hi, lo) float64 as mma_tf32.cuh's split: hi = tf32(x), lo = tf32(x - hi), x rounded to fp32 first (the
    difference x - hi is exact in fp32)."""
    f = x.to(torch.float32)
    hi = round_tf32(f)
    lo = round_tf32(f.to(torch.float64) - hi)
    return hi, lo


def contract(a, b, mode="fp32", eq=None):
    """a @ b (or torch.einsum(eq, a, b)) with the products of `mode`:
      "fp32"        exact in float64, the operands as given
      "3x"          al bh + ah bl + ah bh (mma3)
      "1x"          ah bh
      "2x_no_a_lo"  ah bl + ah bh
      "2x_no_b_lo"  al bh + ah bh
    where (ah, al) = split(a), (bh, bl) = split(b): the operands are rounded to fp32 first, as a kernel holds them."""
    def mm(x, y):
        return x @ y if eq is None else torch.einsum(eq, x, y)

    if mode == "fp32":
        return mm(a, b)
    if mode not in MODES:
        raise ValueError("unknown contraction mode %r" % (mode,))
    ah, al = split(a)
    bh, bl = split(b)
    out = mm(ah, bh)
    if mode in ("3x", "2x_no_a_lo"):
        out = out + mm(ah, bl)
    if mode in ("3x", "2x_no_b_lo"):
        out = out + mm(al, bh)
    return out


def fp32(x):
    """x rounded to fp32, kept in float64: an operand a kernel forms as an fp32 product before it splits it."""
    return x.to(torch.float32).to(torch.float64)


def modes(contraction):
    """{forward, data, weight} -> mode from None (all "fp32"), one mode for all, or a dict (missing ones "fp32")."""
    if contraction is None:
        contraction = {}
    if isinstance(contraction, str):
        contraction = dict.fromkeys(CONTRACTIONS, contraction)
    bad = set(contraction) - set(CONTRACTIONS)
    if bad:
        raise ValueError("unknown contraction %s" % sorted(bad))
    out = {k: contraction.get(k, "fp32") for k in CONTRACTIONS}
    for m in out.values():
        if m not in MODES:
            raise ValueError("unknown contraction mode %r" % (m,))
    return out


def ratio(got, ref, emu1x, select=None):
    """||got - ref||_2 / ||emu1x - ref||_2 over the elements `select` picks (a bool mask, an index or a slice of the
    flattened tensors; all of them by default).  A NaN or inf in got gives inf; an emulation that does not move
    the selected elements at all is an error (the contraction does not feed them)."""
    ref = ref.to(torch.float64)
    g = torch.as_tensor(got).to(device=ref.device, dtype=torch.float64).reshape(ref.shape)
    e = emu1x.to(device=ref.device, dtype=torch.float64).reshape(ref.shape)
    if select is not None:
        if isinstance(select, torch.Tensor) and select.dtype == torch.bool:
            sel = select.to(ref.device).expand(ref.shape)
            g, e, ref = g[sel], e[sel], ref[sel]
        else:
            g, e, ref = g.reshape(-1)[select], e.reshape(-1)[select], ref.reshape(-1)[select]
    if not bool(torch.isfinite(g).all()):
        return float("inf")
    den = float(torch.linalg.vector_norm(e - ref))
    if not den > 0:
        raise AssertionError("the 1xTF32 emulation leaves these elements unchanged")
    return float(torch.linalg.vector_norm(g - ref)) / den


def live_rows(ref, fam):
    """bool mask of the rows of gsum_wide [G, R] / gsum_deep [G, R, 8] below n_unique (the rows a tower writes)."""
    n = ref[fam].shape[1]
    live = torch.arange(n, device=ref[fam].device).unsqueeze(0) < ref["n_unique"].to(ref[fam].device).unsqueeze(1)
    return live.unsqueeze(2) if fam == "gsum_deep" else live
