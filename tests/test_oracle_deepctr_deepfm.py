"""The float64 deepctr DeepFM estimator oracle (oracle/deepctr_deepfm_oracle.py) on the CPU: against float64 torch
autograd of the same model, with samples whose every cell is empty, logits past +-90 and duplicate ids; the literal
parameter table; the oracle's ids against feature_oracle's Fingerprint64 with "" dropped; read_criteo_csv on a
hand-written file; every mutation moving an output; the TF1 Adagrad and FTRL steps against their formulas."""
import math
import os

import numpy as np
import pytest
import torch

from elasticdl_b200.workloads import deepctr_deepfm as M
from oracle import deepctr_deepfm_oracle as O
from oracle import feature_oracle as FO

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "deepctr_deepfm_rows.csv")


def _raw(B, seed, empty_fraction=0.25, distinct=2 ** 32):
    rng = np.random.RandomState(seed)
    raw = []
    for j in range(O.FIELDS):
        col = [b"%08x" % int(v) for v in rng.randint(0, distinct, B, dtype=np.int64)]
        for i in np.nonzero(rng.rand(B) < empty_fraction)[0]:
            col[i] = b""
        raw.append(col)
    return raw


def _batch(B, seed, bias=None, empty_rows=(), distinct=2 ** 32):
    g = torch.Generator().manual_seed(seed)
    raw = _raw(B, seed, distinct=distinct)
    for b in empty_rows:
        for col in raw:
            col[b] = b""
    ids = O.ids_from_raw(raw)
    dense = torch.rand((O.DENSE, B), generator=g, dtype=torch.float64) * 2
    labels = (torch.rand(B, generator=g) < 0.3).to(torch.float64)
    flat = M.initial_params(seed, "cpu").double()
    v = M.flat_views(flat)
    for n in M.LIN_NAMES + M.NUM_NAMES:  # a non-zero linear model, so that every term carries weight
        v[n].copy_(torch.randn(v[n].shape, generator=g, dtype=torch.float64) * 0.05)
    for n in M.EMB_NAMES:
        v[n].mul_(0.3)
    v[M.BIAS_NAME].fill_(0.2 if bias is None else bias)
    return raw, ids, dense, labels, flat


def _autograd(ids, dense, labels, flat):
    """The model in float64 torch autograd: returns (loss, z, flat gradient)."""
    p = {n: t.clone().requires_grad_(True) for n, t in M.flat_views(flat.clone()).items()}
    B = dense.shape[1]
    present = ids >= 0
    rows = ids.clamp(min=0)
    embs = [p[M.EMB_NAMES[j]][rows[j]] * present[j].unsqueeze(1) for j in range(O.FIELDS)]  # [B, 4] each
    e = torch.stack(embs, 1)
    x = torch.cat([e.reshape(B, -1), dense.t()], 1)
    h = x
    for k in range(3):
        h = torch.relu(h @ p["dnn/dnn/kernel%d:0" % k] + p["dnn/dnn/bias%d:0" % k])
    dnn = (h @ p["dnn/dense/kernel:0"])[:, 0]
    S = e.sum(1)
    fm = 0.5 * (S * S - (e * e).sum(1)).sum(1)
    lin = sum(p[M.LIN_NAMES[j]][rows[j], 0] * present[j] for j in range(O.FIELDS))
    lin = lin + sum(dense[i] * p[M.NUM_NAMES[i]][0, 0] for i in range(O.DENSE)) + p[M.BIAS_NAME][0]
    z = lin + fm + dnn
    ce = torch.nn.functional.binary_cross_entropy_with_logits(z, labels, reduction="sum")
    reg = sum(0.5 * (t * t).sum() for t in embs)
    reg = reg + sum(0.5 * (p[n] * p[n]).sum() for n in M.LIN_NAMES + M.NUM_NAMES)
    loss = ce + 1e-5 * reg
    loss.backward()
    return loss.detach(), z.detach(), torch.cat([p[n].grad.reshape(-1) for n in M.NAMES])


@pytest.mark.parametrize("B,bias,empty_rows,distinct", [(1, None, (), 2 ** 32), (37, None, (0, 5), 2 ** 32),
                                                        (200, None, (), 3), (64, 95.0, (1,), 2 ** 32),
                                                        (64, -95.0, (), 2 ** 32), (1, None, (0,), 2 ** 32)])
def test_oracle_matches_autograd(B, bias, empty_rows, distinct):
    """distinct=3: three strings per column, so every row the batch reads has many duplicates; bias +-95 puts every
    logit past +-90, where the loss stays finite and dz = sigmoid(z) - y."""
    _, ids, dense, labels, flat = _batch(B, B + 3, bias, empty_rows, distinct)
    for b in empty_rows:
        assert bool((ids[:, b] == -1).all())
    ref = O.reference(ids, dense, labels, flat)
    loss, z, grads = _autograd(ids, dense, labels, flat)
    assert math.isfinite(float(ref["loss"]))
    torch.testing.assert_close(ref["loss"], loss, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["logits"], z, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["grads"], grads, rtol=1e-9, atol=1e-15)
    if bias is not None:
        assert bool((ref["logits"].abs() > 90).all())
        bw = ref["grads"][O.N_PARAMS - 1]
        assert float(bw) == pytest.approx(float((torch.sigmoid(ref["logits"]) - labels).sum()), rel=1e-12)
    if distinct == 3:
        assert int(ids[0].unique().numel()) <= 4


def test_untouched_rows_get_exact_zero_and_lambda_w():
    _, ids, dense, labels, flat = _batch(50, 7)
    ref = O.reference(ids, dense, labels, flat)
    g = M.flat_views(ref["grads"])
    v = M.flat_views(flat)
    for j in (0, 25):
        touched = torch.zeros(O.ROWS, dtype=torch.bool)
        touched[ids[j][ids[j] >= 0]] = True
        assert bool((g[M.EMB_NAMES[j]][~touched] == 0).all())
        torch.testing.assert_close(g[M.LIN_NAMES[j]][~touched], 1e-5 * v[M.LIN_NAMES[j]][~touched], rtol=0, atol=0)


def test_parameter_table():
    assert len(M.PARAMS) == 73 and M.N_PARAMS == 201438
    assert sum(int(np.prod(s)) for _, s in M.PARAMS) == 201438
    assert len(M.DNN_GROUP) == 33 and len(M.LINEAR_GROUP) == 40
    assert sum(int(np.prod(s)) for _, s in M.DNN_GROUP) == 175424
    # the offsets include/b200_deepctr_deepfm.h states
    assert [M.OFFSETS[n] for n, _ in M.DNN_PARAMS] == [104000, 133952, 134208, 166976, 167104, 175296, 175360]
    assert M.OFFSETS[M.EMB_NAMES[1]] == 4000 and M.OFFSETS[M.LIN_NAMES[1]] == 176424
    assert M.OFFSETS[M.NUM_NAMES[0]] == 201424 and M.OFFSETS[M.BIAS_NAME] == 201437
    assert dict(M.PARAMS)[M.NUM_NAMES[0]] == (1, 1) and dict(M.PARAMS)[M.BIAS_NAME] == (1,)
    flat = M.initial_params(0, "cpu")
    v = M.flat_views(flat)
    assert all(float(v[n].abs().max()) == 0 for n in M.LINEAR_NAMES)
    assert all(float(v[n].abs().max()) == 0 for n in ("dnn/dnn/bias0:0", "dnn/dnn/bias2:0"))
    e = torch.cat([v[n].reshape(-1) for n in M.EMB_NAMES])
    assert float(e.abs().max()) <= 1.0  # truncated at two stddevs of 0.5
    assert abs(float(e.std()) - 0.5 * 0.8796) < 0.01  # the std of a normal truncated at 2 sigma
    k = v["dnn/dnn/kernel0:0"]
    assert abs(float(k.std()) - np.sqrt(2.0 / (117 + 256))) < 0.05 * np.sqrt(2.0 / (117 + 256))
    (lt, la), (dt, da) = M.optimizers()
    assert lt == "Ftrl" and "initial_accumulator_value=0.1;" in la and "learning_rate=0.005;" in la
    assert dt == "Adagrad" and da == "learning_rate=0.01;epsilon=0.0;"


def test_ids_are_fingerprint64_with_empty_dropped():
    raw = _raw(300, 5)
    ids = O.ids_from_raw(raw)
    for j in (0, 7, 25):
        want = [FO.fingerprint64(s) % 1000 if s else -1 for s in raw[j]]
        assert ids[j].tolist() == want
    assert int((ids == -1).sum()) > 0
    assert bool((ids >= -1).all() and (ids < 1000).all())
    assert O.ids_from_raw([[b""]] * 26, drop_empty=False)[0, 0] == FO.fingerprint64(b"") % 1000


def test_read_criteo_csv():
    dense, strings, labels = M.read_criteo_csv(GOLDEN)
    assert labels.tolist() == [1.0, 0.0, 0.0]
    assert dense.shape == (13, 3) and strings.shape == (26, 3, 8) and strings.dtype == torch.uint8
    assert dense[:, 0].tolist() == [3, 0, 7, 0, 1.5, 0, 2, 0, 0, 4, 0, 12, -1]
    assert dense[:, 1].tolist() == [0, 1] + [0] * 11
    assert dense[:, 2].tolist() == [0, 2.25, 0, 5, 0, 1000] + [0] * 6 + [8]
    assert bytes(strings[0, 0].numpy()) == b"68fd1e64" and bytes(strings[25, 2].numpy()) == b"ffffffff"
    assert bytes(strings[21, 0].numpy()) == b"\0" * 8  # C22 empty
    assert int(strings[:, 1].sum()) == 0  # every string of row 2 empty
    raw = [[bytes(strings[j, b].numpy()).rstrip(b"\0") for b in range(3)] for j in range(26)]
    ids = O.ids_from_raw(raw)
    assert int(ids[0, 0]) == FO.fingerprint64(b"68fd1e64") % 1000 and bool((ids[:, 1] == -1).all())
    assert int((ids[:, 2] >= 0).sum()) == 2


def test_every_mutation_moves_an_output():
    B = 256
    raw, ids, dense, labels, flat = _batch(B, 11)
    ref = O.reference(ids, dense, labels, flat)
    got = {k: ref[k].to(torch.float32) for k in ("logits", "loss", "grads")}
    assert not O.caught_by(got, ref)
    muts = O.mutations(ids, dense, labels, flat, raw)
    assert set(muts) == set(O.MUTATIONS)
    for name, mut in muts.items():
        if name not in O.SATURATED_MUTATIONS:
            assert O.caught_by(mut, ref), name
    _, ids, dense, labels, flat = _batch(B, 12, bias=100.0)
    labels = torch.ones_like(labels)
    ref = O.reference(ids, dense, labels, flat)
    assert not O.caught_by({k: ref[k].to(torch.float32) for k in ("logits", "loss", "grads")}, ref)
    for name, mut in O.mutations(ids, dense, labels, flat, names=O.SATURATED_MUTATIONS).items():
        assert O.caught_by(mut, ref), name


def test_adagrad_step_is_tf1s():
    g = torch.tensor([0.0, 0.3, -2.0, 1e-3], dtype=torch.float64)
    p = torch.tensor([0.5, -0.25, 1.0, 0.0], dtype=torch.float64)
    acc = O.adagrad_init(p)
    assert acc.tolist() == [0.1] * 4
    p1, a1 = O.adagrad_step(p, acc, g)
    for i in range(4):
        a = 0.1 + g[i].item() ** 2
        assert a1[i].item() == pytest.approx(a, rel=1e-15)
        assert p1[i].item() == pytest.approx(p[i].item() - 0.01 * g[i].item() / math.sqrt(a), rel=1e-15, abs=1e-300)
    assert p1[0] == p[0] and a1[0] == acc[0]  # a zero gradient leaves the row and its accumulator as they were
    eps, _ = O.adagrad_step(p, acc, g, mutate=("adagrad_epsilon",))
    assert not torch.equal(eps, p1)
    zero, _ = O.adagrad_step(p[1:], O.adagrad_init(p[1:], ("adagrad_zero_accumulator",)), g[1:])
    assert not torch.allclose(zero, p1[1:])


def test_ftrl_step_is_tf1s():
    g = torch.tensor([0.0, 0.3, -2.0, 1e-5], dtype=torch.float64)
    p = torch.tensor([0.0, -0.25, 1.0, 0.02], dtype=torch.float64)
    acc, lin = O.ftrl_init(p)
    p1, a1, l1 = O.ftrl_step(p, acc, lin, g)
    for i in range(4):
        a = 0.1 + g[i].item() ** 2
        li = g[i].item() - (math.sqrt(a) - math.sqrt(0.1)) / 0.005 * p[i].item()
        want = -li / (math.sqrt(a) / 0.005) if li != 0 else 0.0
        assert a1[i].item() == pytest.approx(a, rel=1e-15)
        assert l1[i].item() == pytest.approx(li, rel=1e-12, abs=1e-300)
        assert p1[i].item() == pytest.approx(want, rel=1e-12, abs=1e-300)
    assert p1[0] == 0 and a1[0] == acc[0] and l1[0] == 0  # an untouched zero row stays exactly zero
    # a row touched once and then fed only g = lambda w keeps moving
    w, a, li = p1[1:2], a1[1:2], l1[1:2]
    w2, _, _ = O.ftrl_step(w, a, li, 1e-5 * w)
    assert float(w2) != float(w)
