"""census_model_sqlflow's DNNClassifier (workloads/fc_dnn.py CENSUS_SQLFLOW_DNN) on FeatureColumnDNNEngine, with its
eight 64 x 16 tables kept as dense PS parameters (DESIGN.md section 4, Q36), against the float64 oracles of
oracle/fc_dnn_oracle.py (the tower) and oracle/census_sqlflow_dnn_oracle.py (the ids and the Indexed Adam).

One eager step at B = 1, 63, 64, 65 and 4096 with a share of empty strings: the ids from the raw strings, the
pulled rows against the dense parameters, the loss, logits, MLP gradients and every table's row sums against the
oracle on the pulled state, then the PS after the push (the touched rows and their m / v against the Indexed Adam,
every other row and its slots bit-identical).  Row 0 pushed with a zero gradient by empty strings alone.  Eager
steps against the same steps replayed from the CUDA graph, bit for bit.  evaluate() against numpy's accuracy.  The
drop-in trainer over the torch twin: the same PS names and kinds, the same values within float32 tolerance."""
import types

import numpy as np
import pytest
import torch

from elasticdl_b200.common.evaluation_utils import EvaluationMetrics
from elasticdl_b200.common.model_handler import ParameterServerModelHandler
from elasticdl_b200.layers.dense_table import DenseTableEmbedding
from elasticdl_b200.preprocessing.layers import encode_strings
from elasticdl_b200.ps import PSGroup
from elasticdl_b200.workloads import fc_dnn as M
from oracle import census_sqlflow_dnn_oracle as CO
from oracle import fc_dnn_oracle as FD
from oracle import feature_oracle as FO

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
L = M.CENSUS_SQLFLOW_DNN
OPT_TYPE, OPT_ARGS, LR = L.optimizer


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _batches(B, n, seed, empty_fraction=0.2):
    """Raw Adult-shaped rows, the numeric columns scaled down (as tests/test_gpu_fc_dnn.py does: raw capital
    gains saturate the sigmoid at the clip edge, Q19), a share of every string column empty."""
    out = []
    for s in range(n):
        numeric, strings = M.synthetic_census_batch(B, seed + s, DEV, empty_fraction=empty_fraction)
        labels = (torch.rand(B, generator=torch.Generator(device=DEV).manual_seed(seed + s), device=DEV)
                  < 0.25).float()
        out.append((numeric / 1e4, strings, labels))
    return out


def _make(B, n_shards=2, seed=3):
    group = PSGroup(n_shards, OPT_TYPE, OPT_ARGS, device=0)
    return group, M.FeatureColumnDNNEngine(group, L, B, LR, seed=seed)


def _ps_state(group):
    """{name: (p, m, v)} of every dense parameter, the tables and the MLP."""
    return {n: tuple(group.slot_dense(n, s).clone() for s in range(3)) for n in L.table_names + M.MLP_NAMES}


def _raw(strings):
    host = strings.cpu().numpy()
    return [[bytes(host[c, b]).rstrip(b"\0") for b in range(host.shape[1])] for c in range(host.shape[0])]


def _uniq(eng, k):
    return eng.uniq[k * eng.B:k * eng.B + int(eng.n_unique[k])]


def _check_pushed_tables(eng, before, after, step, label):
    """Each table's touched rows and slots against the Indexed Adam of the row sums the tower pushed; every other
    row and its slots bit-identical."""
    for k, n in enumerate(L.table_names):
        ids = _uniq(eng, k)
        g = eng.tower.table_view(eng.tower.gsum, k)[:ids.numel()]
        want = CO.indexed_adam(*before[n], ids, g, LR, step)
        others = torch.ones(64, dtype=torch.bool, device=DEV)
        others[ids] = False
        for s, (b, a, w) in enumerate(zip(before[n], after[n], want)):
            assert torch.equal(a[others], b[others]), (label, n, s)
            tol = [dict(rtol=1e-6, atol=1e-7), dict(rtol=1e-5, atol=1e-9), dict(rtol=1e-5, atol=1e-12)][s]
            torch.testing.assert_close(a[ids].double(), w[ids], **tol, msg=lambda m: "%s %s slot %d: %s"
                                       % (label, n, s, m))


@pytest.mark.parametrize("B", [1, 63, 64, 65, 4096])
def test_step_matches_oracle(B):
    group, eng = _make(B)
    numeric, strings, labels = _batches(B, 1, 100 + B)[0]
    before = _ps_state(group)
    loss = eng.step(numeric, strings, labels)
    torch.cuda.synchronize()
    eng.check()
    raw = _raw(strings)
    nu = eng.n_unique.tolist()
    empty = torch.stack([strings[L.string_keys.index(k), :, 0] == 0 for k, _, _ in L.tables])
    for k, (key, _, _) in enumerate(L.tables):
        want = CO.ids_from_strings(raw[L.string_keys.index(key)], 64)
        np.testing.assert_array_equal(eng.ids[k].cpu().numpy(), want, err_msg=key)
        ids = _uniq(eng, k)
        assert sorted(ids.tolist()) == sorted(set(want.tolist()))
        if bool(empty[k].any()):
            assert 0 in ids.tolist()  # the fill id of the empty strings is pushed (Q36)
        # pull_rows read the dense parameter's rows
        assert torch.equal(eng.tower.table_view(eng.rows, k)[:nu[k]], before[L.table_names[k]][0][ids])
    assert torch.equal(eng.flat, torch.cat([before[n][0].reshape(-1) for n in M.MLP_NAMES]))
    rows = [eng.tower.table_view(eng.rows, k)[:n] for k, n in enumerate(nu)]
    ref = FD.fc_dnn_reference(L.spec(), numeric, eng.ids, empty, eng.inv, nu, rows, labels, eng.flat)
    out = eng.tower.outputs(nu)
    FD.check({"logits": out["logits"], "loss": out["loss"], "grads": out["grads"], "gsum": out["gsum"]}, ref,
             n_sm=_n_sm(), label="B=%d" % B)
    assert abs(float(loss) - float(ref["loss"])) <= 1e-5 * float(ref["M"]["loss"])
    after = _ps_state(group)
    _check_pushed_tables(eng, before, after, 1, "B=%d" % B)
    # the MLP: Adam on every element (an Indexed update of all rows of the flat view)
    off = 0
    for n in M.MLP_NAMES:
        p, m, v = (t.reshape(-1, 1) for t in before[n])
        k = p.shape[0]
        want = CO.indexed_adam(p, m, v, torch.arange(k, device=DEV), eng.tower.grads[off:off + k], LR, 1)
        off += k
        torch.testing.assert_close(after[n][0].reshape(-1, 1).double(), want[0], rtol=1e-6, atol=1e-7)
    assert [v for v, _, _ in group.snapshot()] == [1, 1]


def _string_hashing_to(bucket, count, exclude=False):
    """`count` distinct strings whose Fingerprint64 % 64 is `bucket` (exclude=False) or is not (exclude=True)."""
    out, i = [], 0
    while len(out) < count:
        s = "s%d" % i
        if (int(FO.hashing([s], 64)[0]) == bucket) != exclude:
            out.append(s)
        i += 1
    return out


def test_row_zero_moves_on_the_zero_gradient_of_empty_strings():
    """Q36: step 1 reads row 0 through real strings (nonzero m); step 2 has empty strings and no string of bucket
    0, so row 0 is pushed with an exactly zero gradient, and the Indexed Adam still moves it."""
    B = 128
    group, eng = _make(B, n_shards=1)
    zero = _string_hashing_to(0, 4)
    other = _string_hashing_to(0, 16, exclude=True)
    col1 = [zero[i % 4] if i % 2 else other[i % 16] for i in range(B)]
    col2 = ["" if i % 3 == 0 else other[i % 16] for i in range(B)]
    g = torch.Generator(device=DEV).manual_seed(1)
    labels = (torch.rand(B, generator=g, device=DEV) < 0.5).float()
    numeric = torch.rand((4, B), generator=g, device=DEV)
    for step, col in enumerate((col1, col2), start=1):
        strings = encode_strings([col] * 8, M.STRING_WIDTH, device=DEV).contiguous()
        before = _ps_state(group)
        eng.step(numeric, strings, labels)
        torch.cuda.synchronize()
        eng.check()
        _check_pushed_tables(eng, before, _ps_state(group), step, "step %d" % step)
        for k, n in enumerate(L.table_names):
            ids = _uniq(eng, k).tolist()
            assert 0 in ids
            g0 = eng.tower.table_view(eng.tower.gsum, k)[ids.index(0)]
            if step == 1:
                assert bool((g0 != 0).any()), n
            else:
                m0 = before[n][1][0] != 0
                assert bool((g0 == 0).all()) and bool(m0.any()), n
                assert bool((group.slot_dense(n, 0)[0] != before[n][0][0])[m0].all()), n


def test_replay_equals_step():
    B = 200
    ga, ea = _make(B, seed=4)
    gb, eb = _make(B, seed=4)
    sa, sb = _ps_state(ga), _ps_state(gb)
    for n in sa:
        assert all(torch.equal(x, y) for x, y in zip(sa[n], sb[n])), n  # the same seeded initial values
    for numeric, strings, labels in _batches(B, 4, 50):
        la = ea.step(numeric, strings, labels)
        lb = eb.replay(numeric, strings, labels)
        torch.cuda.synchronize()
        assert torch.equal(la, lb)
    ea.check()
    eb.check()
    sa, sb = _ps_state(ga), _ps_state(gb)
    for n in sa:
        for s in range(3):
            assert torch.equal(sa[n][s], sb[n][s]), (n, s)
    assert [v for v, _, _ in ga.snapshot()] == [v for v, _, _ in gb.snapshot()] == [4, 4]


def test_evaluate_accuracy_matches_numpy():
    B = 500
    group, eng = _make(B, seed=7)
    metrics = EvaluationMetrics(M.eval_metrics_fn(L))
    hits = n = 0
    for numeric, strings, labels in _batches(B, 3, 900):
        logits = eng.evaluate(numeric, strings, labels, metrics)
        torch.cuda.synchronize()
        nu = eng.n_unique.tolist()
        rows = [eng.tower.table_view(eng.rows, k)[:u] for k, u in enumerate(nu)]
        empty = torch.stack([strings[L.string_keys.index(k), :, 0] == 0 for k, _, _ in L.tables])
        ref = FD.fc_dnn_reference(L.spec(), numeric, eng.ids, empty, eng.inv, nu, rows, labels, eng.flat)
        FD.check({"logits": logits}, ref, n_sm=_n_sm())
        # census_functional.py:60-66: accuracy(int(squeeze(round(p))), int(label)); np.round is half to even
        p = 1.0 / (1.0 + np.exp(-logits.cpu().numpy().astype(np.float64)))
        hits += int((np.round(p).astype(np.int32) == labels.cpu().numpy().astype(np.int32)).sum())
        n += B
    acc = metrics.get_evaluation_summary()["logits"]["accuracy"]
    assert abs(float(acc) - hits / n) < 1e-6
    assert [v for v, _, _ in group.snapshot()] == [0, 0]  # nothing pushed


def test_engine_matches_dropin_trainer():
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    B, steps = 128, 4
    group_e, eng = _make(B, n_shards=1, seed=6)
    group_d = PSGroup(1, OPT_TYPE, OPT_ARGS, device=0)
    twin = ParameterServerModelHandler().get_model_to_train(M.FeatureColumnDNN(L)).to(DEV)
    assert all(isinstance(t, DenseTableEmbedding) for t in twin.tables)
    start = _ps_state(group_e)
    twin.load_mlp(torch.cat([start[n][0].reshape(-1) for n in M.MLP_NAMES]))
    twin.load_tables({n: start[n][0] for n in L.table_names})
    client = PSClient(group_d)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(twin, client, args=types.SimpleNamespace(cuda_graph=True))
    transform = L.transform(DEV)
    for step, (numeric, strings, labels) in enumerate(_batches(B, steps, 700)):
        loss_e = float(eng.step(numeric, strings, labels))
        accepted, version, loss_d = trainer.train_minibatch(M.twin_features(L, numeric, strings, transform), labels)
        assert accepted and version == step + 1
        assert abs(loss_e - float(loss_d)) <= 1e-4 * max(1.0, abs(loss_e)), (step, loss_e, float(loss_d))
        if step == 0:  # the twin lands on the engine's PS names, every one a dense parameter of the same shape
            assert {n: v[2:] for n, v in group_d.tables.items()} == {n: v[2:] for n, v in group_e.tables.items()}
            assert all(group_d.tables[n][2] for n in L.table_names)
    torch.cuda.synchronize()
    group_d.check()
    eng.check()
    assert trainer.graph_fallback_reason is None
    se, sd = _ps_state(group_e), _ps_state(group_d)
    for n in L.table_names + M.MLP_NAMES:
        for s, tol in enumerate((dict(rtol=1e-4, atol=1e-6), dict(rtol=1e-3, atol=1e-7), dict(rtol=1e-3, atol=1e-10))):
            torch.testing.assert_close(se[n][s], sd[n][s], **tol, msg=lambda m: "%s slot %d: %s" % (n, s, m))
    # rows no batch touched stayed at their initial values on both
    for n in L.table_names:
        untouched = (se[n][1] == 0).all(1)
        assert torch.equal(se[n][0][untouched], start[n][0][untouched])
        assert torch.equal(sd[n][0][untouched], start[n][0][untouched])


def test_earlier_layouts_keep_hashed_ps_tables():
    for L0 in (M.CENSUS_DNN, M.HEART):
        group = PSGroup(1, OPT_TYPE, OPT_ARGS, device=0)
        M.FeatureColumnDNNEngine(group, L0, 64, LR)
        for n in L0.table_names:
            _, _, is_dense, shape = group.tables[n]
            assert not is_dense and shape[0] is None, n  # hashed, rows created when pulled
        group.close()
