"""The float64 deepctr WDL oracle (oracle/deepctr_wdl_oracle.py) on the CPU: against float64 torch autograd of the
same model (the drop-in twin in float64), with clipped batches; the literal parameter table; the oracle's ids
against feature_oracle's Fingerprint64, "" included; and every mutation moving an output."""
import numpy as np
import pytest
import torch

from elasticdl_b200.workloads import deepctr_wdl as M
from oracle import deepctr_wdl_oracle as O
from oracle import feature_oracle as FO


def _raw(B, seed, empty_fraction=0.25):
    rng = np.random.RandomState(seed)
    raw = []
    for j in range(O.FIELDS):
        col = [b"%08x" % int(v) for v in rng.randint(0, 2 ** 32, B, dtype=np.int64)]
        for i in np.nonzero(rng.rand(B) < empty_fraction)[0]:
            col[i] = b""
        raw.append(col)
    return raw


def _batch(B, seed, gb=None, scale=0.3):
    g = torch.Generator().manual_seed(seed)
    raw = _raw(B, seed)
    ids = O.ids_from_raw(raw)
    dense = torch.rand((O.DENSE, B), generator=g, dtype=torch.float64) * 3
    labels = (torch.rand(B, generator=g) < 0.3).to(torch.float64)
    flat = M.initial_params(seed, "cpu").double()
    v = M.flat_views(flat)
    for n in M.LINEAR_NAMES[:5]:  # non-zero linear rows and larger deep rows, so that every term carries weight
        v[n].copy_(torch.randn(v[n].shape, generator=g, dtype=torch.float64) * 0.05)
    for n in M.DEEP_NAMES:
        v[n].mul_(scale / 1e-4 * 0.1)
    if gb is not None:
        v["prediction_layer/global_bias:0"].fill_(gb)
    return raw, ids, dense, labels, flat


def _autograd(ids, dense, labels, flat):
    twin = M.DeepctrWdl(optimizer="sgd").double()
    twin.load_flat(flat)
    p = twin({"ids": ids, "dense": dense})
    loss = twin.loss(labels, p)
    loss.backward()
    z = torch.logit(p.detach())
    grads = torch.cat([q.grad.reshape(-1) for q in twin.ordered()])
    return loss.detach(), z, grads


@pytest.mark.parametrize("B,gb", [(1, None), (37, None), (200, None), (64, 40.0), (64, -40.0)])
def test_oracle_matches_autograd(B, gb):
    _, ids, dense, labels, flat = _batch(B, B + 3, gb)
    ref = O.reference(ids, dense, labels, flat)
    loss, z, grads = _autograd(ids, dense, labels, flat)
    torch.testing.assert_close(ref["loss"], loss, rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(ref["grads"], grads, rtol=1e-9, atol=1e-15)
    if gb is None:
        torch.testing.assert_close(ref["logits"], z, rtol=1e-7, atol=1e-9)
    else:  # every p clipped: no gradient through the loss, only the regularizer's 2 lambda W
        _, lin, (wl, *_r) = O.unflatten(flat)
        want = torch.cat([2e-5 * flat[:O.N_TABLES], 2e-5 * wl.reshape(-1), torch.zeros(O.N_PARAMS - O.N_TABLES - 13,
                                                                                       dtype=torch.float64)])
        torch.testing.assert_close(ref["grads"], want, rtol=1e-12, atol=0)


def test_parameter_table():
    assert len(M.PARAMS) == 61 and M.N_PARAMS == 1371438
    assert sum(int(np.prod(s)) for _, s in M.PARAMS) == 1371438
    assert sum(int(np.prod(s)) for _, s in M.PARAMS[:52]) == 1300000
    assert M.PARAMS[0] == ("sparse_emb_C1/embeddings:0", (10000, 4))
    assert M.PARAMS[26] == ("linear0sparse_emb_C1/embeddings:0", (10000, 1))
    assert [n for n, _ in M.PARAMS[52:]] == ["linear/linear_kernel:0", "dnn/kernel0:0", "dnn/bias0:0", "dnn/kernel1:0",
                                             "dnn/bias1:0", "dnn/kernel2:0", "dnn/bias2:0", "dense/kernel:0",
                                             "prediction_layer/global_bias:0"]
    # the offsets include/b200_deepctr_wdl.h states
    assert [M.OFFSETS[n] for n in ("linear/linear_kernel:0", "dnn/kernel0:0", "dnn/bias0:0", "dnn/kernel1:0",
                                   "dnn/bias1:0", "dnn/kernel2:0", "dnn/bias2:0", "dense/kernel:0",
                                   "prediction_layer/global_bias:0")] == \
        [1300000, 1300013, 1329965, 1330221, 1362989, 1363117, 1371309, 1371373, 1371437]
    flat = M.initial_params(0, "cpu")
    v = M.flat_views(flat)
    assert all(float(v[n].abs().max()) == 0 for n in M.LINEAR_NAMES)
    assert abs(float(v["sparse_emb_C1/embeddings:0"].std()) - 1e-4) < 5e-6
    assert all(float(v[n].abs().max()) == 0 for n in ("dnn/bias0:0", "prediction_layer/global_bias:0"))
    k = v["dnn/kernel0:0"]
    assert abs(float(k.std()) - np.sqrt(2.0 / (117 + 256))) < 0.01 * np.sqrt(2.0 / (117 + 256)) * 5
    assert M.optimizer()[0] == "Adam" and M.optimizer()[2] == 1e-3


def test_ids_are_fingerprint64_with_empty_an_ordinary_bucket():
    raw = _raw(300, 5)
    ids = O.ids_from_raw(raw)
    for j in (0, 7, 25):
        want = [FO.fingerprint64(s) % 10000 for s in raw[j]]
        assert ids[j].tolist() == want
    assert FO.fingerprint64(b"") % 10000 == O.ids_from_raw([[b""]] * 26)[0, 0]
    assert bool((ids >= 0).all() and (ids < 10000).all())


def test_every_mutation_moves_an_output():
    B = 256
    raw, ids, dense, labels, flat = _batch(B, 11, gb=0.3)  # a zero global bias would hide its mutation
    ref = O.reference(ids, dense, labels, flat)
    got = {k: ref[k].to(torch.float32) for k in ("logits", "loss", "grads")}
    assert not O.caught_by(got, ref)
    muts = O.mutations(ids, dense, labels, flat, raw)
    assert set(muts) == set(O.MUTATIONS)
    for name, mut in muts.items():
        if name == "unclipped":
            continue
        assert O.caught_by(mut, ref), name
    _, ids, dense, labels, flat = _batch(B, 12, gb=40.0)
    ref = O.reference(ids, dense, labels, flat)
    assert O.caught_by(O.mutations(ids, dense, labels, flat, names=("unclipped",))["unclipped"], ref)
