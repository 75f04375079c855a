"""The float64 census wide & deep oracle (oracle/census_oracle.py) on the CPU: against torch float64 autograd of the
drop-in twin's id-level forward (workloads.census.CensusWideDeep.tower) in both reshape modes, quirk Q11 pinned
by the reference's literal expression, and the parameter names, shapes and flat layout."""
import numpy as np
import pytest
import torch

from elasticdl_b200.workloads import census as C
from oracle import census_oracle as O


def _batch(B, seed):
    gen = torch.Generator().manual_seed(seed)
    ids = torch.cat([torch.randint(0, r, (4, B), generator=gen) for r in O.GROUP_ROWS])
    labels = (torch.rand(B, generator=gen) < 0.3).to(torch.float64)
    flat = O.random_params(gen, "cpu", emb=0.5, dtype=torch.float64)
    return ids, labels, flat


@pytest.mark.parametrize("reference_reshape", [False, True])
@pytest.mark.parametrize("B", [1, 2, 5, 64])
def test_oracle_matches_twin_autograd(B, reference_reshape):
    ids, labels, flat = _batch(B, seed=B + 10 * reference_reshape)
    ref = O.census_reference(ids, labels, flat, reference_reshape)
    model = C.CensusWideDeep(0.1, reference_reshape=reference_reshape).double()
    model.load_mlp(flat)
    v = C.flat_views(flat)
    tables = [v[n].clone().requires_grad_(True) for n in C.TABLE_NAMES]
    wide = torch.stack([tables[g][ids[4 * g:4 * g + 4]].sum(0)[:, 0] for g in range(2)])
    deep = torch.stack([tables[2 + g][ids[4 * g:4 * g + 4]].sum(0) for g in range(3)])
    z = model.tower(wide, deep)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(z, labels)
    lin = list(model.dense)
    params = [p for l in lin for p in (l.weight, l.bias)]
    got = torch.autograd.grad(loss, params + tables)
    torch.testing.assert_close(ref["logits"], z.detach(), rtol=1e-12, atol=1e-14)
    torch.testing.assert_close(ref["loss"], loss.detach(), rtol=1e-12, atol=1e-14)
    mlp = torch.cat([(g.t() if g.dim() == 2 else g).reshape(-1) for g in got[:6]])
    torch.testing.assert_close(ref["grads"], mlp, rtol=1e-10, atol=1e-14)
    for t in range(5):
        torch.testing.assert_close(ref["gsum"][t], got[6 + t], rtol=1e-10, atol=1e-14)
        touched = torch.zeros(O.GROUP_ROWS[O.TABLE_GROUP[t]], dtype=torch.bool)
        touched[ids[4 * O.TABLE_GROUP[t]:4 * O.TABLE_GROUP[t] + 4].reshape(-1)] = True
        assert torch.equal(ref["uniq"][t], torch.nonzero(touched).reshape(-1))
    # the magnitude pass bounds every value
    assert bool((ref["M"]["grads"] >= ref["grads"].abs() * (1 - 1e-12)).all())
    for t in range(5):
        assert bool((ref["M"]["gsum"][t] >= ref["gsum"][t].abs() * (1 - 1e-12)).all())


def test_q11_reference_reshape_pinned():
    """wide_deep_functional_api.py:203: tf.reshape(deep_embeddings, (-1, 24)) of a list of three [B, 8] tensors
    packs them to [3, B, 8] first; at B = 5 the oracle's quirk-mode input equals numpy's literal expression and
    differs from the per-sample concatenation."""
    B = 5
    ids, labels, flat = _batch(B, seed=3)
    ref_q = O.census_reference(ids, labels, flat, True)
    ref_d = O.census_reference(ids, labels, flat, False)
    v = C.flat_views(flat)
    e = [v[C.TABLE_NAMES[2 + g]][ids[4 * g:4 * g + 4]].sum(0).numpy() for g in range(3)]
    literal = np.stack([e[0], e[1], e[2]]).reshape(-1, 24)
    np.testing.assert_allclose(ref_q["x"].numpy(), literal, rtol=1e-14, atol=0)
    np.testing.assert_allclose(ref_d["x"].numpy(), np.concatenate(e, 1), rtol=1e-14, atol=0)
    assert not np.allclose(literal, np.concatenate(e, 1))
    # slot k of row r is group (3r + k) // B, sample (3r + k) % B
    for r in range(B):
        for k in range(3):
            g, s = divmod(3 * r + k, B)
            np.testing.assert_allclose(literal[r, 8 * k:8 * k + 8], e[g][s], rtol=1e-14, atol=0)


def test_parameter_names_shapes_and_layout():
    names = ["dense/kernel:0", "dense/bias:0", "dense_1/kernel:0", "dense_1/bias:0", "dense_2/kernel:0",
             "dense_2/bias:0", "embedding/embeddings:0", "embedding_1/embeddings:0", "embedding_2/embeddings:0",
             "embedding_3/embeddings:0", "embedding_4/embeddings:0"]
    shapes = [(24, 16), (16,), (16, 8), (8,), (8, 4), (4,), (28, 1), (75, 1), (28, 8), (75, 8), (115, 8)]
    assert C.PARAMS == list(zip(names, shapes)) == O.PARAMS
    assert [C.OFFSETS[n] for n in names] == [0, 384, 400, 528, 536, 568, 572, 600, 675, 899, 1499]
    assert C.OFFSETS == O.OFFSETS and C.N_PARAMS == O.N_PARAMS == 2419 and C.N_MLP == 572
    assert C.UNIQ_OFF == O.UNIQ_OFF and C.GSUM_OFF == O.GSUM_OFF
    assert C.GROUP_ROWS == O.GROUP_ROWS == (28, 75, 115)
    flat = torch.arange(C.N_PARAMS, dtype=torch.float32)
    v = C.flat_views(flat)
    assert float(v["dense/kernel:0"][1, 0]) == 16  # [in, out] row-major
    assert float(v["embedding_4/embeddings:0"][114, 7]) == 2418
    init = C.initial_params(5, "cpu")
    iv = C.flat_views(init)
    for n, s in C.PARAMS:
        if n.endswith("bias:0"):
            assert float(iv[n].abs().max()) == 0
        elif n.endswith("embeddings:0"):
            assert 0 < float(iv[n].abs().max()) <= 0.05
        else:
            assert 0 < float(iv[n].abs().max()) <= (6.0 / (s[0] + s[1])) ** 0.5
    assert torch.equal(init, C.initial_params(5, "cpu"))
