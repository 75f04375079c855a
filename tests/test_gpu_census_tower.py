"""The census wide & deep tower (csrc/census_tower.cu, include/b200_census.h) and CensusWideDeepEngine against the
float64 oracle of oracle/census_oracle.py, in both reshape modes.

Kernel level: batches at the tile and grid edges (up to 2^17 and one sample past a full persistent grid's first
pass), id patterns with one touched row per table, every row touched and Zipf; the compacted rows and counts
exactly, everything else within the oracle's bound; the comparator's mutations; determinism and graph replay;
the refusals.  Engine level: raw Adult-shaped batches over SGD and Adam steps on one and two shards, the PS state
read back by name against OracleServer fed the engine's own gradients; raw rows against ids; four graphed workers
on cloned views, concurrent and serialised."""
import threading

import numpy as np
import pytest
import torch

from elasticdl_b200.ps import PSGroup
from elasticdl_b200.workloads import census as C
from elasticdl_b200.workloads.census_features import census_transform, synthetic_raw_batch
from oracle import census_oracle as O
from oracle.ps_oracle import OracleServer

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
OPTS = {"sgd": ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;", 0.1),
        "adam": ("Adam", "learning_rate=0.0003;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;", 3e-4)}


def _n_sm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ids(B, pattern, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    rows = []
    for g, r in enumerate(O.GROUP_ROWS):
        if pattern == "one":
            rows.append(torch.full((4, B), (7 * g + 3) % r, dtype=torch.int32, device=DEV))
        elif pattern == "all":
            rows.append(((torch.arange(4 * B, device=DEV) + g) % r).view(B, 4).t().to(torch.int32))
        else:  # zipf-like: small ids dominate
            u = torch.rand((4, B), generator=gen, device=DEV)
            rows.append(torch.clamp((r * u ** 3).floor(), max=r - 1).to(torch.int32))
    return torch.cat(rows).contiguous()


def _inputs(B, pattern, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    labels = (torch.rand(B, generator=gen, device=DEV) < 0.3).float()
    flat = O.random_params(gen, DEV, emb=0.5)
    return _ids(B, pattern, seed), labels, flat


def _dense(out):
    """The kernel's outputs with the compacted rows scattered into dense [rows, dim] tables."""
    gs = []
    for t in range(5):
        n = int(out["n_unique"][t])
        d = torch.zeros_like(out["gsum"][t])
        d[out["uniq"][t][:n]] = out["gsum"][t][:n]
        gs.append(d)
    return {"logits": out["logits"], "loss": out["loss"], "grads": out["grads"], "gsum": gs}


def _check_exact_rows(out, ref):
    for t in range(5):
        n = int(out["n_unique"][t])
        assert n == ref["n_unique"][t], t
        assert torch.equal(out["uniq"][t][:n].cpu(), ref["uniq"][t].cpu()), t


BATCHES = [1, 3, 64, 127, 128, 129, 4096, "wave+1", 1 << 17]


def _b(B):
    return _n_sm() * C.TILE + 1 if B == "wave+1" else B


@pytest.mark.parametrize("pattern", ["one", "all", "zipf"])
@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("reference_reshape", [False, True])
def test_tower_matches_oracle(reference_reshape, B, pattern):
    Bn = _b(B)
    ids, labels, flat = _inputs(Bn, pattern, seed=Bn % 1000)
    out = C.census_tower(ids, labels, flat, reference_reshape)
    ref = O.census_reference(ids, labels, flat, reference_reshape)
    _check_exact_rows(out, ref)
    O.check(_dense(out), ref, n_sm=_n_sm(), label="B=%d %s q11=%s" % (Bn, pattern, reference_reshape))


@pytest.mark.parametrize("B", [64, 4096, "wave+1"])
@pytest.mark.parametrize("reference_reshape", [False, True])
def test_mutations_are_caught(reference_reshape, B):
    Bn = _b(B)
    ids, labels, flat = _inputs(Bn, "zipf", seed=5)
    ref = O.census_reference(ids, labels, flat, reference_reshape)
    got = _dense(C.census_tower(ids, labels, flat, reference_reshape))
    assert not O.caught_by(got, ref, n_sm=_n_sm())
    for name, mut in O.mutations(ref, (ids, labels, flat, reference_reshape)).items():
        if name in ("drop_one_sample", "last_sample_twice") and Bn > 4096:
            continue  # one sample of 33793 moves each batch sum by less than the sqrt(n)-scaled bound
        assert O.caught_by(mut, ref, n_sm=_n_sm()), (name, Bn)


@pytest.mark.parametrize("reference_reshape", [False, True])
def test_deterministic_and_graph_replay(reference_reshape):
    B = 1 << 17
    ids, labels, flat = _inputs(B, "zipf", seed=9)
    call = C.CensusTowerCall(B, DEV)
    bufs = [call.loss, call.logits, call.grads, call.uniq, call.n_unique, call.gsum]
    call.launch(ids, labels, flat, reference_reshape)
    first = [b.clone() for b in bufs]
    call.launch(ids, labels, flat, reference_reshape)
    for a, b in zip(first, bufs):
        assert torch.equal(a, b)
    for b in bufs:
        b.fill_(float("nan") if b.is_floating_point() else -1)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call.launch(ids, labels, flat, reference_reshape)
    for _ in range(2):  # the arrival counter is back at zero after every replay
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(first, bufs):
            assert torch.equal(a, b)
    call.check_error()


def test_refusals():
    B = 64
    ids, labels, flat = _inputs(B, "zipf", seed=1)
    bad = ids.clone()
    bad[5, 3] = 75  # group 2's rows are 0..74
    bad[11, 0] = -1
    with pytest.raises(ValueError, match="2 census ids outside"):
        C.census_tower(bad, labels, flat)
    with pytest.raises(ValueError, match="ids must be"):
        C.census_tower(ids.long(), labels, flat)
    with pytest.raises(ValueError, match="ids must be"):
        C.census_tower(ids[:11].contiguous(), labels, flat)
    with pytest.raises(ValueError, match="labels must be"):
        C.census_tower(ids, labels.double(), flat)
    with pytest.raises(ValueError, match="params must be"):
        C.census_tower(ids, labels, flat[:-1])
    opt_type, opt_args, lr = OPTS["sgd"]
    with pytest.raises(ValueError, match="sync-SGD"):
        C.CensusWideDeepEngine(PSGroup(1, opt_type, opt_args, device=0, use_async=False), B, lr)
    with pytest.raises(ValueError, match="lr_staleness_modulation"):
        C.CensusWideDeepEngine(PSGroup(1, opt_type, opt_args, device=0, lr_staleness_modulation=True), B, lr)
    group = PSGroup(1, opt_type, opt_args, device=0)
    eng = C.CensusWideDeepEngine(group, B, lr)
    numeric, strings, _, _ = synthetic_raw_batch(B, 3, DEV)
    with pytest.raises(ValueError, match="numeric must be"):
        eng.step(numeric[:, :-1].contiguous(), strings, labels)
    with pytest.raises(ValueError, match="strings must be"):
        eng.step(numeric, strings.int(), labels)
    with pytest.raises(ValueError, match="labels must be"):
        eng.step(numeric, strings, labels[:-1])
    eng.step_ids(bad, labels)
    with pytest.raises(ValueError, match="census ids outside"):
        eng.check()
    eng.check()  # the count was cleared


def _servers(group, eng, opt):
    opt_type, opt_args, _ = OPTS[opt]
    servers = [OracleServer(s, opt_type, opt_args, num_ps=group.n_shards) for s in range(group.n_shards)]
    names = [n for n, _ in C.PARAMS]
    state = group.pull_dense(names)
    for s, srv in enumerate(servers):
        srv.push_model(dense={n: state[n].cpu().numpy() for n in names if eng.owner[n] == s})
    return servers


def _oracle_flat(servers, eng):
    flat = torch.zeros(C.N_PARAMS, dtype=torch.float32)
    v = C.flat_views(flat)
    for n, _ in C.PARAMS:
        v[n].copy_(torch.from_numpy(servers[eng.owner[n]].dense[n]).view(v[n].shape))
    return flat


def _push_to_oracle(servers, eng, lr, ref=None, label=""):
    """The engine's last step (its tower buffers) as one push per shard; with `ref`, its gradients are checked
    against the oracle first."""
    out = eng.tower.outputs()
    if ref is not None:
        _check_exact_rows(out, ref)
        O.check(_dense(out), ref, n_sm=_n_sm(), label=label)
    per = {s: ({}, {}) for s in range(len(servers))}
    for n, s in C.PARAMS[:6]:
        o = C.OFFSETS[n]
        per[eng.owner[n]][0][n] = out["grads"][o:o + int(np.prod(s))].cpu().numpy().reshape(s)
    for t, n in enumerate(C.TABLE_NAMES):
        k = int(out["n_unique"][t])
        per[eng.owner[n]][1][n] = (out["uniq"][t][:k].cpu().numpy().astype(np.int64),
                                   np.ascontiguousarray(out["gsum"][t][:k].cpu().numpy()))
    for s, srv in enumerate(servers):
        ok, _ = srv.push_gradients(per[s][0], per[s][1], lr, 0)
        assert ok


def _compare_state(group, servers, eng, opt):
    names = [n for n, _ in C.PARAMS]
    state = group.pull_dense(names)
    for n in names:
        srv = servers[eng.owner[n]]
        np.testing.assert_allclose(state[n].cpu().numpy(), srv.dense[n], rtol=1e-6, atol=1e-8, err_msg=n)
        if opt == "adam":
            for k, sn in enumerate(("m", "v")):
                np.testing.assert_allclose(group.slot_dense(n, k + 1).cpu().numpy(), srv.opt.dense_slots[sn][n],
                                           rtol=1e-5, atol=1e-12, err_msg=(n, sn))
    versions = [v for v, _, _ in group.snapshot()]
    assert versions == [srv.version for srv in servers]


@pytest.mark.parametrize("reference_reshape", [False, True])
@pytest.mark.parametrize("n_shards", [1, 2])
@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_engine_matches_oracle(opt, n_shards, reference_reshape):
    B, steps = 512, 5
    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(n_shards, opt_type, opt_args, device=0)
    eng = C.CensusWideDeepEngine(group, B, lr, reference_reshape=reference_reshape, seed=11)
    if n_shards == 2:
        assert len({eng.owner[n] for n, _ in C.PARAMS}) == 2
    servers = _servers(group, eng, opt)
    transform = census_transform(torch.int32, device=DEV)
    for step in range(steps):
        numeric, strings, _, _ = synthetic_raw_batch(B, 100 + step, DEV)
        labels = (torch.rand(B, generator=torch.Generator(device=DEV).manual_seed(step), device=DEV) < 0.25).float()
        before = _oracle_flat(servers, eng)
        loss = eng.step(numeric, strings, labels)
        torch.cuda.synchronize()
        eng.check()
        torch.testing.assert_close(eng.flat.cpu(), before, rtol=1e-6, atol=1e-8)
        ids, _ = transform(numeric, strings)
        ref = O.census_reference(ids, labels, eng.flat, reference_reshape)
        assert abs(float(loss) - float(ref["loss"])) <= 1e-5 * float(ref["M"]["loss"])
        _push_to_oracle(servers, eng, lr, ref, label="step %d" % step)
    torch.cuda.synchronize()
    _compare_state(group, servers, eng, opt)
    assert [v for v, _, _ in group.snapshot()] == [steps] * n_shards


def test_raw_rows_step_equals_ids_step():
    B = 300
    opt_type, opt_args, lr = OPTS["adam"]
    ga, gb = (PSGroup(2, opt_type, opt_args, device=0) for _ in range(2))
    ea, eb = C.CensusWideDeepEngine(ga, B, lr, seed=4), C.CensusWideDeepEngine(gb, B, lr, seed=4)
    transform = census_transform(torch.int32, device=DEV)
    for step in range(3):
        numeric, strings, _, _ = synthetic_raw_batch(B, 40 + step, DEV)
        labels = (torch.arange(B, device=DEV) % 3 == step).float()
        ea.step(numeric, strings, labels)
        eb.step_ids(transform(numeric, strings)[0], labels)
    names = [n for n, _ in C.PARAMS]
    sa, sb = ga.pull_dense(names), gb.pull_dense(names)
    for n in names:
        assert torch.equal(sa[n], sb[n]), n
        assert torch.equal(ga.slot_dense(n, 2), gb.slot_dense(n, 2)), n


def _worker_batches(w, B, n):
    out = []
    for s in range(n):
        numeric, strings, _, _ = synthetic_raw_batch(B, 1000 * (w + 1) + s, DEV)
        labels = (torch.rand(B, generator=torch.Generator(device=DEV).manual_seed(7 * w + s), device=DEV) < 0.3).float()
        out.append((numeric, strings, labels))
    return out


def _four_workers(opt, B):
    opt_type, opt_args, lr = OPTS[opt]
    group = PSGroup(2, opt_type, opt_args, device=0)
    engines = [C.CensusWideDeepEngine(group, B, lr, seed=5, register=(w == 0)) for w in range(4)]
    streams = [torch.cuda.Stream(device=DEV) for _ in range(4)]
    for e, s in zip(engines, streams):
        with torch.cuda.stream(s):
            e.capture()
    torch.cuda.synchronize()
    return group, engines, streams, lr


def test_four_workers_concurrent():
    B, steps = 256, 20
    group, engines, streams, _ = _four_workers("sgd", B)
    data = [_worker_batches(w, B, 4) for w in range(4)]
    torch.cuda.synchronize()
    errors = []

    def run(w):
        try:
            with torch.cuda.stream(streams[w]):
                for s in range(steps):
                    engines[w].replay(*data[w][s % 4])
                streams[w].synchronize()
        except Exception as e:  # noqa: BLE001
            errors.append((w, repr(e)))

    threads = [threading.Thread(target=run, args=(w,)) for w in range(4)]
    [t.start() for t in threads]
    [t.join() for t in threads]
    assert not errors, errors
    torch.cuda.synchronize()
    assert [v for v, _, _ in group.snapshot()] == [4 * steps] * 2
    for e in engines:
        e.check()


@pytest.mark.parametrize("opt", ["sgd", "adam"])
def test_four_workers_serialised_match_oracle(opt):
    B, rounds = 256, 3
    group, engines, streams, lr = _four_workers(opt, B)
    servers = _servers(group, engines[0], opt)
    data = [_worker_batches(w, B, rounds) for w in range(4)]
    for r in range(rounds):
        for w in range(4):
            with torch.cuda.stream(streams[w]):
                engines[w].replay(*data[w][r])
            streams[w].synchronize()
            _push_to_oracle(servers, engines[w], lr)
    _compare_state(group, servers, engines[0], opt)
    assert [v for v, _, _ in group.snapshot()] == [4 * rounds] * 2
