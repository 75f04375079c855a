"""GPU tests of the reference-facing layer/trainer mirrors and the fused DeepFM engine.
Vectors follow elasticdl/python/tests/layer_test.py:135-383 (fake lookup returning
[id]*dim rows) and worker_ps_interaction_test.py:203-270 (PS training == local training)."""
import numpy as np
import pytest
import torch

from oracle import ps_oracle as O

pytestmark = pytest.mark.gpu
F = np.float32
SGD = ("SGD", "learning_rate=0.1;momentum=0.0;nesterov=false;")
ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")


def fake_lookup(dim):
    def fn(name, ids):  # layer_test.py:71-101 mock_worker.lookup_embedding
        return ids.to(torch.float32).unsqueeze(1).repeat(1, dim)
    return fn


def test_embedding_layer_forward_and_bet_grads_layer_test_py_135():
    from elasticdl_b200.layers import Embedding

    layer = Embedding(8, input_dim=10, name="emb_a")
    layer.set_lookup_embedding_func(fake_lookup(8))
    ids = torch.tensor([[0, 1, 3], [8, 3, 2], [3, 3, 3]], device="cuda")
    out = layer(ids)
    assert out.shape == (3, 3, 8)
    assert torch.equal(out, ids.float().unsqueeze(-1).expand(3, 3, 8))
    assert layer.embedding_and_ids == []  # nothing recorded without a tape
    layer.set_tape(True)
    out = layer(ids)
    (bet, batch_ids), = layer.embedding_and_ids
    assert batch_ids.tolist() == [0, 1, 3, 8, 2]  # tf.unique order
    up = torch.arange(9 * 8, device="cuda", dtype=torch.float32).reshape(3, 3, 8)
    (g,) = torch.autograd.grad((out * up).sum(), [bet])
    flat = ids.reshape(-1).tolist()
    want = torch.zeros(5, 8, device="cuda")
    for pos, i in enumerate(flat):
        want[[0, 1, 3, 8, 2].index(i)] += up.reshape(9, 8)[pos]
    assert torch.equal(g, want)
    layer.reset()
    assert layer.embedding_and_ids == [] and layer.tape is None
    assert layer.embedding_weight_name == "emb_a/embeddings:0"
    with pytest.raises(ValueError):  # embedding_delegate.py:254-264
        layer(torch.tensor([1, 50], device="cuda"))


@pytest.mark.parametrize("combiner", ["sum", "mean", "sqrtn"])
def test_embedding_layer_sparse_combiners_layer_test_py(combiner):
    from elasticdl_b200.layers import Embedding

    layer = Embedding(4, combiner=combiner, name="emb_s_" + combiner)
    layer.set_lookup_embedding_func(fake_lookup(4))
    # rows: [1,2], [], [3,-1(pruned)], [5,5,7]
    idx = torch.tensor([[0, 0, 2, 2, 3, 3, 3], [0, 1, 0, 1, 0, 1, 2]], device="cuda")
    val = torch.tensor([1, 2, 3, -1, 5, 5, 7], device="cuda")
    sp = torch.sparse_coo_tensor(idx, val, (4, 3))
    out = layer(sp)
    rows = [[1, 2], [], [3], [5, 5, 7]]
    want = torch.zeros(4, 4)
    for r, ids in enumerate(rows):
        if ids:
            s = float(sum(ids))
            want[r] = {"sum": s, "mean": s / len(ids), "sqrtn": s / len(ids) ** 0.5}[combiner]
    assert torch.allclose(out.cpu(), want, atol=1e-6)
    with pytest.raises(ValueError):
        Embedding(4, name="emb_nocomb")(sp)


class TinyModel(torch.nn.Module):
    def __init__(self, dim=8, rows=50):
        super().__init__()
        from elasticdl_b200.layers import Embedding

        self.emb = Embedding(dim, input_dim=rows, embeddings_initializer="zero", name="tiny_emb")
        self.fc = torch.nn.Linear(3 * dim, 1)
        self.optimizer = torch.optim.SGD(self.fc.parameters(), lr=0.1)
        self.loss = lambda labels, out: ((out.squeeze(1) - labels) ** 2).mean()

    def forward(self, ids):
        e = self.emb(ids)
        return self.fc(e.reshape(ids.shape[0], -1))


@pytest.mark.parametrize("n_shards", [1, 2])
def test_trainer_equals_local_training_worker_ps_interaction_test_py_203(n_shards):
    """PS training (SGD) == local torch training on the same data."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    torch.manual_seed(0)
    model = TinyModel().cuda()
    group = PSGroup(n_shards, *SGD, device=0)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client)
    # local twin: nn.Embedding holding the table, same init
    rows, dim = 50, 8
    init = torch.randn(rows, dim, device="cuda") * 0.1
    group.set_rows([("tiny_emb/embeddings:0", torch.arange(rows), init)])
    table = init.clone().requires_grad_(True)
    fc = torch.nn.Linear(3 * dim, 1).cuda()
    fc.load_state_dict(model.fc.state_dict())
    opt = torch.optim.SGD([table] + list(fc.parameters()), lr=0.1)
    gen = torch.Generator().manual_seed(1)
    for step in range(4):
        ids = torch.randint(0, rows, (16, 3), generator=gen).cuda()
        labels = torch.randn(16, generator=gen).cuda()
        accepted, version, loss = trainer.train_minibatch(ids, labels)
        assert accepted and version == step + 1
        opt.zero_grad()
        l2 = ((fc(table[ids].reshape(16, -1)).squeeze(1) - labels) ** 2).mean()
        l2.backward()
        opt.step()
        assert abs(float(loss) - float(l2)) < 1e-5
    got = client.pull_embedding_vectors("tiny_emb/embeddings:0", torch.arange(rows).cuda())
    assert torch.allclose(got, table.detach(), rtol=1e-5, atol=1e-6)
    versions = [-1] * n_shards
    params, _ = client.pull_dense_parameters(list(range(n_shards)), versions)
    assert torch.allclose(params["fc.weight"], fc.weight.detach(), rtol=1e-5, atol=1e-6)
    assert torch.allclose(params["fc.bias"], fc.bias.detach(), rtol=1e-5, atol=1e-6)
    assert trainer.get_model_version() >= 3
    group.close()


@pytest.mark.parametrize("get_model_steps", [1, 3])
def test_train_loop_get_model_steps_worker_py_346(get_model_steps):
    """The worker loop of worker.py:338-370: the dense model is pulled every `get_model_steps` minibatches,
    in between the worker trains on its local model advanced by _update_local_model (ps_trainer.py:139-147).
    With one worker and SGD on both sides the local model tracks the PS exactly, so the run must equal plain
    local torch training -- and _get_model must have run only at minibatches 0, 3, 6."""
    import types

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    torch.manual_seed(0)
    model = TinyModel().cuda()
    group = PSGroup(2, *SGD, device=0)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(get_model_steps=get_model_steps))
    rows, dim, steps = 50, 8, 7
    init = torch.randn(rows, dim, device="cuda") * 0.1
    group.set_rows([("tiny_emb/embeddings:0", torch.arange(rows), init)])
    table = init.clone().requires_grad_(True)
    fc = torch.nn.Linear(3 * dim, 1).cuda()
    fc.load_state_dict(model.fc.state_dict())
    opt = torch.optim.SGD([table] + list(fc.parameters()), lr=0.1)
    gen = torch.Generator().manual_seed(1)
    batches = [(torch.randint(0, rows, (16, 3), generator=gen).cuda(), torch.randn(16, generator=gen).cuda())
               for _ in range(steps)]
    pulls, flags = [], []
    orig = trainer._get_model

    def counting_get_model():
        pulls.append(len(flags))
        orig()

    trainer._get_model = counting_get_model
    out = trainer.train_loop(batches, on_step=lambda local, err: flags.append((local, err)))
    assert [f[1] for f in flags] == [""] * steps
    assert pulls == list(range(0, steps, get_model_steps))
    assert [f[0] for f in flags] == [i % get_model_steps != 0 for i in range(steps)]
    for (ids, labels), (version, loss) in zip(batches, out):
        opt.zero_grad()
        l2 = ((fc(table[ids].reshape(16, -1)).squeeze(1) - labels) ** 2).mean()
        l2.backward()
        opt.step()
        assert abs(float(loss) - float(l2)) < 1e-5
    assert [v for v, _ in out] == list(range(1, steps + 1))
    params, _ = client.pull_dense_parameters([0, 1], [-1, -1])
    assert torch.allclose(params["fc.weight"], fc.weight.detach(), rtol=1e-5, atol=1e-6)
    assert torch.allclose(params["fc.bias"], fc.bias.detach(), rtol=1e-5, atol=1e-6)
    # the worker's local copy after the last local update equals the PS too (single worker, SGD both sides)
    if get_model_steps > 1 and steps % get_model_steps != 0:
        assert torch.allclose(model.fc.weight.detach(), fc.weight.detach(), rtol=1e-5, atol=1e-6)
    group.close()


def _torch_reference_grads(eng, tower, wide0, deep0, ids, dense, labels):
    rows_n = len(wide0)
    wt = [w.clone().requires_grad_(True) for w in wide0]
    dt = [d.clone().requires_grad_(True) for d in deep0]
    wide = torch.stack([wt[g][ids[g]].squeeze(1) for g in range(rows_n)], 1)
    deep = torch.stack([dt[g][ids[g]] for g in range(rows_n)], 1)
    loss = torch.nn.BCEWithLogitsLoss()(tower(dense, wide, deep), labels)
    grads = torch.autograd.grad(loss, wt + dt + list(tower.parameters()))
    return float(loss), grads


@pytest.mark.parametrize("tower_kind,paired", [("tile", False), ("fused", True), ("fused", False), ("torch", True), ("mma", False)])
@pytest.mark.parametrize("n_shards,B,rows", [(1, 256, [5, 9, 300, 2000, 17]), (4, 1000, [3, 50000, 7, 100]),
                                             (2, 4096, None)])
def test_deepfm_engine_step_matches_oracle_adam(n_shards, B, rows, tower_kind, paired):
    """One engine step: (a) the tower's gradients == plain torch fp32 autograd over dense tables,
    (b) the PS state after the push == the oracle's Adam applied to those gradients."""
    import copy

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import GROUP_ROWS, DeepFMPSEngine, synthetic_batch

    full = rows is None
    rows = list(GROUP_ROWS) if full else rows
    if full:  # keep the dense torch replica small: cap the big tables
        rows = [min(r, 20000) for r in rows]
    D, G = 8, len(rows)
    group = PSGroup(n_shards, *ADAM, device=0)
    eng = DeepFMPSEngine(group, B, group_rows=rows, tower=tower_kind, paired=paired)
    dev = torch.device("cuda", 0)
    ids, dense, labels = synthetic_batch(B, 5, dev, "zipf", group_rows=rows)
    wide0 = [group.pull_rows([(n, torch.arange(r))])[0] for n, r in zip(eng.wide_names, rows)]
    deep0 = [group.pull_rows([(n, torch.arange(r))])[0] for n, r in zip(eng.deep_names, rows)]
    tower = copy.deepcopy(eng.tower)
    loss = float(eng.step(ids, dense, labels))
    group.check()
    ref_loss, ref = _torch_reference_grads(eng, tower, wide0, deep0, ids, dense, labels)
    assert abs(loss - ref_loss) < 2e-6
    # (a) gradients
    n_unique = eng.n_unique.cpu().numpy()
    uniq = eng.uniq.cpu().numpy().reshape(G, B)
    gsum_w = eng.gsum_w.cpu().numpy().reshape(G, B)
    gsum_d = eng.gsum_d.cpu().numpy().reshape(G, B, D)
    if tower_kind in ("tile", "fused", "mma"):
        dense_grads = [eng.flat_grads[off:off + n].cpu().numpy() for off, n in eng.flat_views]
    else:
        dense_grads = [g_.cpu().numpy().reshape(-1) for g_ in eng._dense_grads]
    for g in range(G):
        u = int(n_unique[g])
        ids_u = uniq[g, :u]
        assert np.array_equal(ids_u, O.unique_first_occurrence(ids[g].cpu().numpy())[0])
        rw = ref[g].cpu().numpy()[ids_u, 0]
        rd = ref[G + g].cpu().numpy()[ids_u]
        assert np.allclose(gsum_w[g, :u], rw, rtol=1e-4, atol=1e-8), g
        assert np.allclose(gsum_d[g, :u], rd, rtol=1e-4, atol=1e-8), g
    for got, want, (name, _) in zip(dense_grads, ref[2 * G:], eng.params):
        w = want.cpu().numpy().reshape(-1)
        assert np.allclose(got, w, rtol=2e-4, atol=1e-8 + 1e-5 * np.abs(w).max()), name
    # (b) PS state == oracle Adam (step 1) on the gradients the engine pushed
    for names, t0, gsum, dim in ((eng.wide_names, wide0, gsum_w[..., None], 1), (eng.deep_names, deep0, gsum_d, D)):
        for g in range(G):
            u = int(n_unique[g])
            touched = uniq[g, :u]
            p = t0[g].cpu().numpy()[touched].copy()
            m, v = np.zeros_like(p), np.zeros_like(p)
            O.np_adam(gsum[g, :u].reshape(u, dim).copy(), p, m, v, 0.001, 1, 0.9, 0.999, 1e-7)
            got = group.pull_rows([(names[g], torch.from_numpy(touched))])[0].cpu().numpy()
            assert np.array_equal(got, p), (names[g])
            assert np.array_equal(group.slot_rows(names[g], touched, 1).cpu().numpy(), m)
            assert np.array_equal(group.slot_rows(names[g], touched, 2).cpu().numpy(), v)
            assert group.table_size(names[g]) == rows[g]
    for (name, _), gr, pref in zip(eng.params, dense_grads, tower.parameters()):
        want = pref.detach().cpu().numpy().reshape(-1).copy()
        m, v = np.zeros_like(want), np.zeros_like(want)
        O.np_adam(gr.copy(), want, m, v, 0.001, 1, 0.9, 0.999, 1e-7)
        got = group.pull_dense([name])[name].cpu().numpy().reshape(-1)
        assert np.array_equal(got, want), name
    assert [s_[0] for s_ in group.snapshot()] == [1] * n_shards
    # forward-only path agrees with the float64 reference logits of the updated model (rows and dense
    # parameters pulled from the PS)
    if tower_kind in ("fused", "tile"):
        from oracle import tower_oracle as T

        logits = eng.predict(ids, dense)
        _, ref_after = _ps_reference(group, eng, ids, dense, labels)
        T.check({"logits": logits}, ref_after, families=("logits",), label="predict",
                n_sm=torch.cuda.get_device_properties(0).multi_processor_count)
    # training makes progress on a fixed batch
    for _ in range(30):
        l_last = float(eng.step(ids, dense, labels))
    assert l_last < loss
    group.close()


def _ps_reference(group, eng, ids, dense, labels, dense_params=None):
    """The float64 tower reference (oracle/tower_oracle.py) of one batch from what the PS holds now: the
    rows of the batch's ids only (first-occurrence order, like the engine's dedup) and the dense parameters
    (or `dense_params`, {name: values}, where the PS holds none yet).
    Returns ((inv, n_unique, bet_wide, bet_deep, dense, labels, params), reference)."""
    from oracle import tower_oracle as T

    G, B, dev = eng.G, eng.B, eng.device
    inv, n_unique, uniq = T.first_occurrence_inverse(ids)
    bet_w = torch.full((G, B), float("nan"), device=dev)
    bet_d = torch.full((G, B, T.D), float("nan"), device=dev)
    for g in range(G):
        u = int(n_unique[g])
        touched = uniq[g, :u].cpu()
        bet_w[g, :u] = group.pull_rows([(eng.wide_names[g], touched)])[0].reshape(u).to(dev)
        bet_d[g, :u] = group.pull_rows([(eng.deep_names[g], touched)])[0].reshape(u, T.D).to(dev)
    d = group.pull_dense([n for n, _ in eng.params]) if dense_params is None else dense_params
    params = torch.zeros(T.layout(G)["total"], dtype=torch.float32, device=dev)
    for (name, _), (off, n) in zip(eng.params, eng.flat_views):
        params[off:off + n] = torch.as_tensor(d[name]).reshape(-1).to(dev)
    inputs = (inv, n_unique, bet_w, bet_d, dense, labels, params)
    return inputs, T.tower_reference(*inputs)


def _engine_state(group, eng, rows):
    t = [group.pull_rows([(n, torch.arange(r))])[0].cpu().numpy() for n, r in zip(eng.wide_names + eng.deep_names, rows + rows)]
    d = group.pull_dense([n for n, _ in eng.params])
    return t + [d[n].cpu().numpy() for n, _ in eng.params]


@pytest.mark.parametrize("use_graph", [False, True])
def test_engine_lookahead_pipeline_matches_plain_steps(use_graph):
    """prepare/step_ahead (dedup of batch i+1 on a second stream while batch i trains) runs the same
    kernels on the same data as step(): same losses, rows and dense parameters up to the order of the
    fp32 atomic adds in the loss / gradient reductions (two plain runs differ by as much)."""
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, HostFeeder, synthetic_batch

    rows, B, steps = [11, 700, 5000, 9, 64], 256, 6
    batches = [synthetic_batch(B, 40 + i, torch.device("cuda", 0), "zipf", group_rows=rows) for i in range(steps)]
    results = []
    for mode in ("plain", "ahead"):
        group = PSGroup(2, *ADAM, device=0)
        eng = DeepFMPSEngine(group, B, group_rows=rows)
        losses = []
        if mode == "plain":
            for ids, dense, labels in batches:
                losses.append(float(eng.step(ids, dense, labels)))
        elif not use_graph:
            eng.prepare(batches[0][0])
            for i, (_, dense, labels) in enumerate(batches):
                losses.append(float(eng.step_ahead(dense, labels, batches[min(i + 1, steps - 1)][0])))
        else:  # through the host feeder: pinned host batches, captured graphs
            feeder = HostFeeder(eng, 3, lookahead=True)
            host = [tuple(t.cpu().pin_memory() for t in b) for b in batches]
            feeder.submit(*host[0])
            feeder.submit(*host[1])
            for i in range(steps):
                if i + 2 < steps:
                    feeder.submit(*host[i + 2])
                losses.append(float(feeder.run_next()))
        group.check()
        # every step also stored its loss into the pinned host ring (b200_deepfm_publish_loss): same values,
        # read without any D2H copy
        ring = [eng.loss_host(eng.steps - steps + i) for i in range(steps)]
        assert ring == losses, (ring, losses)
        results.append((losses, _engine_state(group, eng, rows), [s_[0] for s_ in group.snapshot()]))
        group.close()
    (l0, s0, v0), (l1, s1, v1) = results
    assert np.allclose(l0, l1, rtol=1e-5, atol=0), (l0, l1)
    assert v0 == v1 == [steps, steps]
    for a, b in zip(s0, s1):
        assert np.allclose(a, b, rtol=0, atol=2e-4), float(np.abs(a - b).max())


def _torchrun_two_ranks(script, port):
    """Two ranks through torchrun: one per GPU when the box has two, otherwise both as processes on cuda:0
    (B200_SHARED_GPU=1: CUDA IPC between the processes, gloo for the host plumbing -- see tests/mgpu_check.py)."""
    import os
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    if torch.cuda.device_count() < 2:
        env["B200_SHARED_GPU"] = "1"
    return subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                           "--master-addr", "127.0.0.1", "--master-port", str(port),
                           os.path.join(root, "tests", script)], capture_output=True, text=True, timeout=900, env=env)


def test_multi_gpu_peer_shards_via_torchrun():
    """Rank-per-process group with CUDA-IPC peer shards (one rank per GPU, or two processes on one GPU)."""
    out = _torchrun_two_ranks("mgpu_check.py", 29533)
    assert out.returncode == 0 and "mgpu_check ok" in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


@pytest.mark.parametrize("script,token", [("mgpu_xchg_check.py", "mgpu_xchg_check ok"),
                                          ("mgpu_allreduce_check.py", "mgpu_allreduce ok")])
def test_multi_gpu_exchange_and_allreduce_via_torchrun(script, token):
    """Owner-computes exchange set-up (create refusals, a DeepFM engine training on it; its data paths are
    tests/test_gpu_exchange_paths.py) and the allreduce controller incl. its fused reduce+update (NCCL with two
    GPUs; on one GPU the two ranks share it)."""
    out = _torchrun_two_ranks(script, 29534)
    assert out.returncode == 0 and token in out.stdout, out.stdout[-3000:] + out.stderr[-3000:]


@pytest.mark.parametrize("n_shards,views", [(1, True), (2, False)])
def test_trainer_batched_lookups_equal_per_layer_lookups(n_shards, views):
    """The trainer's batched lookups (one unique + one gather per layer group, ONE pull launch, counts kept
    on the device) train exactly like the per-layer path of embedding_delegate.py:75-106: same losses, same
    tables and dense parameters after 4 Adam minibatches of a 2 x 5-layer DeepFM -- with far fewer launches and
    no per-layer host reads.  Feature tensors are row views of one array, or separately allocated."""
    import types

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer
    from elasticdl_b200.workloads.deepfm import DeepFMLayersModel

    rows = [7, 300, 5000, 40, 1200]
    B = 512

    def run(batched):
        torch.manual_seed(3)
        model = DeepFMLayersModel(rows, lr=0.01, initializer="uniform").cuda()
        group = PSGroup(n_shards, *ADAM, device=0, seed=11)
        client = PSClient(group)
        client.dense_output = "torch"
        trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
            get_model_steps=1, batched_embedding_lookups=batched))
        gen = torch.Generator().manual_seed(5)
        losses, launches = [], []
        for step in range(4):
            ids = torch.stack([torch.randint(0, r, (B,), generator=gen) for r in rows]).cuda()
            dense = torch.randn(B, 13, generator=gen).cuda()
            labels = (torch.rand(B, generator=gen) < 0.3).float().cuda()
            feats = DeepFMLayersModel.features_of(ids if views else ids.clone(), dense)
            if not views:
                feats.update({"ids_%d" % g: ids[g].clone() for g in range(len(rows))})
            count = lambda: group.launch_count + int(group.lib.b200ps_launch_count(None))  # noqa: E731
            before = count()
            accepted, version, loss = trainer.train_minibatch(feats, labels)
            launches.append(count() - before)
            assert accepted and version == step + 1
            losses.append(float(loss))
        tabs = {}
        for g, r in enumerate(rows):
            for fam in ("deep", "wide"):
                name = "%s_%d/embeddings:0" % (fam, g)
                tabs[name] = client.pull_embedding_vectors(name, torch.arange(r).cuda()).cpu()
        params, _ = client.pull_dense_parameters(list(range(n_shards)), [-1] * n_shards)
        params = {k: v.cpu() for k, v in params.items()}
        plan = trainer._lookup_plan
        group.close()
        return losses, tabs, params, launches, plan

    l_b, t_b, p_b, n_b, plan = run(True)
    l_p, t_p, p_p, n_p, plan_p = run(False)
    assert plan and plan_p is False
    assert sorted((k, dim, len(m)) for k, dim, m in plan) == [(B, 1, 5), (B, 8, 5)]
    assert np.allclose(l_b, l_p, rtol=1e-6, atol=1e-7)
    for name in t_p:
        assert torch.allclose(t_b[name], t_p[name], rtol=1e-5, atol=1e-7), name
    for name in p_p:
        assert torch.allclose(p_b[name], p_p[name], rtol=1e-5, atol=1e-7), name
    assert n_b[0] == n_p[0]          # the first minibatch learns the plan on the per-layer path
    assert n_b[-1] * 2 < n_p[-1]     # afterwards: a handful of launches instead of several per layer


@pytest.mark.parametrize("n_shards,views", [(1, True), (2, False)])
def test_trainer_cuda_graph_minibatch_equals_eager(n_shards, views):
    """args.cuda_graph=True: after the eager warm-up minibatches the whole train_minibatch (dense pull into the
    model, batched lookups, forward, loss, autograd, push) is ONE CUDA-graph replay over static copies of the
    inputs.  Same (accepted, version, loss) per minibatch, same tables and dense parameters as the eager trainer
    after 8 Adam minibatches; an id outside its table still raises (the error word is read after every replay)."""
    import types

    from elasticdl_b200 import _lib
    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer
    from elasticdl_b200.workloads.deepfm import DeepFMLayersModel

    rows = [7, 300, 5000, 40, 1200]
    B = 512

    def batch(gen):
        ids = torch.stack([torch.randint(0, r, (B,), generator=gen) for r in rows]).cuda()
        dense = torch.randn(B, 13, generator=gen).cuda()
        labels = (torch.rand(B, generator=gen) < 0.3).float().cuda()
        feats = DeepFMLayersModel.features_of(ids if views else ids.clone(), dense)
        if not views:
            feats.update({"ids_%d" % g: ids[g].clone() for g in range(len(rows))})
        return feats, labels

    def run(graphed):
        torch.manual_seed(3)
        model = DeepFMLayersModel(rows, lr=0.01, initializer="uniform").cuda()
        group = PSGroup(n_shards, *ADAM, device=0, seed=11)
        client = PSClient(group)
        client.dense_output = "torch"
        trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
            get_model_steps=1, batched_embedding_lookups=True, cuda_graph=graphed, cuda_graph_warmup=2))
        gen = torch.Generator().manual_seed(5)
        losses, modes = [], []
        for step in range(8):
            feats, labels = batch(gen)
            accepted, version, loss = trainer.train_minibatch(feats, labels)
            assert accepted and version == step + 1, (step, version)
            losses.append(float(loss))
            modes.append(isinstance(trainer._graph_state, dict))
        assert trainer.get_model_version() == 7
        tabs = {}
        for g, r in enumerate(rows):
            for fam in ("deep", "wide"):
                name = "%s_%d/embeddings:0" % (fam, g)
                tabs[name] = client.pull_embedding_vectors(name, torch.arange(r).cuda()).cpu()
        params, _ = client.pull_dense_parameters(list(range(n_shards)), [-1] * n_shards)
        params = {k: v.cpu() for k, v in params.items()}
        local = {k: v.detach().cpu().clone() for k, v in model.named_parameters()}
        if graphed:
            assert trainer.graph_fallback_reason is None, trainer.graph_fallback_reason
            assert modes == [False, False] + [True] * 6, modes
            # a one-off short minibatch (the last batch of an epoch) runs eagerly and keeps the graph; the same new
            # shape twice in a row is captured again
            first = trainer._graph_state
            feats, labels = batch(gen)
            half = ({k: v[: B // 2].contiguous() for k, v in feats.items()}, labels[: B // 2].contiguous())
            assert trainer.train_minibatch(*half)[:2] == (True, 9) and trainer._graph_state is first
            assert trainer.train_minibatch(feats, labels)[:2] == (True, 10) and trainer._graph_state is first
            assert trainer.train_minibatch(*half)[:2] == (True, 11) and trainer._graph_state is first
            assert trainer.train_minibatch(*half)[:2] == (True, 12)
            assert isinstance(trainer._graph_state, dict) and trainer._graph_state is not first
            assert trainer._graph_state["recaptures"] == 1 and trainer.graph_fallback_reason is None
            feats, labels = batch(gen)
            feats = {k: v[: B // 2].contiguous() for k, v in feats.items()}
            labels = labels[: B // 2].contiguous()
            feats["ids_1"] = feats["ids_1"] + 10 ** 6  # outside table 1: flagged by the kernels, read after the replay
            with pytest.raises(_lib.PSError):
                trainer.train_minibatch(feats, labels)
        group.close()
        return losses, tabs, params, local

    l_g, t_g, p_g, m_g = run(True)
    l_e, t_e, p_e, m_e = run(False)
    assert np.allclose(l_g, l_e, rtol=1e-5, atol=1e-6), (l_g, l_e)
    for name in t_e:
        assert torch.allclose(t_g[name], t_e[name], rtol=1e-5, atol=1e-7), name
    for name in p_e:
        assert torch.allclose(p_g[name], p_e[name], rtol=1e-5, atol=1e-7), name
    for name in m_e:  # the model's own tensors hold what the last pull wrote, in both modes
        assert torch.allclose(m_g[name], m_e[name], rtol=1e-5, atol=1e-7), name


def test_trainer_cuda_graph_falls_back_when_not_eligible():
    """A staleness-modulated PS (the pulled versions travel with every push) keeps the eager path and says why."""
    import types

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer
    from elasticdl_b200.workloads.deepfm import DeepFMLayersModel

    rows = [7, 300]
    torch.manual_seed(0)
    model = DeepFMLayersModel(rows, lr=0.01).cuda()
    group = PSGroup(1, *ADAM, device=0, lr_staleness_modulation=True)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(cuda_graph=True, cuda_graph_warmup=1))
    gen = torch.Generator().manual_seed(5)
    for step in range(3):
        ids = torch.stack([torch.randint(0, r, (64,), generator=gen) for r in rows]).cuda()
        feats = DeepFMLayersModel.features_of(ids, torch.randn(64, 13, generator=gen).cuda())
        accepted, version, _ = trainer.train_minibatch(feats, (torch.rand(64, generator=gen) < 0.3).float().cuda())
        assert accepted and version == step + 1
    assert trainer._graph_state is False and "staleness" in trainer.graph_fallback_reason
    group.close()


class MnistFunctional(torch.nn.Module):
    """model_zoo/mnist/mnist_functional_api.py:21-31 in torch (BASELINE configs[0]): conv 3x3x1x32, conv 3x3x32x64,
    BatchNorm(64), max-pool 2x2, dense 9216 -> 10 (the Dropout(0.25) is left out: two runs must be comparable)."""

    def __init__(self, lr=0.01):
        super().__init__()
        self.c1 = torch.nn.Conv2d(1, 32, 3)
        self.c2 = torch.nn.Conv2d(32, 64, 3)
        self.bn = torch.nn.BatchNorm2d(64)
        self.fc = torch.nn.Linear(9216, 10)
        self.optimizer = torch.optim.SGD(self.parameters(), lr=lr)  # mnist_functional_api.py:66-67
        ce = torch.nn.CrossEntropyLoss()
        self.loss = lambda labels, logits: ce(logits, labels.reshape(-1))  # :57-63

    def forward(self, image):
        x = torch.relu(self.c1(image.reshape(-1, 1, 28, 28)))
        x = torch.relu(self.c2(x))
        x = torch.nn.functional.max_pool2d(self.bn(x), 2)
        return self.fc(x.flatten(1))


@pytest.mark.parametrize("graphed", [False, True])
def test_trainer_mnist_functional_one_ps_one_worker_config1(graphed, monkeypatch):
    """BASELINE configs[0] (the reference's own CPU-runnable case, here on the device: there is no CPU path): MNIST
    functional model, 1 PS + 1 worker, SGD 0.01, batch 64, uniform[0,1) images, seed 0.  Dense parameters only:
    init handshake (the worker's initial values become the PS's, server.go:209-221), one version per minibatch, and
    PS training == local torch SGD on the same data -- eagerly and as one CUDA graph per minibatch."""
    import types

    from elasticdl_b200.ps import PSGroup
    from elasticdl_b200.worker.ps_client import PSClient
    from elasticdl_b200.worker.ps_trainer import ParameterServerTrainer

    # the model and its local twin must compute bit-identical gradients from identical parameters (this short run at
    # the config's lr is numerically touchy: TF32 / atomically-accumulated conv gradients drift apart by 1e-3 in 4 steps)
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cudnn, "deterministic", True)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    torch.manual_seed(0)
    model = MnistFunctional().cuda()
    twin = MnistFunctional().cuda()
    twin.load_state_dict(model.state_dict())
    n_params = sum(p.numel() for p in model.parameters())
    assert n_params == 32 * 9 + 32 + 64 * 32 * 9 + 64 + 2 * 64 + 9216 * 10 + 10  # ~111 K fp32 (SURVEY 8d item 1)
    group = PSGroup(1, "SGD", "learning_rate=0.01;momentum=0.0;nesterov=false;", device=0)
    client = PSClient(group)
    client.dense_output = "torch"
    trainer = ParameterServerTrainer(model, client, args=types.SimpleNamespace(
        get_model_steps=1, cuda_graph=graphed, cuda_graph_warmup=2))
    gen = torch.Generator().manual_seed(0)
    for step in range(6):
        image = torch.rand(64, 28, 28, generator=gen).cuda()
        label = torch.randint(0, 10, (64,), generator=gen).cuda()
        accepted, version, loss = trainer.train_minibatch(image, label)
        assert accepted and version == step + 1
        twin.optimizer.zero_grad()
        l2 = twin.loss(label, twin(image))
        l2.backward()
        # SGD with the PS kernel's rounding (kernel_api.cc:6-14: p - round(lr * g)); torch.optim.SGD fuses the
        # multiply-add, and that last-bit difference grows ~10x per step in this run (1 ulp after the first step, 2e-3 in
        # c2.weight after the fifth on an H100)
        with torch.no_grad():
            for p in twin.parameters():
                p.sub_(p.grad * 0.01)
        assert abs(float(loss) - float(l2)) < 5e-3 * max(1.0, abs(float(l2))), (step, float(loss), float(l2))
    if graphed:
        assert isinstance(trainer._graph_state, dict), trainer.graph_fallback_reason
    params, _ = client.pull_dense_parameters([0], [-1])
    want = dict(twin.named_parameters())
    assert set(params) == set(want)
    for name, v in params.items():
        assert torch.allclose(v.reshape(want[name].shape), want[name].detach(), rtol=5e-2, atol=1e-3), name
    snap = group.snapshot()
    assert snap[0][0] == 6 and snap[0][2]  # version 6, initialised
    group.close()
