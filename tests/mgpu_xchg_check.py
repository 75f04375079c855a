"""Owner-computes exchange (csrc/ps_exchange.cuh) vs the direct peer path and the oracle
(torchrun, one rank per GPU).  Checks: xchg_create refuses hashed, dense and raw tables and too many
groups; xchg_pull == pull_rows bit for bit; xchg_push (Adam) == oracle applying every rank's push on
disjoint rows; created-row counts; a DeepFM engine in exchange mode trains, one with too many groups
takes the direct path; no wait timed out."""
import ctypes
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from elasticdl_b200 import _lib  # noqa: E402
from elasticdl_b200._lib import check  # noqa: E402
from elasticdl_b200.ps import PSGroup  # noqa: E402
from oracle import ps_oracle as O  # noqa: E402

F = np.float32
ADAM = ("Adam", "learning_rate=0.001;beta_1=0.9;beta_2=0.999;epsilon=1e-07;amsgrad=false;")


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    # B200_SHARED_GPU=1: every rank is a process on cuda:0 (the shards are still separate allocations mapped
    # across PROCESSES with CUDA IPC, the kernels of the ranks time-slice the one device) and the host-side
    # plumbing runs over gloo -- NCCL refuses two ranks on one device.  Lets a 1-GPU box run this check.
    shared = os.environ.get("B200_SHARED_GPU") == "1"
    local = 0 if shared else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if shared:
        dist.init_process_group("gloo")
    else:
        dist.init_process_group("nccl", device_id=dev)
    group = PSGroup(world, *ADAM, device=local, local_shards=[rank])
    rows = [7, 3000, 400000]
    G, B, D = len(rows), 4096, 8
    deep = [group.register_table("d%d" % g, D, "zero", r) for g, r in enumerate(rows)]
    wide = [group.register_table("w%d" % g, 1, "zero", r) for g, r in enumerate(rows)]
    hashed_id = group.register_table("hashed", D, "zero", expected_rows=64)
    dense_id = group.register_dense("dense", (16, D), 0)
    raw_id = check(group.lib.b200ps_raw_register(group._h, b"raw", 64))
    group.commit()

    def create(dt, wt):
        return group.lib.b200ps_xchg_create(group._h, len(dt), B, (ctypes.c_int32 * len(dt))(*dt),
                                            (ctypes.c_int32 * len(wt))(*wt))

    # the exchange serves direct-indexed striped tables only, and at most MAX_SEGS / 2 pairs; a refused
    # create leaves no exchange behind, so the valid one below still succeeds
    kx = _lib.MAX_SEGS // 2 + 1
    for dt, wt in (([hashed_id] + deep[1:], wide), ([dense_id] + deep[1:], wide), (deep, [raw_id] + wide[1:]),
                   ((deep * kx)[:kx], (wide * kx)[:kx])):
        assert create(dt, wt) == _lib.EINVAL, (dt, wt, group.lib.b200ps_last_error())
    group.xchg_create(G, B, deep, wide)
    servers = [O.OracleServer(i, *ADAM, num_ps=world) for i in range(world)]
    oc = O.OraclePSClient(servers)
    oc.push_embedding_table_infos([O.EmbeddingTableInfo("d%d" % g, D, "zero", 1) for g in range(G)] +
                                  [O.EmbeddingTableInfo("w%d" % g, 1, "zero", 1) for g in range(G)])
    rng = np.random.RandomState(7)  # identical stream on every rank
    for g, r in enumerate(rows):
        vd, vw = rng.randn(r, D).astype(F), rng.randn(r, 1).astype(F)
        ids = np.arange(r, dtype=np.int64)
        mine = ids % world == rank
        group.set_rows([("d%d" % g, ids[mine], vd[mine]), ("w%d" % g, ids[mine], vw[mine])])
        for s in servers:
            m = ids % world == s.id
            s.tables["d%d" % g].set(ids[m], vd[m])
            s.tables["w%d" % g].set(ids[m], vw[m])
    torch.cuda.synchronize()
    dist.barrier()
    lib, h = group.lib, group._h
    f32 = dict(dtype=torch.float32, device=dev)
    bet_d, bet_w = torch.zeros((G * B, D), **f32), torch.zeros((G * B, 1), **f32)
    for rnd in range(3):
        # ---- pull: every rank asks for its own random ids --------------------------------------
        r2 = np.random.RandomState(100 * rnd + rank)
        ids = np.stack([r2.randint(0, r, size=B) for r in rows]).astype(np.int64)
        d_ids = torch.from_numpy(ids).to(dev)
        uniq, inv, n_unique = group.unique(d_ids.view(-1), G)
        bet_d.fill_(-7.0)
        bet_w.fill_(-7.0)
        check(lib.b200ps_xchg_pull(h, uniq.data_ptr(), n_unique.data_ptr(), bet_d.data_ptr(), bet_w.data_ptr(), group._stream()))
        group.check()
        nu = n_unique.cpu().numpy()
        for g in range(G):
            u = int(nu[g])
            want_d, want_w = group.pull_rows([("d%d" % g, uniq[g * B:g * B + u]), ("w%d" % g, uniq[g * B:g * B + u])])
            assert torch.equal(bet_d[g * B:g * B + u], want_d), (rnd, g, "deep rows differ from the direct pull")
            assert torch.equal(bet_w[g * B:g * B + u], want_w), (rnd, g, "wide rows differ from the direct pull")
            assert bool((bet_d[g * B + u:(g + 1) * B] == -7.0).all())  # rows beyond n_unique untouched
        dist.barrier()
        # ---- push: disjoint rows per pusher: id = q*N*N + pusher*N + owner ----------------------
        k = 1500
        pid = [(np.random.RandomState(5 * rnd + g).permutation(max(r // (world * world), 1))[:k] * world * world)
               for g, r in enumerate(rows)]
        counts = [min(k, max(r // (world * world), 1)) for r in rows]
        p_ids = torch.zeros((G, B), dtype=torch.int64, device=dev)
        p_n = torch.tensor(counts, dtype=torch.int32, device=dev)
        gs_d, gs_w = torch.zeros((G * B, D), **f32), torch.zeros((G * B, 1), **f32)
        plan = {}
        for pusher in range(world):
            rr = np.random.RandomState(1000 * rnd + pusher)
            for g in range(G):
                c = counts[g]
                owners = rr.randint(0, world, size=c)
                idg = pid[g][:c] + pusher * world + owners
                idg = idg[idg < rows[g]]
                gd, gw = rr.randn(len(idg), D).astype(F), rr.randn(len(idg), 1).astype(F)
                plan[(pusher, g)] = (idg.astype(np.int64), gd, gw)
        for g in range(G):
            idg, gd, gw = plan[(rank, g)]
            p_n[g] = len(idg)
            p_ids[g, :len(idg)] = torch.from_numpy(idg).to(dev)
            gs_d[g * B:g * B + len(idg)] = torch.from_numpy(gd).to(dev)
            gs_w[g * B:g * B + len(idg)] = torch.from_numpy(gw).to(dev)
        # a push rides on the routing of the pull before it: pull the rows about to be updated
        check(lib.b200ps_xchg_pull(h, p_ids.data_ptr(), p_n.data_ptr(), bet_d.data_ptr(), bet_w.data_ptr(), group._stream()))
        for r in range(world):  # deterministic per-shard step order: rank r's ApplyGradients is the r-th
            if r == rank:
                group.push_begin(0.001, [0] * world)
            torch.cuda.synchronize()
            dist.barrier()
        check(lib.b200ps_xchg_push(h, gs_d.data_ptr(), gs_w.data_ptr(), group._stream()))
        group.push_end(sync=True)
        group.check()
        dist.barrier()
        for pusher in range(world):
            edl = []
            for g in range(G):
                idg, gd, gw = plan[(pusher, g)]
                edl += [O.Tensor("d%d" % g, gd.copy(), idg), O.Tensor("w%d" % g, gw.copy(), idg)]
            oc.push_gradients([], edl, 0.001, [0] * world)
        for g, r in enumerate(rows):
            allids = np.arange(r, dtype=np.int64)
            gd_, gw_ = group.pull_rows([("d%d" % g, allids), ("w%d" % g, allids)])
            for name, got in (("d%d" % g, gd_), ("w%d" % g, gw_)):
                want = np.zeros(tuple(got.shape), dtype=F)
                for s in servers:
                    keys = s.tables[name].keys()
                    want[keys] = s.tables[name].get(keys)
                assert np.array_equal(got.cpu().numpy(), want), (rnd, name, "push result differs from the oracle")
        dist.barrier()
    state = group.snapshot()
    assert [s[0] for s in state] == [3 * world] * world and [s[1] for s in state] == [3 * world] * world, state
    # ---- the DeepFM engine in exchange mode trains ------------------------------------------------
    from elasticdl_b200.workloads.deepfm import DeepFMPSEngine, synthetic_batch

    g2 = PSGroup(world, *ADAM, device=local, local_shards=[rank])
    erows = [11, 5000, 60000, 9]
    eng = DeepFMPSEngine(g2, 1024, group_rows=erows)
    assert eng.exchange == "owner"
    ids, dense, labels = synthetic_batch(1024, 50 + rank, dev, "zipf", group_rows=erows)
    dist.barrier()
    l0 = float(eng.step(ids, dense, labels))
    for _ in range(30):
        l1 = float(eng.step(ids, dense, labels))
    g2.check()
    assert np.isfinite(l0) and l1 < l0, (l0, l1)
    eng.capture()
    for _ in range(5):
        l2 = float(eng.step_graph(ids, dense, labels))
    g2.check()
    assert l2 <= l1 + 1e-3
    # ---- more id groups than the exchange moves: the engine takes the direct path ------------------
    g3 = PSGroup(world, *ADAM, device=local, local_shards=[rank])
    assert DeepFMPSEngine(g3, 64, group_rows=[16] * kx).exchange == "direct"
    dist.barrier()
    if rank == 0:
        print("mgpu_xchg_check ok: world=%d exchange pull bit-exact vs direct, push bit-exact vs oracle, "
              "engine loss %.4f -> %.4f -> %.4f" % (world, l0, l1, l2))
    g3.close()
    g2.close()
    group.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
