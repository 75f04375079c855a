"""PyTorchAllReduceController / create_elastic_controller
(elasticai_api/pytorch/controller.py:41-203) over torch.distributed."""
import os
import time
import traceback

import torch
import torch.distributed as dist

from elasticdl_b200.elasticai_api.common import base_controller as bc
from elasticdl_b200.elasticai_api.common.base_controller import AllReduceController, comm_rank, comm_size
from elasticdl_b200.elasticai_api.common.data_shard_service import RecordIndexService
from elasticdl_b200.elasticai_api.common.master_client import build_master_client


def create_elastic_controller(batch_size, num_epochs=None, dataset_size=None, shuffle=False, master_client=None,
                              backend=None):
    """controller.py:41-94.  `master_client` defaults to the in-process stand-in for the
    ElasticDL master (out of scope here), see common/master_client.py."""
    master_client = master_client or build_master_client(
        batch_size=batch_size, num_epochs=num_epochs or 1, dataset_size=dataset_size or 0, shuffle=shuffle)
    record_index_service = RecordIndexService(master_client=master_client, batch_size=batch_size,
                                              num_epochs=num_epochs, dataset_size=dataset_size, shuffle=shuffle)
    controller = PyTorchAllReduceController(master_client, record_index_service, backend=backend)
    controller.init_horovod_locally()
    return controller


def _flat_broadcast(tensors, root_rank=0):
    """One coalesced broadcast per (device, dtype) instead of one per tensor."""
    groups = {}
    for t in tensors:
        groups.setdefault((t.device, t.dtype), []).append(t)
    for plist in groups.values():
        flat = torch.cat([t.detach().reshape(-1) for t in plist])
        dist.broadcast(flat, src=root_rank)
        off = 0
        with torch.no_grad():
            for t in plist:
                t.copy_(flat[off:off + t.numel()].view_as(t))
                off += t.numel()


def broadcast_parameters(state_dict, root_rank=0):
    if comm_size() > 1:
        _flat_broadcast([v for v in state_dict.values() if isinstance(v, torch.Tensor)], root_rank)


def broadcast_object(obj, root_rank=0, name=None):
    if comm_size() <= 1:
        return obj
    box = [obj]
    dist.broadcast_object_list(box, src=root_rank)
    return box[0]


def broadcast_optimizer_state(optimizer, root_rank=0):
    """Tensors of the optimizer state are broadcast flat; scalars (step counts, lr ...) as an object.
    A rank whose optimizer holds no (or less) state than the root -- an elastic joiner, or a rank whose
    warm-up call did not step -- first materialises the root's entries (the Horovod original does the
    same before broadcasting), so every rank enters the same collectives."""
    if comm_size() <= 1:
        return
    sd = optimizer.state_dict()
    layout = {pid: {k: ((tuple(v.shape), str(v.dtype).replace("torch.", "")) if isinstance(v, torch.Tensor) else None)
                    for k, v in st.items()} for pid, st in sd["state"].items()}
    meta = broadcast_object({"param_groups": sd["param_groups"], "layout": layout}, root_rank)
    if comm_rank() != root_rank:
        params = [p for g in optimizer.param_groups for p in g["params"]]
        for pid, entries in meta["layout"].items():
            st = sd["state"].setdefault(pid, {})
            dev = params[pid].device if isinstance(pid, int) and pid < len(params) else torch.device("cpu")
            for k, spec in entries.items():
                if spec is not None and not isinstance(st.get(k), torch.Tensor):
                    st[k] = torch.zeros(spec[0], dtype=getattr(torch, spec[1]), device=dev)
                elif spec is None:
                    st.setdefault(k, None)
        for pid in [q for q in sd["state"] if q not in meta["layout"]]:
            del sd["state"][pid]
    tensors, scalars = [], {}
    for pid in sorted(sd["state"], key=str):
        st = sd["state"][pid]
        for k in sorted(st, key=str):
            v = st[k]
            if isinstance(v, torch.Tensor):
                tensors.append(v)
            else:
                scalars[(pid, k)] = v
    if tensors:
        _flat_broadcast(tensors, root_rank)
    scalars = broadcast_object(scalars, root_rank)
    for (pid, k), v in scalars.items():
        if pid in sd["state"]:
            sd["state"][pid][k] = v
    for g, mg in zip(sd["param_groups"], meta["param_groups"]):
        for k, v in mg.items():
            if k != "params":
                g[k] = v
    optimizer.load_state_dict(sd)


class PyTorchAllReduceController(AllReduceController):
    def __init__(self, master_client, data_shard_service, backend=None):
        super(PyTorchAllReduceController, self).__init__(master_client, data_shard_service, backend)
        self._model = None
        self._optimizer = None
        self.backward_passes_per_step = 1
        self.global_batch_num_per_step = int(os.getenv("WORKER_NUM", 1))
        self.global_completed_batch_num = 0
        self.batch_count_per_epoch = self.data_shard_service.get_minibatch_count_per_epoch()

    def get_current_epoch(self):
        return self.global_completed_batch_num // max(self.batch_count_per_epoch, 1)

    def set_resume_epoch(self, epoch):
        self.global_completed_batch_num = epoch * self.batch_count_per_epoch

    def set_broadcast_model(self, model):
        self._model = model

    def set_broadcast_optimizer(self, optimizer):
        self._optimizer = optimizer

    def broadcast(self):  # controller.py:126-131
        broadcast_parameters(self._model.state_dict(), root_rank=0)
        broadcast_optimizer_state(self._optimizer, root_rank=0)
        self.global_completed_batch_num = broadcast_object(self.global_completed_batch_num,
                                                           name="GlobalCompletedBatchNum")

    def train_one_batch_with_retries(self, func, *args, **kwargs):  # controller.py:133-157
        self.reset_backward_passes_per_step()
        allreduce_success = False
        result = None
        for _ in range(bc.DEFAULT_MAX_ALLREDUCE_RETRY_NUM):
            try:
                self._broadcast_if_needed()
                result = func(*args, **kwargs)
                allreduce_success = True
                break
            except RuntimeError:
                # a failed collective (peer died / group rebuilt) surfaces as RuntimeError in torch
                traceback.print_exc()
                self.restore()
        if not allreduce_success:
            raise RuntimeError("Failed to perform allreduce.")
        self._update_completed_minibatches()
        return result

    def restore(self):  # controller.py:159-164
        time.sleep(bc.RETRY_ALLREDUCE_INTERVAL_SECS)
        self._optimizer.load_state_dict(self._optimizer.state_dict())
        self._optimizer.zero_grad()
        self._rendezvous_manager.init_horovod_if_needed()

    def _update_completed_minibatches(self):  # controller.py:166-176
        if getattr(self._optimizer, "fixed_global_batch_size", False):
            if self._optimizer.update_gradients:
                self.global_completed_batch_num += self.global_batch_num_per_step
        else:
            self.global_completed_batch_num += comm_size()

    def reset_backward_passes_per_step(self):  # controller.py:178-203
        if getattr(self._optimizer, "fixed_global_batch_size", False):
            world_size, rank = comm_size(), comm_rank()
            self.backward_passes_per_step = self.global_batch_num_per_step // world_size
            if rank < self.global_batch_num_per_step % world_size:
                self.backward_passes_per_step += 1
            if self.backward_passes_per_step != self._optimizer.backward_passes_per_step:
                self._optimizer.set_backward_passes_per_step(self.backward_passes_per_step)
