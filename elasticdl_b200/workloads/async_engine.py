"""What the fixed-model engines (census, frappe) share: one async worker of a model whose step is a fixed set of
launches over a flat dense buffer, pushed to the parameter server without model versions, and replayable as one
CUDA graph over static inputs."""
import torch

from elasticdl_b200._lib import check


def check_tensor(t, name, dtype, shape, device):
    """ValueError unless `t` is a contiguous `dtype` tensor of `shape` on `device`."""
    if not (isinstance(t, torch.Tensor) and t.device == device and t.dtype == dtype and tuple(t.shape) == shape
            and t.is_contiguous()):
        got = (tuple(t.shape), t.dtype, t.device) if isinstance(t, torch.Tensor) else type(t)
        raise ValueError("%s must be a contiguous %s tensor of shape %s on %s, not %s"
                         % (name, dtype, shape, device, got))


def truncated_normal(shape, std, gen, device):
    """TF's truncated_normal initializer: a normal of stddev `std`, every draw outside two stddevs redrawn (not
    rescaled).  `gen` is a torch.Generator on `device`."""
    x = torch.randn(shape, generator=gen, device=device)
    while True:
        bad = x.abs() > 2
        if not bool(bad.any()):
            return x * std
        x[bad] = torch.randn(int(bad.sum()), generator=gen, device=device)


class AsyncEngine:
    """The part of one async worker on the parameter-server step that the census and frappe engines share.

    group: an async PSGroup without lr staleness modulation (ValueError otherwise: the captured step carries no
    pulled versions; the drop-in ParameterServerTrainer covers those modes).  register=False attaches to a
    group.clone_view(), for another worker thread.

    A subclass sets `inputs`, its step's inputs as [(name, dtype, shape)], `tower` (whose `loss` the step leaves),
    `push_dense_segs` and `push_rows_segs`, and defines _step(*inputs), which ends in _push()."""

    def __init__(self, group, batch, lr, register, lr_schedule=None):
        self._check_group(group)
        self.B = int(batch)
        if self.B < 1:
            raise ValueError("batch size must be >= 1, not %d" % self.B)
        self.group = group if register else group.clone_view()
        self.device = self.group.device
        self.lr = float(lr)
        self.zero_versions = [0] * self.group.n_shards
        self.graph = None
        self._graph_lr = None
        self.steps = 0
        self.lr_schedule = None
        if lr_schedule is not None:
            self.set_lr_schedule(lr_schedule)

    def _check_group(self, group):
        """ValueError for a group the engine cannot push to."""
        name = type(self).__name__
        if not getattr(group, "use_async", True):
            raise ValueError("%s trains async only: a sync-SGD group needs the drop-in trainer" % name)
        if getattr(group, "lr_staleness_modulation", False):
            raise ValueError("%s pushes without model versions: a group with lr_staleness_modulation needs the "
                             "drop-in trainer" % name)

    def _check_batch(self, *tensors):
        """Check a batch, one tensor per declared input, against the declaration."""
        if len(tensors) != len(self.inputs):
            raise TypeError("a batch is %d tensors (%s), not %d"
                            % (len(self.inputs), ", ".join(n for n, _, _ in self.inputs), len(tensors)))
        for t, (name, dtype, shape) in zip(tensors, self.inputs):
            check_tensor(t, name, dtype, shape, self.device)

    def step(self, *inputs):
        """One training step on a batch, one tensor per declared input; returns the loss (device scalar, not
        synchronised)."""
        self._check_batch(*inputs)
        out = self._step(*inputs)
        self.steps += 1
        return out

    def _push(self, st):
        """push_begin -> push_dense -> push_rows -> push_end on stream `st`, with no host read."""
        g, lib = self.group, self.group.lib
        g.push_begin(self.lr, self.zero_versions)
        arr, n = self.push_dense_segs
        check(lib.b200ps_push_dense(g._h, arr, n, st))
        arr, n = self.push_rows_segs
        check(lib.b200ps_push_rows(g._h, arr, n, st))
        g.push_end(sync=False)

    def set_lr(self, lr):
        """The learning rate the next pushes carry (the reference's schedule callback sets it per version);
        the captured graph is re-captured on the next replay.  ValueError while a schedule is installed."""
        if self.lr_schedule is not None:
            raise ValueError("the learning rate comes from the installed schedule: set_lr_schedule(None) first")
        self.lr = float(lr)

    def set_lr_schedule(self, schedule):
        """Evaluate `schedule` (an elasticdl_b200.callbacks.LearningRateSchedule) on the device at every push, in
        place of `lr`, from the shard versions the push begins on; None goes back to `lr`.  The captured graph is
        re-captured on the next replay, and then replays the schedule with no re-capture."""
        self.group.set_lr_schedule(schedule)
        self.lr_schedule = schedule

    def _graph_key(self):
        return self.lr if self.lr_schedule is None else self.lr_schedule.key()

    def capture(self):
        """Capture one step over static inputs (self.statics, one per declared input) into a CUDA graph on the
        current stream's device; the learning rate, or the schedule, is baked in."""
        if self.graph is None:
            self.statics = [torch.zeros(shape, dtype=dtype, device=self.device) for _, dtype, shape in self.inputs]
        torch.cuda.current_stream(self.device).synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._step(*self.statics)
        self.graph, self._graph_lr = graph, self._graph_key()
        return graph

    def replay(self, *inputs):
        """step() through the captured graph (captured now if there is none or the learning rate or the schedule
        changed)."""
        self._check_batch(*inputs)
        if self.graph is None or self._graph_lr != self._graph_key():
            self.capture()
        for s, t in zip(self.statics, inputs):
            s.copy_(t)
        self.graph.replay()
        self.steps += 1
        return self.tower.loss.reshape(())
