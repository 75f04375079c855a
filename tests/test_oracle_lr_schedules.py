"""The learning-rate schedules without a GPU: the float64 oracle at hand-computed points and edges, the model zoo's
schedules as declarative schedules against the zoo's literal callables, callbacks.py's host evaluation against the
oracle, and the refusals that come before any device work."""
import math

import numpy as np
import pytest

from elasticdl_b200 import callbacks as cb
from elasticdl_b200.workloads import census, frappe
from oracle import lr_schedule_oracle as orc


def test_piecewise_oracle_edges():
    b, v = [10, 20], [1.0, 0.5, 0.25]
    assert orc.piecewise_constant(0, b, v) == 1.0
    assert orc.piecewise_constant(10, b, v) == 1.0  # x <= b0
    assert orc.piecewise_constant(11, b, v) == 0.5
    assert orc.piecewise_constant(20, b, v) == 0.5
    assert orc.piecewise_constant(21, b, v) == 0.25
    assert orc.piecewise_constant(5, [], [0.3]) == float(np.float32(0.3))


def test_decay_oracles_by_hand():
    assert orc.exponential(0, 0.1, 10, 0.5) == 0.1
    assert orc.exponential(10, 0.1, 10, 0.5) == pytest.approx(0.05, rel=1e-15)
    assert orc.exponential(5, 0.1, 10, 0.25) == pytest.approx(0.05, rel=1e-15)
    assert orc.exponential(19, 0.1, 10, 0.5, staircase=True) == pytest.approx(0.05, rel=1e-15)
    assert orc.exponential(20, 0.1, 10, 0.5, staircase=True) == pytest.approx(0.025, rel=1e-15)
    assert orc.inverse_time(0, 0.1, 10, 1.0) == 0.1
    assert orc.inverse_time(10, 0.1, 10, 1.0) == pytest.approx(0.05, rel=1e-15)
    assert orc.inverse_time(15, 0.1, 10, 1.0, staircase=True) == pytest.approx(0.05, rel=1e-15)
    assert orc.polynomial(0, 0.1, 10, end=0.0) == 0.1
    assert orc.polynomial(5, 0.1, 10, end=0.0) == pytest.approx(0.05, rel=1e-15)
    assert orc.polynomial(10, 0.1, 10, end=0.01) == pytest.approx(0.01, rel=1e-15)
    assert orc.polynomial(25, 0.1, 10, end=0.01) == pytest.approx(0.01, rel=1e-15)  # held past decay_steps
    assert orc.polynomial(5, 0.1, 10, end=0.0, power=2.0) == pytest.approx(0.025, rel=1e-15)


def test_polynomial_cycle_oracle():
    # cycle: D = decay_steps * max(1, ceil(x / decay_steps)); at x = 0 the multiplier is 1, at a multiple k of
    # decay_steps the cycle has just ended (s / D = 1), one step later a new cycle of length (k + 1) begins
    assert orc.polynomial(0, 0.1, 10, end=0.0, cycle=True) == 0.1
    assert orc.polynomial(10, 0.1, 10, end=0.0, cycle=True) == 0.0
    assert orc.polynomial(20, 0.1, 10, end=0.0, cycle=True) == 0.0
    assert orc.polynomial(11, 0.1, 10, end=0.0, cycle=True) == pytest.approx(0.1 * (1 - 11 / 20), rel=1e-15)
    assert orc.polynomial(15, 0.1, 10, end=0.0, cycle=True) == pytest.approx(0.025, rel=1e-15)


def test_version_rule_and_fallback_oracle():
    assert orc.schedule_argument([0]) == 0.0
    assert orc.schedule_argument([0, 0, 0]) == 0.0
    assert orc.schedule_argument([1]) == 0.0
    assert orc.schedule_argument([5, 9, 7]) == 8.0
    assert orc.effective_lr(0.25, 0.1) == 0.25
    assert orc.effective_lr(0.0, 0.1) == float(np.float32(0.1))
    assert orc.effective_lr(-1.0, 0.1) == float(np.float32(0.1))
    assert orc.effective_lr(0.25, 0.1, staleness=4) == 0.0625


def test_acceptable_f32_window():
    one = np.float32(1.0)
    mid = (1.0 + float(np.nextafter(one, np.float32(2)))) / 2.0
    assert orc.acceptable_f32(0.5) == {0.5}
    assert len(orc.acceptable_f32(mid * (1 + 2.0 ** -45))) == 2
    assert len(orc.acceptable_f32(mid * (1 + 2.0 ** -30))) == 1


def _census_zoo(model_version):  # model_zoo/census_wide_deep_model/wide_deep_functional_api.py:74-83
    if model_version < 5000:
        return 0.0003
    elif model_version < 12000:
        return 0.0002
    else:
        return 0.0001


def _frappe_zoo(model_version):  # model_zoo/deepfm_functional_api/deepfm_functional_api.py:140-145
    return 0.5 if model_version < 100 else 0.2


@pytest.mark.parametrize("module,zoo", [(census, _census_zoo), (frappe, _frappe_zoo)])
def test_workload_schedules_equal_the_zoo_callables(module, zoo):
    (scheduler,) = module.callbacks()
    assert isinstance(scheduler, cb.LearningRateScheduler)
    sched = scheduler.schedule
    assert isinstance(sched, cb.PiecewiseConstantDecay)
    for v in range(0, 20001):
        assert sched(v) == float(np.float32(zoo(v))), v
    # the reference calls the callable with -1 first; a declarative schedule is clamped at 0
    assert sched(-1) == sched(0) == float(np.float32(zoo(0)))


SCHEDULES = [
    (cb.PiecewiseConstantDecay([3, 7.5, 100], [0.1, 0.05, 0.02, 0.001]),
     lambda x: orc.piecewise_constant(x, [3, 7.5, 100], [0.1, 0.05, 0.02, 0.001])),
    (cb.ExponentialDecay(0.1, 7, 0.9), lambda x: orc.exponential(x, 0.1, 7, 0.9)),
    (cb.ExponentialDecay(0.3, 4, 0.5, staircase=True), lambda x: orc.exponential(x, 0.3, 4, 0.5, True)),
    (cb.InverseTimeDecay(0.2, 3, 0.7), lambda x: orc.inverse_time(x, 0.2, 3, 0.7)),
    (cb.InverseTimeDecay(0.2, 3, 0.7, staircase=True), lambda x: orc.inverse_time(x, 0.2, 3, 0.7, True)),
    (cb.PolynomialDecay(0.1, 9), lambda x: orc.polynomial(x, 0.1, 9)),
    (cb.PolynomialDecay(0.1, 5, 0.01, power=0.5, cycle=True), lambda x: orc.polynomial(x, 0.1, 5, 0.01, 0.5, True)),
]


@pytest.mark.parametrize("i", range(len(SCHEDULES)))
def test_host_call_matches_oracle(i):
    sched, ref = SCHEDULES[i]
    for v in range(-1, 60):
        assert sched(v) == pytest.approx(ref(max(v, 0)), rel=1e-15, abs=0), v


@pytest.mark.parametrize("i", range(len(SCHEDULES)))
def test_struct_carries_the_parameters(i):
    sched, _ = SCHEDULES[i]
    s = sched.struct()
    assert s.kind in (1, 2, 3, 4)
    assert sched.key() == bytes(s)
    if isinstance(sched, cb.PiecewiseConstantDecay):
        assert list(s.boundaries[:s.n_boundaries]) == sched.boundaries
        assert list(s.values[:s.n_boundaries + 1]) == sched.values
    else:
        assert s.decay_steps == sched.decay_steps and s.initial_learning_rate == sched.initial_learning_rate


@pytest.mark.parametrize("make", [
    lambda: cb.PiecewiseConstantDecay([1, 2], [0.1, 0.2]),  # len(values) != len(boundaries) + 1
    lambda: cb.PiecewiseConstantDecay([2, 1], [0.1, 0.2, 0.3]),  # not increasing
    lambda: cb.PiecewiseConstantDecay([1, 1], [0.1, 0.2, 0.3]),  # not strictly increasing
    lambda: cb.PiecewiseConstantDecay(list(range(33)), [0.1] * 34),  # more than 32 boundaries
    lambda: cb.PiecewiseConstantDecay([1], [0.1, math.nan]),
    lambda: cb.PiecewiseConstantDecay([math.inf], [0.1, 0.2]),
    lambda: cb.ExponentialDecay(0.1, 0, 0.5),
    lambda: cb.ExponentialDecay(0.1, -3, 0.5),
    lambda: cb.ExponentialDecay(math.nan, 3, 0.5),
    lambda: cb.InverseTimeDecay(0.1, 3, math.inf),
    lambda: cb.PolynomialDecay(0.1, 0),
    lambda: cb.PolynomialDecay(0.1, 10, power=math.nan),
])
def test_schedule_refusals(make):
    with pytest.raises(ValueError):
        make()


class _Model:
    pass


class _Opt:
    def __init__(self, lr):
        self.param_groups = [{"lr": lr}, {"lr": lr}]


def test_scheduler_raises_as_the_reference():  # elasticdl/python/tests/callbacks_test.py:93-107
    s = cb.LearningRateScheduler(lambda v: 1 if v < 2 else 2)
    model = _Model()
    model.optimizer = None
    s.set_model(model)
    with pytest.raises(ValueError, match="lr"):
        s.on_train_batch_begin(1)
    model.optimizer = _Opt(0.1)
    with pytest.raises(ValueError, match="float"):
        s.on_train_batch_begin(1)


def test_scheduler_sets_every_param_group():  # callbacks_test.py:109-116
    s = cb.LearningRateScheduler(lambda v: 0.2 if v < 2 else 0.1)
    model = _Model()
    model.optimizer = _Opt(0.3)
    s.set_model(model)
    s.on_train_batch_begin(1)
    assert [g["lr"] for g in model.optimizer.param_groups] == [0.2, 0.2]
    s.on_train_batch_begin(2)
    assert [g["lr"] for g in model.optimizer.param_groups] == [0.1, 0.1]
    s = cb.LearningRateScheduler(cb.ExponentialDecay(0.1, 2, 0.5))
    s.set_model(model)
    s.on_train_batch_begin(-1)
    assert model.optimizer.param_groups[0]["lr"] == 0.1
    s.on_train_batch_begin(4)
    assert model.optimizer.param_groups[0]["lr"] == pytest.approx(0.025, rel=1e-15)


def test_device_schedule_picks_the_declarative_one():
    d = cb.ExponentialDecay(0.1, 2, 0.5)
    assert cb.device_schedule(None) is None
    assert cb.device_schedule([cb.LearningRateScheduler(lambda v: 0.1)]) is None
    assert cb.device_schedule([cb.Callback(), cb.LearningRateScheduler(d)]) is d
