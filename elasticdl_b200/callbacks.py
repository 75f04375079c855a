"""Training callbacks (elasticdl/python/elasticdl/callbacks.py) over torch: LearningRateScheduler, and the four
declarative learning-rate schedules of tf.keras.optimizers.schedules (TF 2.5) that the parameter server can
evaluate on the device instead (b200ps_set_lr_schedule, include/b200ps.h).

A schedule's argument is a model version.  The reference's worker calls its schedule with the version its previous
minibatch pulled (-1 before the first); the device evaluates a declarative schedule at max_s(version_s) - 1 of the
shard versions the push begins on, clamped at 0.  With one worker the two are the same version; __call__ clamps
at 0 too, so the host and the device agree.  The host value is float64, the device's is the float64 value rounded
once to float32 (Keras evaluates in float32, which can differ in the last bits).
"""
import math

import numpy as np
import torch

from elasticdl_b200 import _lib


class LearningRateSchedule:
    """A declarative schedule: __call__(model_version) on the host, struct() for the device."""

    def __call__(self, model_version):
        return self._at(max(float(model_version), 0.0))

    def key(self):
        """Bytes that identify the schedule (two schedules with one key compute the same lr)."""
        return bytes(self.struct())

    @staticmethod
    def _finite(name, *xs):
        for x in xs:
            if not math.isfinite(float(x)):
                raise ValueError("%s must be finite, not %r" % (name, x))

    def _decay(self, initial_learning_rate, decay_steps, *others):
        self._finite("the schedule's parameters", initial_learning_rate, decay_steps, *others)
        if not float(decay_steps) > 0:
            raise ValueError("decay_steps must be > 0, not %r" % (decay_steps,))
        self.initial_learning_rate, self.decay_steps = float(initial_learning_rate), float(decay_steps)


class PiecewiseConstantDecay(LearningRateSchedule):
    """values[0] for x <= boundaries[0], values[i] for boundaries[i-1] < x <= boundaries[i], values[-1] past the
    last boundary.  At most 32 strictly increasing boundaries; values are float32 and returned exactly."""

    def __init__(self, boundaries, values):
        if len(boundaries) != len(values) - 1:
            raise ValueError("The length of boundaries should be 1 less than the length of values")
        if len(boundaries) > _lib.LR_MAX_BOUNDARIES:
            raise ValueError("at most %d boundaries, not %d" % (_lib.LR_MAX_BOUNDARIES, len(boundaries)))
        self._finite("boundaries and values", *boundaries, *values)
        if any(not float(b) > float(a) for a, b in zip(boundaries, boundaries[1:])):
            raise ValueError("boundaries must be strictly increasing: %r" % (list(boundaries),))
        self.boundaries = [float(b) for b in boundaries]
        self.values = [float(np.float32(v)) for v in values]

    def _at(self, x):
        for b, v in zip(self.boundaries, self.values):
            if x <= b:
                return v
        return self.values[-1]

    def struct(self):
        s = _lib.LrSchedule(kind=_lib.LR_PIECEWISE, n_boundaries=len(self.boundaries))
        s.boundaries[:len(self.boundaries)] = self.boundaries
        s.values[:len(self.values)] = self.values
        return s


class ExponentialDecay(LearningRateSchedule):
    """initial_learning_rate * decay_rate ^ (x / decay_steps), the exponent floored if staircase."""

    def __init__(self, initial_learning_rate, decay_steps, decay_rate, staircase=False):
        self._decay(initial_learning_rate, decay_steps, decay_rate)
        self.decay_rate, self.staircase = float(decay_rate), bool(staircase)

    def _p(self, x):
        p = x / self.decay_steps
        return math.floor(p) if self.staircase else p

    def _at(self, x):
        return self.initial_learning_rate * math.pow(self.decay_rate, self._p(x))

    def struct(self):
        return _lib.LrSchedule(kind=_lib.LR_EXPONENTIAL, staircase=int(self.staircase),
                               initial_learning_rate=self.initial_learning_rate, decay_steps=self.decay_steps,
                               decay_rate=self.decay_rate)


class InverseTimeDecay(ExponentialDecay):
    """initial_learning_rate / (1 + decay_rate * x / decay_steps), x / decay_steps floored if staircase."""

    def _at(self, x):
        return self.initial_learning_rate / (1.0 + self.decay_rate * self._p(x))

    def struct(self):
        s = super().struct()
        s.kind = _lib.LR_INVERSE_TIME
        return s


class PolynomialDecay(LearningRateSchedule):
    """(initial_learning_rate - end_learning_rate) * (1 - s / D) ^ power + end_learning_rate with s = min(x,
    decay_steps) and D = decay_steps, or with cycle s = x and D = decay_steps * max(1, ceil(x / decay_steps))."""

    def __init__(self, initial_learning_rate, decay_steps, end_learning_rate=0.0001, power=1.0, cycle=False):
        self._decay(initial_learning_rate, decay_steps, end_learning_rate, power)
        self.end_learning_rate, self.power, self.cycle = float(end_learning_rate), float(power), bool(cycle)

    def _at(self, x):
        if self.cycle:
            s, d = x, self.decay_steps * max(1.0, math.ceil(x / self.decay_steps))
        else:
            s, d = min(x, self.decay_steps), self.decay_steps
        return (self.initial_learning_rate - self.end_learning_rate) * math.pow(1.0 - s / d, self.power) \
            + self.end_learning_rate

    def struct(self):
        return _lib.LrSchedule(kind=_lib.LR_POLYNOMIAL, cycle=int(self.cycle),
                               initial_learning_rate=self.initial_learning_rate, decay_steps=self.decay_steps,
                               end_learning_rate=self.end_learning_rate, power=self.power)


class Callback:
    """The part of tf.keras.callbacks.Callback the worker drives: the model it trains and the batch hook."""

    model = None
    params = None

    def set_model(self, model):
        self.model = model

    def set_params(self, params):
        self.params = params

    def on_train_batch_begin(self, batch, logs=None):
        pass


class LearningRateScheduler(Callback):
    """Sets the learning rate of the model's optimizer from `schedule(model_version)` before every minibatch
    (callbacks.py:69-109; the worker passes the model version, worker.py:198).  `schedule` is any callable
    returning a float, or a LearningRateSchedule, which ParameterServerTrainer.train_loop also installs on the
    parameter server so that the push evaluates it on the device."""

    def __init__(self, schedule):
        self._schedule = schedule

    @property
    def schedule(self):
        return self._schedule

    def on_train_batch_begin(self, batch, logs=None):
        opt = getattr(self.model, "optimizer", None)
        groups = getattr(opt, "param_groups", None)
        if not groups or any("lr" not in g for g in groups):
            raise ValueError('Optimizer must have a "lr" attribute.')
        lr = self._schedule(batch)
        if isinstance(lr, torch.Tensor) and lr.numel() == 1 and lr.is_floating_point():
            lr = lr.item()
        if not isinstance(lr, (float, np.float32, np.float64)):
            raise ValueError('The output of the "schedule" function should be float.')
        for g in groups:
            g["lr"] = float(lr)


def device_schedule(callbacks):
    """The declarative schedule of the LearningRateScheduler among `callbacks`, None if it has none."""
    for cb in callbacks or ():
        if isinstance(cb, LearningRateScheduler) and isinstance(cb.schedule, LearningRateSchedule):
            return cb.schedule
    return None
