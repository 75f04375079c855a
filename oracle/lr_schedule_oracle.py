"""Float64 oracle of the learning-rate schedules the push evaluates on the device (tf.keras.optimizers.schedules
of TF 2.5, the version the reference pins), the version they are evaluated at, and the server.go:178-187 rule
that applies their value.  Restated from the formulas, independently of elasticdl_b200/callbacks.py."""
import math

import numpy as np


def piecewise_constant(x, boundaries, values):
    i = 0
    while i < len(boundaries) and x > boundaries[i]:
        i += 1
    return float(np.float32(values[i]))


def exponential(x, initial, decay_steps, decay_rate, staircase=False):
    p = x / decay_steps
    if staircase:
        p = math.floor(p)
    return initial * decay_rate ** p


def inverse_time(x, initial, decay_steps, decay_rate, staircase=False):
    p = x / decay_steps
    if staircase:
        p = math.floor(p)
    return initial / (1.0 + decay_rate * p)


def polynomial(x, initial, decay_steps, end=1e-4, power=1.0, cycle=False):
    if cycle:
        d = decay_steps * max(1.0, math.ceil(x / decay_steps))
        s = x
    else:
        d = decay_steps
        s = min(x, decay_steps)
    return (initial - end) * (1.0 - s / d) ** power + end


def schedule_argument(versions):
    """The x a push evaluates its schedule at: the largest shard version it begins on, minus 1, clamped at 0."""
    return float(max(max(versions) - 1, 0))


def acceptable_f32(v):
    """The float32 values a device evaluation of the float64 value `v` may round to: the nearest one, and its
    neighbour across the rounding midpoint when `v` lies within 2^-40 (relative) of that midpoint (the device's
    pow and the host's may differ in the last bits of the double)."""
    f = np.float32(v)
    out = {float(f)}
    if v == 0.0 or not math.isfinite(v):
        return out
    up = np.nextafter(f, np.float32(np.inf))
    down = np.nextafter(f, np.float32(-np.inf))
    for n in (up, down):
        mid = (float(f) + float(n)) / 2.0
        if abs(v - mid) <= abs(v) * 2.0 ** -40:
            out.add(float(n))
    return out


def effective_lr(scheduled, opt_lr, staleness=1):
    """server.go:178-187 in float32: 1 / staleness when the push is stale, times the scheduled value, or times the
    optimizer's lr when that value is <= 0."""
    lr = np.float32(1.0)
    if staleness > 1:
        lr = np.float32(lr / np.float32(staleness))
    s = np.float32(scheduled)
    return float(np.float32(lr * (s if s > 0 else np.float32(opt_lr))))
