"""CPU referee for the Acrobot-v1 and MountainCar-v0 tests (test infrastructure, imported by tests/test_discrete_host.py
and tests/test_gpu_discrete.py only).

gymnasium's classic_control acrobot.py ("book" dynamics, no torque noise) and mountain_car.py from their published
equations, in Python float64 and in the operation order DESIGN.md 3.5 writes down (Python evaluates products left to
right; ``x**2`` is ``x * x``).  Whole episodes are played through ``oracle.oracle.forward``.  gym itself is not a
dependency.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List

import numpy as np

from oracle import oracle as O

ACROBOT_MAX_STEPS, MOUNTAINCAR_MAX_STEPS = 500, 200
PI = math.pi
MAX_VEL_1, MAX_VEL_2 = 4 * PI, 9 * PI
_M1 = _M2 = _L1 = 1.0
_LC1 = _LC2 = 0.5
_I1 = _I2 = 1.0
_G = 9.8
_DT = 0.2
WRAP_MAX_TURNS = 4096                    # the kernel's bound on gym's wrap() loops (never reached from a reset)


def acrobot_dsdt(s, a, book=True):
    """acrobot.py ``_dsdt``: (dtheta1, dtheta2, ddtheta1, ddtheta2) of the state ``s`` (float64 [..., 4]) under torque
    ``a``.  ``book=False`` is gym's "nips" variant (no ``m2 * l1 * lc2 * dtheta1**2 * sin(theta2)`` term), a wrong
    referee for the tests."""
    m1, m2, l1, lc1, lc2, I1, I2, g = _M1, _M2, _L1, _LC1, _LC2, _I1, _I2, _G
    s = np.asarray(s, dtype=np.float64)
    theta1, theta2, dtheta1, dtheta2 = s[..., 0], s[..., 1], s[..., 2], s[..., 3]
    d1 = m1 * (lc1 * lc1) + m2 * (l1 * l1 + lc2 * lc2 + 2 * l1 * lc2 * np.cos(theta2)) + I1 + I2
    d2 = m2 * (lc2 * lc2 + l1 * lc2 * np.cos(theta2)) + I2
    phi2 = m2 * lc2 * g * np.cos(theta1 + theta2 - PI / 2.0)
    phi1 = (-m2 * l1 * lc2 * (dtheta2 * dtheta2) * np.sin(theta2)
            - 2 * m2 * l1 * lc2 * dtheta2 * dtheta1 * np.sin(theta2)
            + (m1 * lc1 + m2 * l1) * g * np.cos(theta1 - PI / 2) + phi2)
    if book:
        ddtheta2 = (a + d2 / d1 * phi1 - m2 * l1 * lc2 * (dtheta1 * dtheta1) * np.sin(theta2) - phi2) / (
            m2 * (lc2 * lc2) + I2 - (d2 * d2) / d1)
    else:
        ddtheta2 = (a + d2 / d1 * phi1 - phi2) / (m2 * (lc2 * lc2) + I2 - (d2 * d2) / d1)
    ddtheta1 = -(d2 * ddtheta2 + phi1) / d1
    return np.stack(np.broadcast_arrays(dtheta1, dtheta2, ddtheta1, ddtheta2), axis=-1)


def _wrap(x, m, M):
    diff = M - m
    x = np.array(x, dtype=np.float64)
    for _ in range(WRAP_MAX_TURNS):
        if not (x > M).any():
            break
        x = np.where(x > M, x - diff, x)
    for _ in range(WRAP_MAX_TURNS):
        if not (x < m).any():
            break
        x = np.where(x < m, x + diff, x)
    return x


def _bound(x, m, M):
    """min(max(x, m), M), NaN passing through as Python's min / max pass it."""
    x = np.where(m > x, m, x)
    return np.where(M < x, M, x)


def acrobot_terminal_value(s):
    """``-cos(theta1) - cos(theta2 + theta1)``: done when it exceeds 1.0."""
    s = np.asarray(s, dtype=np.float64)
    return -np.cos(s[..., 0]) - np.cos(s[..., 1] + s[..., 0])


def acrobot_step(state, action, book=True, torque_offset=0):
    """One Acrobot-v1 step of float64 [..., 4] states under int actions: returns (new states, rewards, done, the states
    before the wrap and the clamps).  ``torque_offset`` shifts the torque index modulo 3 (a wrong referee for the
    tests)."""
    torque = np.array([-1.0, 0.0, 1.0])[(np.asarray(action, dtype=np.int64) + torque_offset) % 3]
    y0 = np.asarray(state, dtype=np.float64)
    dt = _DT - 0.0
    dt2 = dt / 2.0
    k1 = acrobot_dsdt(y0, torque, book)
    k2 = acrobot_dsdt(y0 + dt2 * k1, torque, book)
    k3 = acrobot_dsdt(y0 + dt2 * k2, torque, book)
    k4 = acrobot_dsdt(y0 + dt * k3, torque, book)
    raw = y0 + dt / 6.0 * (k1 + 2 * k2 + 2 * k3 + k4)
    ns = np.stack([_wrap(raw[..., 0], -PI, PI), _wrap(raw[..., 1], -PI, PI), _bound(raw[..., 2], -MAX_VEL_1, MAX_VEL_1),
                   _bound(raw[..., 3], -MAX_VEL_2, MAX_VEL_2)], axis=-1)
    done = acrobot_terminal_value(ns) > 1.0
    reward = np.where(done, 0.0, -1.0)
    if ns.ndim == 1:
        return ns, float(reward), bool(done), raw
    return ns, reward, done, raw


def acrobot_obs(state):
    s = np.asarray(state, dtype=np.float64)
    return np.stack([np.cos(s[..., 0]), np.sin(s[..., 0]), np.cos(s[..., 1]), np.sin(s[..., 1]), s[..., 2], s[..., 3]],
                    axis=-1).astype(np.float32)


def acrobot_margin(state, raw):
    """Smallest distance of a visited quantity to a threshold it is compared against: the termination line, the wrap
    bounds +-pi (before wrapping), the speed bounds (before clamping)."""
    raw = np.asarray(raw)
    return np.min(np.stack([np.abs(acrobot_terminal_value(state) - 1.0), np.abs(np.abs(raw[..., 0]) - PI),
                            np.abs(np.abs(raw[..., 1]) - PI), np.abs(np.abs(raw[..., 2]) - MAX_VEL_1),
                            np.abs(np.abs(raw[..., 3]) - MAX_VEL_2)]), axis=0)


def mountaincar_step(state, action):
    """One MountainCar-v0 step: returns (new_state float64 [2], reward, done, margin) -- ``margin`` the smallest distance
    of this step's compared quantities (speed before the clip, position before the clip, the goal test) to their
    thresholds."""
    position, velocity = float(state[0]), float(state[1])
    velocity = velocity + ((int(action) - 1) * 0.001 + math.cos(3 * position) * (-0.0025))
    margin = abs(abs(velocity) - 0.07)
    velocity = min(max(velocity, -0.07), 0.07)
    position = position + velocity
    margin = min(margin, abs(position + 1.2), abs(position - 0.6), abs(position - 0.5))
    position = min(max(position, -1.2), 0.6)
    if position == -1.2 and velocity < 0:
        velocity = 0.0
    if position >= 0.5 - 1e-9:
        margin = min(margin, abs(velocity))
    done = position >= 0.5 and velocity >= 0
    return np.array([position, velocity], dtype=np.float64), -1.0, bool(done), margin


@dataclass
class Episode:
    length: int
    ret: float                       # float64 sum of the rewards in step order
    final_state: np.ndarray          # float64, the state after the last step
    min_logit_gap: float             # smallest gap between the largest and the second-largest logit over the decisions
    min_threshold_margin: float      # smallest distance of a visited quantity to a termination / wrap / clip threshold
    actions: List[int] = field(default_factory=list)


def _logit_gap(logits):
    top = np.sort(logits.astype(np.float64))[::-1]
    return float(top[0] - top[1]) if len(top) > 1 else math.inf


def episode(task: str, net: O.Net, theta: np.ndarray, init_state, max_steps: int) -> Episode:
    """One episode of the weights ``theta`` on ``task`` ('acrobot' | 'mountaincar'): observation -> ``oracle.forward`` ->
    argmax (first maximum, first NaN) -> step, until done or ``max_steps`` steps."""
    state = np.asarray(init_state, dtype=np.float64).copy()
    gap, margin, acts, ret, length = math.inf, math.inf, [], 0.0, 0
    while True:
        obs = acrobot_obs(state) if task == "acrobot" else np.array(state, dtype=np.float32)
        logits, _ = O.forward(net, theta, obs[None, :])
        a = int(np.argmax(logits[0]))
        gap = min(gap, _logit_gap(logits[0]))
        acts.append(a)
        if task == "acrobot":
            state, r, done, raw = acrobot_step(state, a)
            margin = min(margin, float(acrobot_margin(state, raw)))
        else:
            state, r, done, mg = mountaincar_step(state, a)
            margin = min(margin, mg)
        ret += r
        length += 1
        if done or length >= max_steps:
            break
    return Episode(length, ret, state, gap, margin, acts)
