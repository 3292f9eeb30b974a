"""CPU referee for the Pendulum-v1 tests (test infrastructure, imported by tests/test_pendulum_host.py and
tests/test_gpu_pendulum.py only).

* gymnasium's Pendulum-v1 step (classic_control pendulum.py) from its published equations, in scalar Python float64 in
  Python's left-to-right order: ``u`` is the float32 clip of the action, ``u**2`` a float32 product, everything after it
  float64 (numpy 1.x scalar promotion).  gym itself is not a dependency.
* whole episodes of a ``MujocoPolicy`` net played through ``oracle.oracle.forward`` (float32, observation normalisation
  clip((o - mean) / std, -5, 5)), with the runner's return bookkeeping: float32 rewards summed in float64 in step order.
"""
from __future__ import annotations

import dataclasses
import math
from dataclasses import dataclass

import numpy as np

from oracle import oracle as O

MAX_STEPS = 200                          # gymnasium registers Pendulum-v1 with TimeLimit(max_episode_steps=200)
G, M, L, DT, MAX_SPEED, MAX_TORQUE = 10.0, 1.0, 1.0, 0.05, 8.0, 2.0


def angle_normalize(x: float) -> float:
    """((x + pi) % (2 pi)) - pi with Python's float modulo (the result takes the divisor's sign, as numpy's)."""
    return ((x + math.pi) % (2 * math.pi)) - math.pi


def pendulum_step(th: float, thdot: float, a) -> tuple:
    """One Pendulum-v1 step from (th, thdot) with the float32 action ``a``.  Returns (newth, newthdot, reward float64)."""
    u = np.clip(np.float32(a), np.float32(-MAX_TORQUE), np.float32(MAX_TORQUE))
    costs = angle_normalize(th) ** 2 + 0.1 * thdot ** 2 + 0.001 * float(u * u)
    newthdot = thdot + (3 * G / (2 * L) * math.sin(th) + 3.0 / (M * L ** 2) * float(u)) * DT
    newthdot = min(max(newthdot, -MAX_SPEED), MAX_SPEED)
    newth = th + newthdot * DT
    return newth, newthdot, -costs


def observation(th: float, thdot: float) -> np.ndarray:
    return np.array([math.cos(th), math.sin(th), thdot], dtype=np.float32)


def policy_net(hidden=(64, 64)) -> O.Net:
    """The MujocoPolicy 'continuous:' net on Pendulum: 3 -> hidden (tanh) -> 1, observation normalisation."""
    return O.make_net("MujocoPolicy", ob_dim=3, hidden=tuple(hidden), ac_dim=1)


@dataclass
class Episode:
    th: float
    thdot: float
    ret: np.float32                  # float32 rewards summed in float64, rounded once
    signret: np.float32
    ob_sum: np.ndarray               # float64 [3] of the observations fed to the forward
    ob_sumsq: np.ndarray
    length: int


def pendulum_episode(net: O.Net, theta: np.ndarray, init, max_steps: int = MAX_STEPS, ob_mean=None, ob_std=None,
                     ac_noise=None) -> Episode:
    """One episode: observation -> ``oracle.forward`` (normalised when ``ob_mean`` is given) -> head + ac_noise[t]
    (float32) -> ``pendulum_step``, exactly ``max_steps`` steps (no termination)."""
    if ob_mean is None:
        net = dataclasses.replace(net, ob_norm=False)
    th, thdot = float(init[0]), float(init[1])
    ret = sret = 0.0
    s, q = np.zeros(3), np.zeros(3)
    for t in range(max_steps):
        o = observation(th, thdot)
        s += o.astype(np.float64)
        q += np.square(o.astype(np.float64))
        y, _ = O.forward(net, theta, o[None, :], ob_mean=ob_mean, ob_std=ob_std)
        a = np.float32(y[0, 0]) if ac_noise is None else np.float32(y[0, 0]) + np.float32(ac_noise[t])
        th, thdot, r = pendulum_step(th, thdot, a)
        r32 = np.float32(r)
        ret += float(r32)
        sret += float(np.sign(r32))
    return Episode(th, thdot, np.float32(ret), np.float32(sret), s, q, max_steps)
