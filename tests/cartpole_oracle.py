"""CPU referee for the CartPole-v1 tests (test infrastructure, imported by tests/test_cartpole_host.py and
tests/test_gpu_cartpole.py only).

* The reference GPU path's classifiers as ``oracle.oracle.Net`` layouts (gpu_implementation/neuroevolution/models/simple.py):
  SimpleClassifier (fc1 16 relu, fc2 16 relu, out std 0.1) and LinearClassifier (out only), in variable creation order --
  pinned to the reference classes by tests/golden/ref_classifiers.npz.
* gym's CartPole-v1 (classic_control cartpole.py) from its published equations, in numpy float64 and gym's operation
  order, and whole episodes played through ``oracle.oracle.forward``.  gym itself is not a dependency.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List

import numpy as np

from oracle import oracle as O


def make_classifier(name: str, num_actions: int = 2, ob_dim: int = 4) -> O.Net:
    """simple.py:23-34 on ``dqn.Model``: dense layers with 'w' then 'b', ReLU hidden layers, linear head."""
    def dense(cin, cout, act="relu", std=1.0):
        return O.Layer("dense", cin, cout, act=act, std=std,
                       vars=[O.Var("w", (cin, cout), "w", std), O.Var("b", (cout,), "b")])
    if name == "SimpleClassifier":
        layers = [dense(ob_dim, 16), dense(16, 16), dense(16, num_actions, act="none", std=0.1)]
    elif name == "LinearClassifier":
        layers = [dense(ob_dim, num_actions, act="none")]
    else:
        raise KeyError(name)
    return O._finish(O.Net(name, layers, (ob_dim,)))


def dense_net(widths, name="dense") -> O.Net:
    """An MLP of the given widths: ReLU hidden layers, linear head, biases."""
    layers = [O.Layer("dense", a, b, act="relu" if i + 2 < len(widths) else "none",
                      vars=[O.Var("w", (a, b), "w"), O.Var("b", (b,), "b")])
              for i, (a, b) in enumerate(zip(widths[:-1], widths[1:]))]
    return O._finish(O.Net(name, layers, (widths[0],)))


MAX_STEPS = 500                          # gym registers CartPole-v1 with TimeLimit(max_episode_steps=500)
_GRAVITY, _MASSCART, _MASSPOLE, _LENGTH, _FORCE, _TAU = 9.8, 1.0, 0.1, 0.5, 10.0, 0.02
_TOTAL_MASS = _MASSPOLE + _MASSCART
_POLEMASS_LENGTH = _MASSPOLE * _LENGTH
THETA_THRESHOLD = 12 * 2 * math.pi / 360
X_THRESHOLD = 2.4


def cartpole_step(state, action):
    """gym CartPole-v1 ``step``: Euler integration of the cart-pole equations in float64, gym's operation order (Python
    evaluates products left to right).  Returns (new_state float64 [4], done).  The reward is 1.0 on every step, the
    terminating one included."""
    x, x_dot, theta, theta_dot = (float(v) for v in state)
    force = _FORCE if int(action) == 1 else -_FORCE
    costheta, sintheta = math.cos(theta), math.sin(theta)
    temp = (force + _POLEMASS_LENGTH * (theta_dot * theta_dot) * sintheta) / _TOTAL_MASS
    thetaacc = (_GRAVITY * sintheta - costheta * temp) / (
        _LENGTH * (4.0 / 3.0 - _MASSPOLE * (costheta * costheta) / _TOTAL_MASS))
    xacc = temp - _POLEMASS_LENGTH * thetaacc * costheta / _TOTAL_MASS
    x = x + _TAU * x_dot
    x_dot = x_dot + _TAU * xacc
    theta = theta + _TAU * theta_dot
    theta_dot = theta_dot + _TAU * thetaacc
    done = x < -X_THRESHOLD or x > X_THRESHOLD or theta < -THETA_THRESHOLD or theta > THETA_THRESHOLD
    return np.array([x, x_dot, theta, theta_dot], dtype=np.float64), bool(done)


@dataclass
class Episode:
    length: int                      # steps taken (= return: reward 1 per step)
    final_state: np.ndarray          # float64 [4], the state after the last step
    min_logit_gap: float             # smallest |logit1 - logit0| over the episode's decisions
    min_threshold_margin: float      # smallest distance of a visited state's x / theta to its termination threshold
    actions: List[int] = field(default_factory=list)


def cartpole_episode(net: O.Net, theta: np.ndarray, init_state, max_steps: int = MAX_STEPS) -> Episode:
    """One CartPole-v1 episode of the weights ``theta``: observation ``np.array(state, dtype=np.float32)`` (as gym returns
    it) -> ``oracle.forward`` -> argmax (first max on ties) -> ``cartpole_step``, until done or ``max_steps`` steps.  The
    logit gap and threshold margin let a caller recognise episodes whose outcome hinges on the last bits of float32 /
    float64 rounding."""
    state = np.asarray(init_state, dtype=np.float64).copy()
    gap, margin, acts = math.inf, math.inf, []
    length = 0
    while True:
        logits, _ = O.forward(net, theta, np.array(state, dtype=np.float32)[None, :])
        a = int(np.argmax(logits[0]))
        gap = min(gap, abs(float(logits[0, 1]) - float(logits[0, 0])))
        acts.append(a)
        state, done = cartpole_step(state, a)
        length += 1
        margin = min(margin, abs(abs(state[0]) - X_THRESHOLD), abs(abs(state[2]) - THETA_THRESHOLD))
        if done or length >= max_steps:
            break
    return Episode(length, state, gap, margin, acts)
