"""CPU tests of the Pendulum-v1 pieces: the referee's step against hand-derived values, the host environment against the
referee, the reset stream, registration, the episode runner's choice and the shipped configuration."""
import json
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pendulum_oracle as PO                       # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations", "pendulum_es.json")
# numpy's vectorised sin / cos against math.sin / cos: the host step may differ from the scalar referee by a few ulps
HOST_STEP_ULPS = 4


def test_hand_derived_steps():
    # from rest with full torque: thdot = (0 + 3 * 2) * 0.05 = 0.3, th = 0.3 * 0.05 = 0.015, cost 0.001 * 4
    th, thdot, r = PO.pendulum_step(0.0, 0.0, np.float32(2.0))
    assert thdot == pytest.approx(0.3, rel=1e-15) and th == pytest.approx(0.015, rel=1e-15)
    assert np.float32(r) == np.float32(-0.004)
    # (pi/2, 7.9): 7.9 + (15 + 6) * 0.05 = 8.95 is clipped to max_speed 8
    th, thdot, r = PO.pendulum_step(math.pi / 2, 7.9, np.float32(2.0))
    assert 7.9 + (15.0 * math.sin(math.pi / 2) + 6.0) * 0.05 == pytest.approx(8.95, rel=1e-15)
    assert thdot == 8.0 and th == math.pi / 2 + 8.0 * 0.05
    assert r == pytest.approx(-((math.pi / 2) ** 2 + 0.1 * 7.9 ** 2 + 0.001 * 4.0), rel=1e-15)
    # th = 3 pi / 2 is -pi / 2 in the cost
    assert PO.angle_normalize(3 * math.pi / 2) == pytest.approx(-math.pi / 2, rel=1e-15)
    _, _, r = PO.pendulum_step(3 * math.pi / 2, 0.0, np.float32(0.0))
    assert r == pytest.approx(-(math.pi / 2) ** 2, rel=1e-15)
    assert PO.angle_normalize(-3 * math.pi / 2) == pytest.approx(math.pi / 2, rel=1e-15)
    # a = +-5 is clipped to +-2
    for a in (5.0, -5.0):
        assert PO.pendulum_step(0.3, -1.0, np.float32(a)) == PO.pendulum_step(0.3, -1.0, np.float32(math.copysign(2.0, a)))


def test_host_step_agrees_with_referee():
    from dne.envs import PendulumEnv
    rs = np.random.RandomState(3)
    k = 4096
    env = PendulumEnv(k, seed=1, pin=False)
    slots = np.arange(k)
    env.reset(slots)
    env.state[: k // 4, 0] = rs.uniform(-40, 40, size=k // 4)           # large |th|
    env.state[k // 4: k // 2, 1] = rs.choice([-8.0, 8.0, 7.95, -7.95], size=k // 4)      # speeds at the clip
    worst = 0.0
    for _ in range(20):
        st = env.state.copy()
        acts = (rs.randn(k, 1) * 2.5).astype(np.float32)                      # saturated both ways too
        rew, done = env.step(slots, acts)
        assert not done.any() and rew.dtype == np.float32
        for m in range(0, k, 7):
            th, thd, r = PO.pendulum_step(st[m, 0], st[m, 1], acts[m, 0])
            for got, want in ((env.state[m, 0], th), (env.state[m, 1], thd)):
                err = abs(got - want) / np.spacing(max(abs(want), 1.0))
                worst = max(worst, err)
                assert err <= HOST_STEP_ULPS, (m, got, want)
            assert abs(float(rew[m]) - float(np.float32(r))) <= np.spacing(np.float32(abs(r))), (m, rew[m], r)
            np.testing.assert_array_equal(env.obs[m].numpy(), PO.observation(env.state[m, 0], env.state[m, 1]))
    print(f"host step vs scalar referee: worst {worst:.2f} ulps")
    np.testing.assert_array_equal(env.get_ram(np.array([5, 2])), env.state[[5, 2]])


def test_initial_states_are_successive_resets():
    from dne.envs import PendulumEnv
    env = PendulumEnv(4, seed=7, pin=False)
    a = env.initial_states(5)
    env.reset(np.array([0, 1]))                    # reset draws from the same stream
    b = env.initial_states(3)
    rs = np.random.RandomState(7)
    want = np.stack([rs.uniform(low=[-np.pi, -1.0], high=[np.pi, 1.0]) for _ in range(10)])
    assert a.dtype == np.float64 and a.shape == (5, 2)
    np.testing.assert_array_equal(a, want[:5])
    np.testing.assert_array_equal(env.state[:2], want[5:7])
    np.testing.assert_array_equal(b, want[7:])
    np.testing.assert_array_equal(env.obs[:2].numpy(), np.stack([PO.observation(*s) for s in want[5:7]]))


def test_registration(monkeypatch):
    from dne.envs import PendulumEnv, make_env
    monkeypatch.delenv("DNE_ALLOW_SYNTHETIC_ENV", raising=False)
    env = make_env("Pendulum-v1", 16, seed=3)
    assert isinstance(env, PendulumEnv) and not getattr(env, "synthetic", False)
    assert env.device_episodes and env.host_step and env.state_dim == 2 and env.max_episode_steps == 200
    np.testing.assert_array_equal(env.observation_space.low, [-1, -1, -8])
    np.testing.assert_array_equal(env.observation_space.high, [1, 1, 8])
    assert env.action_space.shape == (1,) and env.action_space.low[0] == -2 and env.action_space.high[0] == 2
    with pytest.raises(KeyError):
        make_env("Pendulum-v0", 16)
    with pytest.raises(ValueError):
        make_env("Pendulum-v1", 16, episode_len=50)


def test_pendulum_es_config_builds_mujoco_policy():
    from es_distributed import policies
    from es_distributed.es import Config
    from dne.envs import PendulumEnv
    with open(CONFIG) as f:
        exp = json.load(f)
    cfg = Config(**exp["config"])
    assert exp["env_id"] == "Pendulum-v1" and exp["policy"]["type"] == "MujocoPolicy"
    assert cfg.calc_obstat_prob == 0.01 and cfg.episode_cutoff_mode == "env_default" and cfg.l2coeff == 0.0
    assert exp["optimizer"]["type"] == "adam"
    args = exp["policy"]["args"]
    assert args["ac_bins"] == "continuous:" and args["ac_noise_std"] == 0.01 and args["nonlin_type"] == "tanh"
    env = PendulumEnv(2, pin=False)
    pol = policies.MujocoPolicy.__new__(policies.MujocoPolicy)
    net = pol._initialize(env.observation_space, env.action_space, **args)
    h = args["hidden_dims"]
    dims = [3] + list(h) + [1]
    assert net.num_params == sum(a * b + b for a, b in zip(dims[:-1], dims[1:]))
    assert net.num_params == PO.policy_net(h).num_params
    assert net.ob_dim == 3 and net.n_out == 1
