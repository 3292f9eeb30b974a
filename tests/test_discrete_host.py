"""CPU tests of the Acrobot-v1 and MountainCar-v0 pieces: the float64 referee against hand-derived steps, the environment
backends (registration, spaces, reset streams) and the shipped configurations."""
import json
import math
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cartpole_oracle as CP                       # noqa: E402
import discrete_oracle as D                        # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations")
PI = math.pi
C0 = math.cos(-PI / 2)                             # 6.1e-17: gravity's lever at rest is not exactly 0 in float64


# ---- Acrobot-v1 --------------------------------------------------------------------------------------------------------
def test_acrobot_derivative_at_rest_by_hand():
    # at rest cos(theta2) = 1, sin(theta2) = 0: d1 = 0.25 + 2.25 + 2 = 4.5, d2 = 1.75, m2 * lc2**2 + I2 - d2**2 / d1 = 41/72
    for a in (-1.0, 0.0, 1.0):
        phi2 = 4.9 * C0
        phi1 = 14.7 * C0 + phi2
        dd2 = (a + 1.75 / 4.5 * phi1 - phi2) / (1.25 - 1.75 * 1.75 / 4.5)
        dd1 = -(1.75 * dd2 + phi1) / 4.5
        got = D.acrobot_dsdt([0.0, 0.0, 0.0, 0.0], a)
        assert got[:2].tolist() == [0.0, 0.0]
        np.testing.assert_allclose(got[2:], [dd1, dd2], rtol=1e-15, atol=1e-30)
        np.testing.assert_allclose(got[2:], [-28 / 41 * a, 72 / 41 * a], rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("action", [0, 1, 2])
def test_acrobot_step_from_rest_each_torque(action):
    torque = action - 1.0
    s, r, done, raw = D.acrobot_step(np.zeros(4), action)
    assert not done and r == -1.0
    if torque == 0.0:
        assert np.abs(s).max() < 1e-13                               # only gravity's 6e-17 lever moves it
        return
    # constant acceleration to first order: dtheta ~ dt * ddtheta, theta ~ dt**2 / 2 * ddtheta (the angles feed back
    # into the accelerations within the step, so up to 10 %)
    dd1, dd2 = -28 / 41 * torque, 72 / 41 * torque
    np.testing.assert_allclose(s[2:], [0.2 * dd1, 0.2 * dd2], rtol=0.1)
    np.testing.assert_allclose(s[:2], [0.02 * dd1, 0.02 * dd2], rtol=0.1)
    assert np.sign(s[3]) == np.sign(torque) and np.sign(s[2]) == -np.sign(torque)
    # mirror symmetry: torque -a from rest gives the negated state, up to gravity's 6e-17 lever
    m, *_ = D.acrobot_step(np.zeros(4), 2 - action)
    np.testing.assert_allclose(m, -s, rtol=0, atol=1e-14)


def test_acrobot_rk4_by_hand():
    """One step written out once more: RK4 with dt2 = 0.1, the weights (1, 2, 2, 1) / 6, the torque constant in the step."""
    y0 = [0.3, -0.7, 1.1, -2.0]
    for action in (0, 1, 2):
        a = [-1.0, 0.0, 1.0][action]
        k1 = np.array(D.acrobot_dsdt(y0, a))
        k2 = np.array(D.acrobot_dsdt(list(np.array(y0) + 0.1 * k1), a))
        k3 = np.array(D.acrobot_dsdt(list(np.array(y0) + 0.1 * k2), a))
        k4 = np.array(D.acrobot_dsdt(list(np.array(y0) + 0.2 * k3), a))
        want = np.array(y0) + 0.2 / 6.0 * (k1 + 2 * k2 + 2 * k3 + k4)
        s, r, done, raw = D.acrobot_step(y0, action)
        np.testing.assert_array_equal(raw, want)
        np.testing.assert_array_equal(s, want)                      # inside every bound: nothing wrapped or clamped
        assert not done


def test_acrobot_angle_wrap():
    s, _, _, raw = D.acrobot_step([PI - 1e-3, 0.0, 4 * PI, 0.0], 1)
    assert raw[0] > PI and s[0] == raw[0] - 2 * PI and -PI <= s[0] <= PI
    s, _, _, raw = D.acrobot_step([-PI + 1e-3, 0.0, -4 * PI, 0.0], 1)
    assert raw[0] < -PI and s[0] == raw[0] + 2 * PI and -PI <= s[0] <= PI
    assert D._wrap(3 * PI + 0.5, -PI, PI) == pytest.approx(-PI + 0.5, abs=1e-14)     # two turns
    assert D._wrap(PI, -PI, PI) == PI and D._wrap(-PI, -PI, PI) == -PI                # the bounds stay


def test_acrobot_speed_clamps():
    for sign in (1.0, -1.0):
        s, _, _, raw = D.acrobot_step([0.0, 0.0, sign * 4 * PI, sign * 9 * PI], 1)
        assert sign * raw[2] > 4 * PI and sign * raw[3] > 9 * PI
        assert s[2] == sign * 4 * PI and s[3] == sign * 9 * PI
        # both angles moved past pi and wrapped
        assert sign * raw[0] > PI and sign * raw[1] > PI and abs(s[0]) <= PI and abs(s[1]) <= PI


def test_acrobot_termination_line():
    # -cos(theta1) - cos(theta2 + theta1) > 1.0
    assert D.acrobot_terminal_value([PI, 0.0, 0, 0]) == 2.0
    assert D.acrobot_terminal_value([0.0, 0.0, 0, 0]) == -2.0
    above, below = [2 * PI / 3 + 1e-6, 0.0, 0, 0], [2 * PI / 3 - 1e-6, 0.0, 0, 0]
    assert D.acrobot_terminal_value(above) > 1.0 > D.acrobot_terminal_value(below)
    # a step from the top stays above the line: done, reward 0; from rest: not done, reward -1
    s, r, done, _ = D.acrobot_step([PI, 0.0, 0.0, 0.0], 1)
    assert done and r == 0.0 and D.acrobot_terminal_value(s) > 1.0
    s, r, done, _ = D.acrobot_step([0.0, 0.0, 0.0, 0.0], 2)
    assert not done and r == -1.0


def test_acrobot_nips_variant_and_torque_offset_differ():
    y = [0.3, -0.7, 1.1, -2.0]
    book, nips = D.acrobot_dsdt(y, 1.0), D.acrobot_dsdt(y, 1.0, book=False)
    assert np.array_equal(book[:2], nips[:2]) and abs(book[3] - nips[3]) > 0.1
    assert np.abs(D.acrobot_step(y, 1)[0] - D.acrobot_step(y, 1, torque_offset=1)[0]).max() > 1e-3


# ---- MountainCar-v0 ----------------------------------------------------------------------------------------------------
def test_mountaincar_step_by_hand():
    x, v = -0.5, 0.01
    for a in (0, 1, 2):
        nv = v + ((a - 1) * 0.001 + math.cos(3 * x) * (-0.0025))
        s, r, done, _ = D.mountaincar_step([x, v], a)
        assert s.tolist() == [x + nv, nv] and r == -1.0 and not done


def test_mountaincar_left_wall_stop():
    s, r, done, _ = D.mountaincar_step([-1.19, -0.05], 0)
    assert s.tolist() == [-1.2, 0.0] and r == -1.0 and not done
    s, *_ = D.mountaincar_step([-1.2, 0.0], 2)                     # at the wall with v >= 0: no stop
    assert s[1] > 0 and s[0] > -1.2


def test_mountaincar_speed_clip():
    x = -PI / 3                                                    # cos(3x) = -1: gravity pushes right at 0.0025
    s, *_ = D.mountaincar_step([x, 0.069], 2)
    assert s[1] == 0.07 and s[0] == x + 0.07
    s, *_ = D.mountaincar_step([0.0, -0.069], 0)                   # cos(0) = 1: gravity pushes left
    assert s[1] == -0.07 and s[0] == -0.07


def test_mountaincar_goal():
    # v after the step exactly 0 at x = 0.5: done (goal_velocity 0 is inclusive)
    x = 0.5
    v = -((2 - 1) * 0.001 + math.cos(3 * x) * (-0.0025))
    s, r, done, margin = D.mountaincar_step([x, v], 2)
    assert s.tolist() == [0.5, 0.0] and done and r == -1.0 and margin == 0.0
    # past the goal position but moving left: not done
    x = 0.55
    v = -0.001 - ((1 - 1) * 0.001 + math.cos(3 * x) * (-0.0025))
    s, r, done, _ = D.mountaincar_step([x, v], 1)
    assert s[0] >= 0.5 and s[1] < 0 and not done
    # reaching the right edge clips the position
    s, _, done, _ = D.mountaincar_step([0.59, 0.06], 2)
    assert s[0] == 0.6 and done


def test_oracle_episode_accounting():
    net = CP.make_classifier("LinearClassifier", num_actions=3, ob_dim=2)
    theta = np.zeros(net.num_params, np.float32)                   # all logits 0: argmax picks action 0 every step
    ep = D.episode("mountaincar", net, theta, [-0.5, 0.0], 200)
    assert ep.length == 200 and ep.ret == -200.0 and set(ep.actions) == {0} and ep.min_logit_gap == 0.0
    st = np.array([-0.5, 0.0])
    for _ in range(200):
        st, *_ = D.mountaincar_step(st, 0)
    np.testing.assert_array_equal(st, ep.final_state)
    anet = CP.make_classifier("LinearClassifier", num_actions=3, ob_dim=6)
    ep = D.episode("acrobot", anet, np.zeros(anet.num_params, np.float32), [0.05, -0.02, 0.0, 0.01], 7)
    assert ep.length == 7 and ep.ret == -7.0


# ---- backends and configurations ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("env_id,cls,ob,n,limit", [
    ("Acrobot-v1", "AcrobotEnv", 6, 3, 500), ("gym.Acrobot-v1", "AcrobotEnv", 6, 3, 500),
    ("MountainCar-v0", "MountainCarEnv", 2, 3, 200), ("gym.MountainCar-v0", "MountainCarEnv", 2, 3, 200)])
def test_make_env_registers(env_id, cls, ob, n, limit, monkeypatch):
    from dne import envs
    monkeypatch.delenv("DNE_ALLOW_SYNTHETIC_ENV", raising=False)
    env = envs.make_env(env_id, 16, seed=3)
    assert type(env).__name__ == cls and not getattr(env, "synthetic", False)
    assert env.device_episodes is True and env.host_step is False and env.kernel_policy_io is False
    assert env.observation_space.shape == (ob,) and env.action_space.n == n and env.max_episode_steps == limit
    assert env.state_dim == (4 if cls == "AcrobotEnv" else 2)
    with pytest.raises(NotImplementedError):
        env.step(np.array([0]), np.array([1]))
    with pytest.raises(NotImplementedError):
        env.reset(np.array([0]))
    with pytest.raises(ValueError):
        envs.make_env(env_id, 4, episode_len=100)


def test_spaces_are_gyms():
    from dne.envs import AcrobotEnv, MountainCarEnv
    a = AcrobotEnv(1)
    np.testing.assert_array_equal(a.observation_space.high,
                                  np.array([1, 1, 1, 1, 4 * np.pi, 9 * np.pi], np.float32))
    np.testing.assert_array_equal(a.observation_space.low, -a.observation_space.high)
    m = MountainCarEnv(1)
    np.testing.assert_array_equal(m.observation_space.low, np.array([-1.2, -0.07], np.float32))
    np.testing.assert_array_equal(m.observation_space.high, np.array([0.6, 0.07], np.float32))


def test_continuous_mountaincar_is_not_registered():
    from dne.envs import make_env
    with pytest.raises(KeyError):
        make_env("MountainCarContinuous-v0", 4)


def test_reset_streams_are_successive_gym_resets():
    from dne.envs import AcrobotEnv, MountainCarEnv
    env = AcrobotEnv(4, seed=7)
    a, b = env.initial_states(5), env.initial_states(3)            # the stream continues across calls
    rs = np.random.RandomState(7)
    want = np.stack([rs.uniform(low=-0.1, high=0.1, size=(4,)).astype(np.float32) for _ in range(8)])
    got = np.concatenate([a, b])
    assert got.dtype == np.float64 and got.shape == (8, 4)
    np.testing.assert_array_equal(got, want.astype(np.float64))
    env = MountainCarEnv(4, seed=9)
    a, b = env.initial_states(2), env.initial_states(4)
    rs = np.random.RandomState(9)
    want = np.array([[rs.uniform(low=-0.6, high=-0.4), 0.0] for _ in range(6)])
    got = np.concatenate([a, b])
    assert got.dtype == np.float64 and got.shape == (6, 2)
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("fname,env_id,ob", [("acrobot_es.json", "Acrobot-v1", 6),
                                             ("mountaincar_ga.json", "MountainCar-v0", 2)])
def test_configs_build_their_policy_nets(fname, env_id, ob):
    from dne import nets
    from dne import _ffi as F
    from dne.envs import make_env
    from es_distributed.es import Config
    with open(os.path.join(CONFIGS, fname)) as f:
        exp = json.load(f)
    Config(**exp["config"])
    assert exp["env_id"] == env_id and exp["policy"] == {"type": "SimpleClassifierPolicy", "args": {}}
    if fname.startswith("mountaincar"):
        assert exp["population_size"] == 20 and exp["num_elites"] == 1 and "algo_type" not in exp
    env = make_env(exp["env_id"], 8)
    # SimpleClassifierPolicy._initialize: the classifier for the env's action count and observation width
    net = nets.make_net("SimpleClassifier", num_actions=env.action_space.n, ob_dim=int(env.observation_space.shape[0]))
    assert net.ob_dim == ob and net.n_out == 3 and net.ob_kind == F.OB_VECTOR
    assert [(l.cin, l.cout, l.act) for l in net.layers] == [(ob, 16, F.ACT_RELU), (16, 16, F.ACT_RELU), (16, 3, F.ACT_NONE)]
    assert CP.make_classifier("SimpleClassifier", num_actions=3, ob_dim=ob).num_params == net.num_params


def test_oracle_argmax_rule():
    # np.argmax, which the oracle acts with, is the kernel's rule: the first NaN, else the first maximum
    assert int(np.argmax(np.array([1.0, 3.0, 3.0], np.float32))) == 1
    assert int(np.argmax(np.array([1.0, np.nan, np.nan], np.float32))) == 1
    assert int(np.argmax(np.array([np.inf, 1.0, np.nan], np.float32))) == 2
    assert int(np.argmax(np.array([-np.inf] * 3, np.float32))) == 0
    assert O is not None
