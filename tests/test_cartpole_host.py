"""CPU tests of the CartPole-v1 pieces: classifier layouts against the reference's own classes, the env backend, the
oracle's dynamics, the episode runner's argument contract and the shipped configuration."""
import json
import math
import os
import sys

import numpy as np
import pytest

from oracle import oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cartpole_oracle as CP                       # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_classifiers.npz")
CONFIG = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations", "cartpole_es.json")


@pytest.fixture(scope="module")
def ref():
    return np.load(GOLDEN)


@pytest.mark.parametrize("name,P", [("SimpleClassifier", 386), ("LinearClassifier", 10)])
def test_classifier_layouts_match_reference(ref, name, P):
    from dne import nets
    from dne import _ffi as F
    names = [str(s) for s in ref[f"{name}.names"]]
    sizes, offsets = ref[f"{name}.sizes"], ref[f"{name}.offsets"]
    scale_by = ref[f"{name}.var_scale_by"]
    assert int(ref[f"{name}.num_params"]) == P
    # dne.nets: w then b per layer, in creation order
    net = nets.make_net(name, num_actions=2, ob_dim=4)
    assert net.num_params == P and net.ob_kind == F.OB_VECTOR and net.ob_dim == 4 and net.n_out == 2
    got = []
    for l in net.layers:
        got.append(("w", l.off_w, l.cin * l.cout, np.float64(l.std) / np.sqrt(l.cin)))
        got.append(("b", l.off_b, l.cout, 0.0))
    assert [g[0] for g in got] == [n.rsplit("/", 1)[1] for n in names]
    assert [g[1] for g in got] == list(offsets) and [g[2] for g in got] == list(sizes)
    np.testing.assert_allclose([g[3] for g in got], scale_by, rtol=1e-15, atol=0)
    assert [l.act for l in net.layers] == [F.ACT_RELU] * (len(net.layers) - 1) + [F.ACT_NONE]
    # oracle: same variables, and its scale_by vector equals the reference's after float32 rounding
    onet = CP.make_classifier(name)
    assert onet.num_params == P
    assert [(v.kind, v.offset, v.size) for v in onet.variables()] == [(g[0], g[1], g[2]) for g in got]
    np.testing.assert_array_equal(O.ga_scale_by(onet), ref[f"{name}.scale_by"].astype(np.float32))


@pytest.mark.parametrize("env_id", ["CartPole-v1", "gym.CartPole-v1"])
def test_make_env_cartpole_without_opt_in(env_id, monkeypatch):
    from dne.envs import CartPoleEnv, make_env
    monkeypatch.delenv("DNE_ALLOW_SYNTHETIC_ENV", raising=False)
    env = make_env(env_id, 16, seed=3)
    assert isinstance(env, CartPoleEnv) and not getattr(env, "synthetic", False)
    assert env.device_episodes is True
    assert env.observation_space.shape == (4,) and env.action_space.n == 2 and env.max_episode_steps == 500
    with pytest.raises(NotImplementedError):
        env.step(np.array([0]), np.array([1]))
    with pytest.raises(NotImplementedError):
        env.reset(np.array([0]))


def test_initial_states_are_successive_gym_resets():
    from dne.envs import CartPoleEnv
    env = CartPoleEnv(4, seed=7)
    a = env.initial_states(5)
    b = env.initial_states(3)                       # the stream continues across calls
    rs = np.random.RandomState(7)
    want = np.stack([rs.uniform(-0.05, 0.05, size=4) for _ in range(8)])
    assert a.dtype == np.float64 and a.shape == (5, 4)
    np.testing.assert_array_equal(np.concatenate([a, b]), want)


def test_cartpole_step_first_step_by_hand():
    # from rest (all zeros) every trigonometric term is exact: cos 0 = 1, sin 0 = 0
    for action, force in ((1, 10.0), (0, -10.0)):
        temp = force / 1.1
        thetaacc = (0.0 - temp) / (0.5 * (4.0 / 3.0 - 0.1 / 1.1))
        xacc = temp - 0.05 * thetaacc / 1.1
        s, done = CP.cartpole_step(np.zeros(4), action)
        np.testing.assert_allclose(s, [0.0, 0.02 * xacc, 0.0, 0.02 * thetaacc], rtol=1e-15, atol=0)
        assert not done
        assert abs(s[1]) == pytest.approx(0.1951219512195122, rel=1e-12)     # 0.02 * 160 / 16.4
        assert abs(s[3]) == pytest.approx(0.2926829268292683, rel=1e-12)     # 0.02 * 10 / (1.1 * 0.5 * 41/33)
    # a general state, the published equations written out once more
    x, xd, th, thd = 0.01, -0.02, 0.03, 0.04
    for action in (0, 1):
        f = 10.0 if action == 1 else -10.0
        c, s_ = math.cos(th), math.sin(th)
        temp = (f + 0.05 * thd * thd * s_) / 1.1
        ta = (9.8 * s_ - c * temp) / (0.5 * (4.0 / 3.0 - 0.1 * c * c / 1.1))
        xa = temp - 0.05 * ta * c / 1.1
        s, done = CP.cartpole_step([x, xd, th, thd], action)
        np.testing.assert_allclose(s, [x + 0.02 * xd, xd + 0.02 * xa, th + 0.02 * thd, thd + 0.02 * ta], rtol=1e-14,
                                   atol=1e-17)
        assert not done
    # termination: beyond either threshold after the step
    assert CP.cartpole_step([2.4, 1.0, 0.0, 0.0], 1)[1]
    assert CP.cartpole_step([0.0, 0.0, -0.2094, -1.0], 0)[1]
    assert CP.THETA_THRESHOLD == 12 * 2 * math.pi / 360


def test_oracle_episode_accounting():
    net = CP.make_classifier("LinearClassifier")
    theta = np.zeros(net.num_params, np.float32)           # all logits 0: argmax picks action 0 every step
    ep = CP.cartpole_episode(net, theta, [0.0, 0.0, 0.0, 0.0], 500)
    assert set(ep.actions) == {0} and 1 <= ep.length < 500 and ep.min_logit_gap == 0.0
    st = np.zeros(4)
    for _ in range(ep.length):
        st, done = CP.cartpole_step(st, 0)
    np.testing.assert_array_equal(st, ep.final_state)
    assert done
    assert CP.cartpole_episode(net, theta, [0.0, 0.0, 0.0, 0.0], 3).length == 3


def test_episode_runner_rejects_what_the_kernel_does_not_do():
    import torch
    from dne import nets
    from dne.envs import CartPoleEnv
    from dne.rollout import EpisodeKernelRunner, Unit

    class _Ctx:                                            # run() validates its arguments before touching the device
        device, handle = 0, None
    r = EpisodeKernelRunner(_Ctx(), nets.make_net("SimpleClassifier", num_actions=2, ob_dim=4), CartPoleEnv(2), n_slots=2)
    th = torch.zeros(386)
    u = [Unit(0, (0.0, 0.0))]
    with pytest.raises(NotImplementedError):
        r.run(th, u, collect_bc="trace")
    with pytest.raises(NotImplementedError):
        r.run(th, u, ob_mean=th[:4], ob_std=th[:4])
    with pytest.raises(NotImplementedError):
        r.run(th, u, save_obs_prob=0.01)
    res = r.run(th, [])
    assert res.returns.shape == (0, 2) and res.steps == 0 and res.ticks == 0


def test_cartpole_es_config_parses():
    from es_distributed.es import Config
    with open(CONFIG) as f:
        exp = json.load(f)
    cfg = Config(**exp["config"])
    assert exp["env_id"] == "CartPole-v1" and exp["policy"]["type"] == "SimpleClassifierPolicy"
    assert cfg.episodes_per_batch == 5000 and cfg.noise_stdev == 0.02 and cfg.l2coeff == 0.005
    assert cfg.return_proc_mode == "centered_rank" and cfg.episode_cutoff_mode == 5000
    assert exp["optimizer"] == {"type": "adam", "args": {"stepsize": 0.01}}
