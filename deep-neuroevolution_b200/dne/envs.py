"""Batched environment interface.  Emulator stepping stays on the HOST (north_star: "ALE env-step stays on the
host behind pinned cudaMemcpyAsync"); the device only ever sees uint8 frame stacks (or float vectors) and
returns actions.

Reference counterparts: gym env + ``wrap_deepmind`` (es_distributed/atari_wrappers.py:204-222) stepped one at a
time by each worker (policies.py:398-409); on the reference GPU path the TF ops ``EnvironmentReset/Observation/
Step`` over a batch of ALE instances (gpu_implementation/gym_tensorflow/tf_env.cpp:115-316).

ALE / gym / MuJoCo are not vendored by the reference and are absent from this image, so the environment shipped
here is the synthetic Frostbite-shaped stub the measurement plan names (SURVEY.md 8d): i.i.d. uint8 84x84x4
observations from a fixed pool, rewards 10*Bernoulli(0.05), fixed or ragged episode lengths.  A real emulator
plugs in by subclassing ``BatchEnv``.  Four real tasks need no emulator: CartPole-v1 (``CartPoleEnv``), Acrobot-v1
(``AcrobotEnv``), MountainCar-v0 (``MountainCarEnv``), Pendulum-v1 (``PendulumEnv``) and the reference's hard maze
(``MazeEnv``), whose episodes run whole on the device (``dne.rollout.EpisodeKernelRunner``).  The same maze seen as an
84x84 image (``ImageMazeEnv``, ``ImageHardMaze-v0``) is the conv policies' real task: stepped and rendered on the device
one tick at a time under the per-tick runner.

An environment with device episodes (``device_episodes = True``) supplies ``state_dim``, ``initial_states(k)``,
``episode_net_supported(net)`` and ``launch_episodes(...)``; ``kernel_policy_io`` says whether its kernel also takes
observation statistics, action noise and observation sums (MujocoPolicy), and ``host_step`` whether the per-tick
``RolloutRunner`` can step it on the host instead.  ``bc_dim`` (default ``state_dim``) is how many leading components of
the final state form the 'final' behaviour characterisation.
"""
from __future__ import annotations

from typing import Optional, Sequence

import ctypes as C
import os

import numpy as np
import torch

from . import _ffi as F


class Discrete:
    def __init__(self, n):
        self.n = int(n)
        self.shape = ()


class Box:
    def __init__(self, low, high, shape=None, dtype=np.float32):
        self.low = np.broadcast_to(np.asarray(low, dtype=dtype), shape if shape is not None else np.shape(low)).copy()
        self.high = np.broadcast_to(np.asarray(high, dtype=dtype), self.low.shape).copy()
        self.shape = self.low.shape


class BatchEnv:
    """``n_slots`` independent environments.  Observations live in a pinned host tensor ``obs`` [n_slots, ...]
    so the engine can cudaMemcpyAsync them without staging."""
    observation_space = None
    action_space = None
    n_slots = 0
    max_episode_steps: Optional[int] = None     # env.spec...max_episode_steps of the reference (policies.py:383)

    def reset(self, slots: np.ndarray) -> None:
        raise NotImplementedError

    def step(self, slots: np.ndarray, actions: np.ndarray):
        """Step the listed slots.  Returns (rewards float32 [k], done bool [k]); new observations are written
        into ``self.obs[slots]``."""
        raise NotImplementedError

    def obs_block(self, lo: int, hi: int) -> torch.Tensor:
        """Pinned host view of the observations of slots [lo, hi) for the next forward."""
        return self.obs[lo:hi]

    def get_ram(self, slots: np.ndarray) -> np.ndarray:
        """Behaviour characterisation source (policies.py:410): uint8 [k,128]."""
        raise NotImplementedError

    def random_actions(self, k: int, rs: np.random.RandomState) -> np.ndarray:
        return rs.randint(0, self.action_space.n, size=k)


class SyntheticAtariEnv(BatchEnv):
    """Frostbite-shaped stub (SURVEY.md 8d config 2): 18 actions, 84x84x4 uint8 observations drawn i.i.d. uniform
    from ``torch.Generator(seed)`` (a pool of frames, rotated every tick), reward 10*Bernoulli(0.05), episode
    length fixed (``episode_len``) or ragged ``U{lo..hi}`` per episode (seeded)."""

    def __init__(self, n_slots: int, num_actions: int = 18, episode_len=1000, seed: int = 0, pool_blocks: int = 4,
                 pin: bool = True):
        self.n_slots = int(n_slots)
        self.observation_space = Box(0, 255, (84, 84, 4), dtype=np.uint8)
        self.action_space = Discrete(num_actions)
        g = torch.Generator().manual_seed(seed)
        self.pool_blocks = int(pool_blocks)
        pool = torch.randint(0, 256, (self.pool_blocks, self.n_slots, 84, 84, 4), dtype=torch.uint8, generator=g)
        self.pool = pool.pin_memory() if (pin and torch.cuda.is_available()) else pool
        self.obs = self.pool[0]
        self._tick = 0
        self.rs = np.random.RandomState(seed)
        self.episode_len_spec = episode_len
        self.max_episode_steps = episode_len if isinstance(episode_len, int) else int(episode_len[1])
        self.ep_len = np.zeros(self.n_slots, dtype=np.int64)
        self.t = np.zeros(self.n_slots, dtype=np.int64)
        self.ram = self.rs.randint(0, 256, size=(self.n_slots, 128)).astype(np.uint8)

    def _draw_len(self, k):
        if isinstance(self.episode_len_spec, int):
            return np.full(k, self.episode_len_spec, dtype=np.int64)
        lo, hi = self.episode_len_spec
        return self.rs.randint(lo, hi + 1, size=k).astype(np.int64)

    def reset(self, slots):
        slots = np.asarray(slots, dtype=np.int64)
        self.ep_len[slots] = self._draw_len(len(slots))
        self.t[slots] = 0

    def step(self, slots, actions):
        slots = np.asarray(slots, dtype=np.int64)
        assert len(actions) == len(slots)
        self.t[slots] += 1
        rew = (self.rs.random_sample(len(slots)) < 0.05).astype(np.float32) * np.float32(10.0)
        done = self.t[slots] >= self.ep_len[slots]
        # behaviour characterisation stand-in: RAM drifts with the action taken
        self.ram[slots, self.t[slots] % 128] = (np.asarray(actions).astype(np.int64) * 13 + self.t[slots]) & 255
        return rew, done

    def advance(self):
        """Rotate the observation pool: the next forward sees a fresh block of frames (obs do not depend on the
        actions in the stub, but the engine still waits for the actions before calling ``step``)."""
        self._tick += 1
        self.obs = self.pool[self._tick % self.pool_blocks]

    def get_ram(self, slots):
        return self.ram[np.asarray(slots, dtype=np.int64)].copy()


class DeterministicAtariEnv(BatchEnv):
    """Atari-shaped test environment whose episodes are a pure function of the ACTIONS: the observation after t steps is
    frame ``t % R`` of one fixed seeded sequence, the reward is 10 when ``(7*action + t) % 11 == 0``, the episode length is
    fixed, the RAM drifts with the actions.  An episode's return / length / behaviour characterisation therefore depend
    only on the policy weights, not on which slot, wave or rank ran it: world-size-1 and world-size-N runs of a driver
    must agree exactly (tests/test_gpu_multi.py)."""

    def __init__(self, n_slots: int, num_actions: int = 18, episode_len: int = 6, seed: int = 0, frames: int = 8,
                 pin: bool = True):
        self.n_slots = int(n_slots)
        self.observation_space = Box(0, 255, (84, 84, 4), dtype=np.uint8)
        self.action_space = Discrete(num_actions)
        g = torch.Generator().manual_seed(seed)
        self.frames = torch.randint(0, 256, (frames, 84, 84, 4), dtype=torch.uint8, generator=g)
        obs = torch.zeros(self.n_slots, 84, 84, 4, dtype=torch.uint8)
        self.obs = obs.pin_memory() if (pin and torch.cuda.is_available()) else obs
        self.max_episode_steps = int(episode_len)
        self.t = np.zeros(self.n_slots, dtype=np.int64)
        self.ram = np.zeros((self.n_slots, 128), dtype=np.uint8)

    def reset(self, slots):
        slots = np.asarray(slots, dtype=np.int64)
        self.t[slots] = 0
        self.ram[slots] = 0
        self.obs[torch.from_numpy(slots)] = self.frames[0]

    def step(self, slots, actions):
        slots = np.asarray(slots, dtype=np.int64)
        a = np.asarray(actions).astype(np.int64)
        t = self.t[slots]
        rew = (((7 * a + t) % 11) == 0).astype(np.float32) * np.float32(10.0)
        self.ram[slots, t % 128] = (a * 13 + t + 1) & 255
        self.t[slots] = t + 1
        self.obs[torch.from_numpy(slots)] = self.frames[torch.from_numpy((t + 1) % len(self.frames))]
        return rew, self.t[slots] >= self.max_episode_steps

    def get_ram(self, slots):
        return self.ram[np.asarray(slots, dtype=np.int64)].copy()


class SyntheticVectorEnv(BatchEnv):
    """Humanoid-shaped stub (SURVEY.md 8d config 5): float32 observations ~ N(0,1) of dimension ``ob_dim``,
    continuous actions of dimension ``ac_dim``, reward = -|a|^2*1e-3 + 1 (alive bonus), fixed length."""

    def __init__(self, n_slots: int, ob_dim: int = 376, ac_dim: int = 17, episode_len: int = 1000, seed: int = 0,
                 pool_blocks: int = 4, pin: bool = True):
        self.n_slots = int(n_slots)
        self.observation_space = Box(-np.inf, np.inf, (ob_dim,))
        self.action_space = Box(-0.4, 0.4, (ac_dim,))
        g = torch.Generator().manual_seed(seed)
        pool = torch.randn(pool_blocks, self.n_slots, ob_dim, generator=g)
        self.pool = pool.pin_memory() if (pin and torch.cuda.is_available()) else pool
        self.pool_blocks = pool_blocks
        self.obs = self.pool[0]
        self._tick = 0
        self.max_episode_steps = int(episode_len)
        self.t = np.zeros(self.n_slots, dtype=np.int64)
        self.pos = np.zeros((self.n_slots, 2), dtype=np.float64)

    def reset(self, slots):
        slots = np.asarray(slots, dtype=np.int64)
        self.t[slots] = 0
        self.pos[slots] = 0

    def step(self, slots, actions):
        slots = np.asarray(slots, dtype=np.int64)
        a = np.asarray(actions, dtype=np.float32).reshape(len(slots), -1)
        self.t[slots] += 1
        self.pos[slots] += a[:, :2]
        rew = (1.0 - 1e-3 * np.square(a).sum(axis=1)).astype(np.float32)
        return rew, self.t[slots] >= self.max_episode_steps

    def advance(self):
        self._tick += 1
        self.obs = self.pool[self._tick % self.pool_blocks]

    def get_ram(self, slots):          # final (x, y) position BC (policies.py:292-299)
        return self.pos[np.asarray(slots, dtype=np.int64)].copy()

    def random_actions(self, k, rs):
        return rs.uniform(-0.4, 0.4, size=(k, self.action_space.shape[0])).astype(np.float32)


def make_env(env_id: str, n_slots: int, seed: int = 0, episode_len=None, allow_synthetic: bool = False, **kw) -> BatchEnv:
    """``gym.make(exp['env_id'])`` (es.py:131) for a whole slot table.

    ALE / gym / MuJoCo are not vendored by the reference and are absent from this image, so apart from CartPole-v1,
    Acrobot-v1, MountainCar-v0 and Pendulum-v1 (registered in ``ENV_BACKENDS``) the only backends here are the synthetic stubs.  They are returned for the explicit ids ``SyntheticAtari*`` / ``SyntheticVector*``; for a REAL id
    (``FrostbiteNoFrameskip-v4``, ``Humanoid-v1`` ...) they are returned only when the caller opts in
    (``exp['allow_synthetic_env'] = true`` or ``DNE_ALLOW_SYNTHETIC_ENV=1``), with a loud warning -- a run that silently
    optimised random frames while logging and snapshotting like a real one would be worse than an error.  A real emulator
    backend registers itself in ``ENV_BACKENDS`` (id prefix -> factory)."""
    import logging
    import os
    for prefix, factory in ENV_BACKENDS.items():
        if env_id.startswith(prefix):
            return factory(env_id, n_slots, seed=seed, episode_len=episode_len, **kw)
    atari = env_id.endswith("NoFrameskip-v4") or env_id.startswith("SyntheticAtari")
    vector = env_id.startswith("Humanoid") or env_id.startswith("SyntheticVector")
    if not (atari or vector):
        raise KeyError(f"no environment backend for {env_id!r} in this build (gym/ALE/MuJoCo are not vendored)")
    if not env_id.startswith("Synthetic"):
        if not (allow_synthetic or os.environ.get("DNE_ALLOW_SYNTHETIC_ENV") == "1"):
            raise KeyError(f"no real environment backend for {env_id!r} in this build (gym/ALE/MuJoCo are not vendored); "
                           "register one in dne.envs.ENV_BACKENDS, or opt in to the synthetic stand-in with "
                           "exp['allow_synthetic_env'] = true / DNE_ALLOW_SYNTHETIC_ENV=1")
        logging.getLogger(__name__).warning(
            "SYNTHETIC ENVIRONMENT standing in for %r: observations are random frames / vectors and rewards are Bernoulli "
            "noise -- throughput measurements only, NOT training on the real task", env_id)
    if atari:
        env = SyntheticAtariEnv(n_slots, episode_len=episode_len if episode_len is not None else 1000, seed=seed, **kw)
    else:
        env = SyntheticVectorEnv(n_slots, episode_len=episode_len if episode_len is not None else 1000, seed=seed, **kw)
    env.synthetic = True
    return env


class DiscreteDeviceEnv(BatchEnv):
    """Base of gym's discrete-action classic_control tasks whose whole episodes run ON THE DEVICE, one warp per member
    (``dne_discrete_episodes``, ``dne.rollout.EpisodeKernelRunner``): a subclass supplies the spaces, the time limit,
    ``state_dim``, its ``DNE_EPISODE_*`` id and ``initial_states(k)``, drawn from one ``RandomState(seed)`` stream that
    continues across calls, as one gym env reset k times in a row would.  There is no host step."""
    device_episodes = True
    host_step = False
    kernel_policy_io = False       # no observation normalisation, action noise or observation statistics in the kernel
    episode_env: int = -1          # DNE_EPISODE_*

    def episode_net_supported(self, net) -> bool:
        return True                # the only path: the kernel itself rejects a net it cannot run

    def launch_episodes(self, ctx, net, theta, d_idx, d_scale, d_row, n, d_init, limit, d_ret, d_sret, d_len, d_fin,
                        **_):
        F.check(F.lib().dne_discrete_episodes(
            ctx.handle, self.episode_env, C.byref(net.desc), F.ptr(theta, torch.float32), F.ptr(d_idx), F.ptr(d_scale),
            F.ptr(d_row), n, F.ptr(d_init), int(limit), F.ptr(d_ret), F.ptr(d_len), F.ptr(d_fin), F.stream_ptr()))
        d_sret.copy_(d_ret)        # every reward is -1, 0 or +1: the sign-return is the return

    def _host_stepping(self, *a, **kw):
        raise NotImplementedError(f"{type(self).__name__} runs whole episodes on the device: use dne.rollout.make_runner "
                                  "(EpisodeKernelRunner), not the per-tick host reset / step")
    reset = step = obs_block = get_ram = _host_stepping


class CartPoleEnv(DiscreteDeviceEnv):
    """gym's CartPole-v1 (classic_control cartpole.py) for a whole population, stepped ON THE DEVICE: whole episodes run in
    one launch of ``dne_cartpole_episodes`` (``dne.rollout.EpisodeKernelRunner``), so this object only supplies the spaces,
    the time limit, the reset states and the launch.  ``initial_states(k)`` draws k resets ``uniform(-0.05, 0.05, size=4)``
    from one ``RandomState(seed)`` stream that continues across calls, as one gym env reset k times in a row would."""
    state_dim = 4
    episode_env = F.EPISODE_CARTPOLE

    def __init__(self, n_slots: int, seed: int = 0):
        self.n_slots = int(n_slots)
        high = np.array([2.4 * 2, np.finfo(np.float32).max, (12 * 2 * np.pi / 360) * 2, np.finfo(np.float32).max],
                        dtype=np.float32)                                        # gym's observation_space bounds
        self.observation_space = Box(-high, high)
        self.action_space = Discrete(2)
        self.max_episode_steps = 500                                             # TimeLimit of CartPole-v1
        self.rs = np.random.RandomState(seed)

    def initial_states(self, k: int) -> np.ndarray:
        """float64 [k, 4] reset states (gym ``reset``: ``uniform(low=-0.05, high=0.05, size=(4,))`` per episode)."""
        return self.rs.uniform(-0.05, 0.05, size=(int(k), 4))

    def launch_episodes(self, ctx, net, theta, d_idx, d_scale, d_row, n, d_init, limit, d_ret, d_sret, d_len, d_fin,
                        **_):
        F.check(F.lib().dne_cartpole_episodes(
            ctx.handle, C.byref(net.desc), F.ptr(theta, torch.float32), F.ptr(d_idx), F.ptr(d_scale), F.ptr(d_row), n,
            F.ptr(d_init), int(limit), F.ptr(d_ret), F.ptr(d_len), F.ptr(d_fin), F.stream_ptr()))
        d_sret.copy_(d_ret)        # every reward is +1: the sign-return is the return


def _make_cartpole(env_id, n_slots, seed=0, episode_len=None, **kw):
    if episode_len is not None:
        raise ValueError("CartPole-v1 has a fixed 500-step time limit; use the episode cutoff of the config instead")
    return CartPoleEnv(n_slots, seed=seed)


class AcrobotEnv(DiscreteDeviceEnv):
    """gymnasium's Acrobot-v1 (classic_control acrobot.py, "book" dynamics, no torque noise; DESIGN.md 3.5) for a whole
    population, stepped on the device.  State (theta1, theta2, dtheta1, dtheta2); observation float32([cos theta1,
    sin theta1, cos theta2, sin theta2, dtheta1, dtheta2]); 3 actions (torque -1, 0, +1); reward -1 per step, 0 on the
    terminating one; TimeLimit 500.  Resets draw ``uniform(-0.1, 0.1, size=4)`` per episode, rounded to float32 as gym
    stores them."""
    state_dim = 4
    episode_env = F.EPISODE_ACROBOT

    def __init__(self, n_slots: int, seed: int = 0):
        self.n_slots = int(n_slots)
        high = np.array([1.0, 1.0, 1.0, 1.0, 4 * np.pi, 9 * np.pi], dtype=np.float32)   # gym's observation_space bounds
        self.observation_space = Box(-high, high)
        self.action_space = Discrete(3)
        self.max_episode_steps = 500                                             # TimeLimit of Acrobot-v1
        self.rs = np.random.RandomState(seed)

    def initial_states(self, k: int) -> np.ndarray:
        """float64 [k, 4] reset states."""
        return self.rs.uniform(-0.1, 0.1, size=(int(k), 4)).astype(np.float32).astype(np.float64)


class MountainCarEnv(DiscreteDeviceEnv):
    """gymnasium's MountainCar-v0 (classic_control mountain_car.py; DESIGN.md 3.5) for a whole population, stepped on the
    device.  State and observation (position, velocity); 3 actions (push left, none, right); reward -1 on every step; done
    at position >= 0.5 with velocity >= 0; TimeLimit 200.  Resets draw the position ``uniform(-0.6, -0.4)`` per episode,
    velocity 0."""
    state_dim = 2
    episode_env = F.EPISODE_MOUNTAINCAR

    def __init__(self, n_slots: int, seed: int = 0):
        self.n_slots = int(n_slots)
        self.observation_space = Box(np.array([-1.2, -0.07], np.float32), np.array([0.6, 0.07], np.float32))
        self.action_space = Discrete(3)
        self.max_episode_steps = 200                                             # TimeLimit of MountainCar-v0
        self.rs = np.random.RandomState(seed)

    def initial_states(self, k: int) -> np.ndarray:
        """float64 [k, 2] reset states (position, 0)."""
        return np.stack([self.rs.uniform(-0.6, -0.4, size=int(k)), np.zeros(int(k))], axis=1)


def _fixed_limit_factory(cls, name, limit):
    def make(env_id, n_slots, seed=0, episode_len=None, **kw):
        if episode_len is not None:
            raise ValueError(f"{name} has a fixed {limit}-step time limit; use the episode cutoff of the config instead")
        return cls(n_slots, seed=seed)
    return make


_make_acrobot = _fixed_limit_factory(AcrobotEnv, "Acrobot-v1", 500)
_make_mountaincar = _fixed_limit_factory(MountainCarEnv, "MountainCar-v0", 200)


class PendulumEnv(BatchEnv):
    """gymnasium's Pendulum-v1 (classic_control pendulum.py; DESIGN.md 3.6) for a whole population.  Whole episodes run on the
    device in one launch of ``dne_pendulum_episodes`` (``dne.rollout.EpisodeKernelRunner``); for nets that kernel does not
    take (wider hidden layers, discretised heads whose ``action_fn`` runs on the host) the same dynamics step here, on the
    host, vectorised in numpy float64 in the same operation order, under the per-tick ``RolloutRunner``.  There is no
    termination; TimeLimit 200.  Resets draw ``uniform(low=[-pi, -1], high=[pi, 1])`` per episode from one
    ``RandomState(seed)`` stream that continues across calls (``initial_states`` and ``reset`` share it).  ``get_ram``
    returns the state ``(th, thdot)``: the 'final' behaviour characterisation."""
    device_episodes = True
    host_step = True
    kernel_policy_io = True
    state_dim = 2
    HIGH = np.array([np.pi, 1.0])

    def __init__(self, n_slots: int, seed: int = 0, pin: bool = True):
        self.n_slots = int(n_slots)
        self.observation_space = Box(np.array([-1.0, -1.0, -8.0], np.float32), np.array([1.0, 1.0, 8.0], np.float32))
        self.action_space = Box(-2.0, 2.0, (1,))
        self.max_episode_steps = 200                                             # TimeLimit of Pendulum-v1
        self.rs = np.random.RandomState(seed)
        self.state = np.zeros((self.n_slots, 2), dtype=np.float64)
        obs = torch.zeros(self.n_slots, 3, dtype=torch.float32)
        self.obs = obs.pin_memory() if (pin and torch.cuda.is_available()) else obs

    def initial_states(self, k: int) -> np.ndarray:
        """float64 [k, 2] reset states (th, thdot)."""
        return self.rs.uniform(low=-self.HIGH, high=self.HIGH, size=(int(k), 2))

    def episode_net_supported(self, net, action_bins=None) -> bool:
        """Whether ``dne_pendulum_episodes`` takes ``net`` (with ``action_bins``, the policy's [1, nb] bin table:
        whether ``dne_pendulum_binned_episodes`` takes it, on one CTA or a cluster)."""
        if action_bins is not None:
            return F.lib().dne_pendulum_binned_net_supported(C.byref(net.desc), _bin_table(action_bins, 1).shape[1]) == 0
        return F.lib().dne_pendulum_net_supported(C.byref(net.desc)) == 0

    def launch_episodes(self, ctx, net, theta, d_idx, d_scale, d_row, n, d_init, limit, d_ret, d_sret, d_len, d_fin,
                        d_ob_mean=None, d_ob_std=None, d_ac_noise=None, d_ob_sum=None, d_ob_sumsq=None,
                        action_bins=None):
        """One member per CTA group (``dne_pendulum_episodes``) when the net fits a CTA, otherwise one member per
        thread-block cluster (``dne_pendulum_cluster_episodes``, automatic size): the same numbers either way.
        ``action_bins``: the policy's float32 [1, nb] bin table of a discretised head, run by
        ``dne_pendulum_binned_episodes`` (which picks the kernel the same way; ``d_ac_noise`` is then [n, limit, 1])."""
        args = (C.byref(net.desc), F.ptr(theta, torch.float32), F.ptr(d_idx), F.ptr(d_scale), F.ptr(d_row), n,
                F.ptr(d_init), int(limit), F.ptr(d_ob_mean), F.ptr(d_ob_std), F.ptr(d_ac_noise), F.ptr(d_ret),
                F.ptr(d_sret), F.ptr(d_len), F.ptr(d_fin), F.ptr(d_ob_sum), F.ptr(d_ob_sumsq))
        if action_bins is not None:
            tab = _bin_table(action_bins, 1)
            F.check(F.lib().dne_pendulum_binned_episodes(ctx.handle, *args, tab.ctypes.data_as(C.c_void_p),
                                                         tab.shape[1], 0, F.stream_ptr()))
        elif self.episode_net_supported(net):
            F.check(F.lib().dne_pendulum_episodes(ctx.handle, *args, F.stream_ptr()))
        else:
            F.check(F.lib().dne_pendulum_cluster_episodes(ctx.handle, *args, 0, F.stream_ptr()))

    def _write_obs(self, slots):
        th, thdot = self.state[slots, 0], self.state[slots, 1]
        self.obs[torch.from_numpy(slots)] = torch.from_numpy(np.stack([np.cos(th), np.sin(th), thdot], axis=1)
                                                             .astype(np.float32))

    def reset(self, slots):
        slots = np.asarray(slots, dtype=np.int64)
        self.state[slots] = self.initial_states(len(slots))
        self._write_obs(slots)

    def step(self, slots, actions):
        """gymnasium ``step`` for the listed slots; ``actions`` float32 [k, 1].  Rewards float32 [k], done all False."""
        slots = np.asarray(slots, dtype=np.int64)
        u = np.clip(np.asarray(actions, dtype=np.float32).reshape(len(slots), 1), -2.0, 2.0)[:, 0]   # float32
        th, thdot = self.state[slots, 0], self.state[slots, 1]
        an = np.mod(th + np.pi, 2 * np.pi) - np.pi                                                    # angle_normalize
        costs = an ** 2 + 0.1 * thdot ** 2 + 0.001 * (u * u).astype(np.float64)
        newthdot = np.clip(thdot + (15.0 * np.sin(th) + 3.0 * u.astype(np.float64)) * 0.05, -8.0, 8.0)
        self.state[slots, 0] = th + newthdot * 0.05
        self.state[slots, 1] = newthdot
        self._write_obs(slots)
        return (-costs).astype(np.float32), np.zeros(len(slots), dtype=bool)

    def get_ram(self, slots):
        return self.state[np.asarray(slots, dtype=np.int64)].copy()

    def random_actions(self, k, rs):
        return rs.uniform(-2.0, 2.0, size=(k, 1)).astype(np.float32)


def _bin_table(action_bins, adim: int) -> np.ndarray:
    """The policy's bin table as the binned entries take it: C-contiguous float32 [adim, nb]."""
    tab = np.ascontiguousarray(action_bins, dtype=np.float32)
    if tab.ndim != 2 or tab.shape[0] != adim:
        raise ValueError(f"action_bins must be [{adim}, n_bins] (one row per action dimension), got {tab.shape}")
    return tab


def _make_pendulum(env_id, n_slots, seed=0, episode_len=None, **kw):
    if episode_len is not None:
        raise ValueError("Pendulum-v1 has a fixed 200-step time limit; use the episode cutoff of the config instead")
    return PendulumEnv(n_slots, seed=seed, **kw)


class MazeEnv(BatchEnv):
    """The hard maze of the reference's GPU path (``gym_tensorflow.make('maze', batch_size)``: gym_tensorflow/maze/maze.h
    stepped as tf_maze.cpp does; DESIGN.md 3.7) for a whole population, stepped on the device in one launch of
    ``dne_maze_episodes`` (``dne.rollout.EpisodeKernelRunner``).  A navigator with 6 rangefinders and a 4-sector goal
    radar (11 float32 observations, the first a constant 1) and two continuous outputs (turn, speed), played for a fixed
    400 steps; the only reward is -distance to the goal on the 400th step, so a truncated episode pays 0.  Every episode
    starts from the maze file's start.  The state is (x, y, heading, speed, ang_vel, t, collided); the 'final' behaviour
    characterisation is its first ``bc_dim`` = 2 components, the final (x, y) of the reference's ``MazeFinalState``.
    ``maze_file``: a maze in the reference's text format (default: the reference's hard maze, tests/golden/hard_maze.txt).
    There is no host step."""
    device_episodes = True
    host_step = False
    kernel_policy_io = True
    state_dim = 7
    bc_dim = 2
    MAX_STEPS = 400

    def __init__(self, n_slots: int, maze_file: Optional[str] = None, seed: int = 0):
        self.n_slots = int(n_slots)
        self.maze_file = maze_file or DEFAULT_MAZE_FILE
        self.walls, self.start, self.goal, self.collisions_stick = parse_maze(self.maze_file)
        self.observation_space = Box(-np.inf, np.inf, (11,))
        self.action_space = Box(-0.5, 0.5, (2,))
        self.max_episode_steps = self.MAX_STEPS
        self.desc = maze_desc(self.walls, self.goal, self.collisions_stick)

    def initial_states(self, k: int) -> np.ndarray:
        """float64 [k, 7]: the start, heading, speed and angular velocity 0, no steps taken, no collision."""
        s = np.zeros((int(k), self.state_dim))
        s[:, 0], s[:, 1] = self.start
        return s

    def episode_net_supported(self, net, action_bins=None) -> bool:
        return True                # the only path: the kernel itself rejects a net it cannot run

    def launch_episodes(self, ctx, net, theta, d_idx, d_scale, d_row, n, d_init, limit, d_ret, d_sret, d_len, d_fin,
                        d_ob_mean=None, d_ob_std=None, d_ac_noise=None, d_ob_sum=None, d_ob_sumsq=None,
                        action_bins=None):
        """One member per CTA group (``dne_maze_episodes``) when the net fits a CTA, otherwise one member per
        thread-block cluster (``dne_maze_cluster_episodes``, automatic size; MujocoPolicy's hidden [256, 256]): the same
        numbers either way.  A net neither kernel takes raises with the cluster entry's reason.  ``action_bins``: the
        policy's float32 [2, nb] bin table of a discretised head, run by ``dne_maze_binned_episodes`` (which picks the
        kernel the same way; ``d_ac_noise`` is then [n, limit, 2])."""
        L = F.lib()
        args = (C.byref(self.desc), C.byref(net.desc), F.ptr(theta, torch.float32), F.ptr(d_idx), F.ptr(d_scale),
                F.ptr(d_row), n, F.ptr(d_init), int(limit), F.ptr(d_ob_mean), F.ptr(d_ob_std), F.ptr(d_ac_noise),
                F.ptr(d_ret), F.ptr(d_sret), F.ptr(d_len), F.ptr(d_fin), F.ptr(d_ob_sum), F.ptr(d_ob_sumsq))
        if action_bins is not None:
            tab = _bin_table(action_bins, 2)
            F.check(L.dne_maze_binned_episodes(ctx.handle, *args, tab.ctypes.data_as(C.c_void_p), tab.shape[1], 0,
                                               F.stream_ptr()))
        elif L.dne_maze_net_supported(C.byref(net.desc)) == 0:
            F.check(L.dne_maze_episodes(ctx.handle, *args, F.stream_ptr()))
        else:
            F.check(L.dne_maze_cluster_episodes(ctx.handle, *args, 0, F.stream_ptr()))

    def _host_stepping(self, *a, **kw):
        raise NotImplementedError("MazeEnv runs whole episodes on the device: use dne.rollout.make_runner "
                                  "(EpisodeKernelRunner), not the per-tick host reset / step")
    reset = step = obs_block = get_ram = _host_stepping


DEFAULT_MAZE_FILE = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))), "tests",
                                 "golden", "hard_maze.txt")


def parse_maze(path: str):
    """A maze in the reference's text format (maze.h ``load_from``): the collision flag, the step count (unused: episodes
    are 400 steps, as tf_maze.cpp fixes them), the wall count, the start (x, y), the start heading (unused: ``reset``
    sets 0), the goal (x, y), a point of interest (unused), then one wall (ax, ay, bx, by) per line.  Returns (float32
    walls [n, 4], start, goal, collision flag)."""
    with open(path) as f:
        tok = f.read().split()
    try:
        flag, n = int(tok[0]), int(tok[2])
        v = [float(t) for t in tok[3:10 + 4 * n]]
    except (IndexError, ValueError) as e:
        raise ValueError(f"{path}: not a maze file ({e})") from None
    if len(v) != 7 + 4 * n or n < 0:
        raise ValueError(f"{path}: {n} walls announced, {max(len(v) - 7, 0) / 4:g} given")
    if n > F.MAZE_MAX_WALLS:
        raise ValueError(f"{path}: {n} walls, the device maze takes at most {F.MAZE_MAX_WALLS}")
    f32 = np.float32
    return (np.array(v[7:], dtype=np.float32).reshape(n, 4), (float(f32(v[0])), float(f32(v[1]))),
            (float(f32(v[3])), float(f32(v[4]))), bool(flag))


def maze_desc(walls, goal, collisions_stick) -> F.MazeDesc:
    """The C ABI's dne_maze_desc of a parsed maze."""
    desc = F.MazeDesc(n_walls=len(walls), collisions_stick=int(collisions_stick))
    desc.goal[0], desc.goal[1] = goal
    for j, w in enumerate(walls):
        for k in range(4):
            desc.walls[j][k] = float(w[k])
    return desc


def _make_maze(env_id, n_slots, seed=0, episode_len=None, maze_file=None, **kw):
    if episode_len is not None:
        raise ValueError("the maze has a fixed 400-step episode; use the episode cutoff of the config instead")
    return MazeEnv(n_slots, maze_file=maze_file, seed=seed)


class ImageMazeEnv(BatchEnv):
    """The hard maze seen from above as an 84x84 image (DESIGN.md 3.10), for the Atari conv policies (``LargeModelPolicy``,
    ``GAAtariPolicy``, ``ESAtariPolicy``) under the per-tick ``dne.rollout.RolloutRunner``.  The dynamics are
    ``MazeEnv``'s (the same device code, ``dne_image_maze_step``); a discrete action index picks a (turn, speed) row of
    ``actions`` (default: 9 rows, each of turn and speed in {-0.5, 0, +0.5}, turn major).  Episodes are 400 steps from the
    maze file's start; the only reward is -distance to the goal on the 400th step.  The observation is a uint8 84x84x4
    frame stack, newest frame last, that never leaves the device: ``device_obs(lo, hi)``.  ``get_ram`` returns the final
    (x, y), the 'final' behaviour characterisation (``bc_kind``); there is no RAM trace.  The image rule and the action
    table are this project's definitions, not the Deep GA paper's."""
    bc_kind = "final"
    bc_dim = 2
    MAX_STEPS = 400
    DEFAULT_ACTIONS = tuple((turn, speed) for turn in (-0.5, 0.0, 0.5) for speed in (-0.5, 0.0, 0.5))

    def __init__(self, n_slots: int, maze_file: Optional[str] = None, seed: int = 0, actions=None, device=None):
        self.n_slots = int(n_slots)
        self.maze_file = maze_file or DEFAULT_MAZE_FILE
        self.walls, self.start, self.goal, self.collisions_stick = parse_maze(self.maze_file)
        if len(self.walls) == 0:
            raise ValueError(f"{self.maze_file}: the image maze needs at least one wall to frame the image")
        tab = np.ascontiguousarray(self.DEFAULT_ACTIONS if actions is None else actions, dtype=np.float32)
        if tab.ndim != 2 or tab.shape[1] != 2 or not 1 <= len(tab) <= F.IMAGE_MAZE_MAX_ACTIONS:
            raise ValueError(f"actions must be [n, 2] (turn, speed) rows, 1 <= n <= {F.IMAGE_MAZE_MAX_ACTIONS}; got "
                             f"{tab.shape}")
        self.action_table = tab
        self.observation_space = Box(0, 255, (84, 84, 4), dtype=np.uint8)
        self.action_space = Discrete(len(tab))
        self.max_episode_steps = self.MAX_STEPS
        self.desc = maze_desc(self.walls, self.goal, self.collisions_stick)
        self.final_xy = np.tile(np.array(self.start, dtype=np.float64), (self.n_slots, 1))
        self.pending = np.zeros(self.n_slots, dtype=bool)      # reset, first frame not yet rendered
        if device is None and torch.cuda.is_available():
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = device
        self._b = None

    def initial_states(self, k: int) -> np.ndarray:
        """float64 [k, 7]: ``MazeEnv.initial_states``, the start at rest."""
        s = np.zeros((int(k), 7))
        s[:, 0], s[:, 1] = self.start
        return s

    def _bufs(self):
        if self._b is None:
            if self.device is None:
                raise F.DneError("ImageMazeEnv steps on the device: no CUDA device")
            n, dev = self.n_slots, self.device
            pin = lambda t: t.pin_memory()                                    # noqa: E731
            b = dict(background=torch.empty(84, 84, dtype=torch.uint8, device=dev),
                     state=torch.zeros(n, 7, dtype=torch.float64, device=dev),
                     stack=torch.zeros(n, 84, 84, 4, dtype=torch.uint8, device=dev),
                     start=torch.from_numpy(self.initial_states(n)).to(dev),
                     d_in=torch.empty(2 * n, dtype=torch.int32, device=dev),
                     h_in=pin(torch.empty(2 * n, dtype=torch.int32)),
                     rew=torch.empty(n, dtype=torch.float32, device=dev),
                     done=torch.empty(n, dtype=torch.uint8, device=dev),
                     pos=torch.empty(n, 2, dtype=torch.float64, device=dev),
                     h_rew=pin(torch.empty(n, dtype=torch.float32)), h_done=pin(torch.empty(n, dtype=torch.uint8)),
                     h_pos=pin(torch.empty(n, 2, dtype=torch.float64)))
            F.check(F.lib().dne_image_maze_background(C.byref(self.desc), F.ptr(b["background"]), F.stream_ptr()))
            self._b = b
        return self._b

    def _flush_resets(self, slots: np.ndarray) -> None:
        """Render the first frame of the listed slots that were reset since, on the current stream."""
        todo = slots[self.pending[slots]]
        if len(todo) == 0:
            return
        b = self._bufs()
        d_slots = torch.from_numpy(todo.astype(np.int32)).to(self.device)       # pageable: staged before the call returns
        F.check(F.lib().dne_image_maze_reset(C.byref(self.desc), F.ptr(b["background"]), F.ptr(b["start"]),
                                             F.ptr(d_slots), len(todo), F.ptr(b["state"]), F.ptr(b["stack"]),
                                             F.stream_ptr()))
        self.pending[todo] = False

    def reset(self, slots):
        """Marks the slots reset; their first frames are rendered on the stream of the next ``device_obs`` / ``step`` /
        ``obs_block`` that covers them."""
        slots = np.asarray(slots, dtype=np.int64)
        self.pending[slots] = True
        self.final_xy[slots] = self.start

    def step(self, slots, actions):
        """Steps the listed slots on the current stream (one small upload, one launch, one copy back and one sync).
        ``actions``: indices into the action table.  Returns host (rewards float32 [k], done bool [k])."""
        slots = np.asarray(slots, dtype=np.int64)
        a = np.asarray(actions).astype(np.int64).reshape(-1)
        k = len(slots)
        if len(a) != k:
            raise ValueError(f"{len(a)} actions for {k} slots")
        if k == 0:
            return np.zeros(0, np.float32), np.zeros(0, bool)
        if a.min() < 0 or a.max() >= len(self.action_table):
            raise ValueError(f"action index outside 0..{len(self.action_table) - 1}")
        self._flush_resets(slots)
        b = self._bufs()
        b["h_in"][:k] = torch.from_numpy(slots.astype(np.int32))
        b["h_in"][k:2 * k] = torch.from_numpy(a.astype(np.int32))
        b["d_in"][:2 * k].copy_(b["h_in"][:2 * k], non_blocking=True)
        F.check(F.lib().dne_image_maze_step(
            C.byref(self.desc), F.ptr(b["background"]), self.action_table.ctypes.data_as(C.c_void_p),
            len(self.action_table), F.ptr(b["d_in"]), C.c_void_p(b["d_in"].data_ptr() + 4 * k), k, F.ptr(b["state"]),
            F.ptr(b["stack"]), F.ptr(b["rew"]), F.ptr(b["done"]), F.ptr(b["pos"]), F.stream_ptr()))
        b["h_rew"][:k].copy_(b["rew"][:k], non_blocking=True)
        b["h_done"][:k].copy_(b["done"][:k], non_blocking=True)
        b["h_pos"][:k].copy_(b["pos"][:k], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.final_xy[slots] = b["h_pos"][:k].numpy()
        return b["h_rew"][:k].numpy().copy(), b["h_done"][:k].numpy().astype(bool)

    def device_obs(self, lo: int, hi: int) -> torch.Tensor:
        """uint8 [hi-lo, 84, 84, 4] frame stacks of slots [lo, hi), ready on the current CUDA stream (a view: the next
        ``step`` of these slots rewrites it)."""
        self._flush_resets(np.arange(lo, hi))
        return self._bufs()["stack"][lo:hi]

    def obs_block(self, lo: int, hi: int) -> torch.Tensor:
        """A host copy of the frame stacks of slots [lo, hi) (the virtual batch norm's reference batch)."""
        return self.device_obs(lo, hi).cpu()

    def get_ram(self, slots):
        """float64 [k, 2]: the (x, y) after each slot's last step (the start after a reset)."""
        return self.final_xy[np.asarray(slots, dtype=np.int64)].copy()


def _make_image_maze(env_id, n_slots, seed=0, episode_len=None, maze_file=None, actions=None, **kw):
    if episode_len is not None:
        raise ValueError("the image maze has a fixed 400-step episode; use the episode cutoff of the config instead")
    return ImageMazeEnv(n_slots, maze_file=maze_file, seed=seed, actions=actions)


ENV_BACKENDS = {         # id prefix -> factory(env_id, n_slots, seed=, episode_len=, **kw) -> BatchEnv (real emulators plug in here)
    "CartPole-v1": _make_cartpole,
    "gym.CartPole-v1": _make_cartpole,   # the id of the reference GPU path's configurations/es_gym_config.json
    "Pendulum-v1": _make_pendulum,
    "Acrobot-v1": _make_acrobot,
    "gym.Acrobot-v1": _make_acrobot,
    "MountainCar-v0": _make_mountaincar,         # MountainCarContinuous-v0 does not match this prefix
    "gym.MountainCar-v0": _make_mountaincar,
    "maze": _make_maze,                          # gym_tensorflow.make('maze', ...) of the reference GPU path
    "ImageHardMaze-v0": _make_image_maze,        # the same maze as an 84x84 image (Such et al. 2017's Image Hard Maze)
}
