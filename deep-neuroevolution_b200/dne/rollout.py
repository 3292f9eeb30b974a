"""Episode scheduler: runs a list of rollout units (antithetic pairs / GA offspring / eval episodes) to completion
on a fixed table of environment slots, refilling slots as episodes end, with the host environment step of one
half of the slots overlapped with the device forward of the other half.

Reference behaviour reproduced:
  * worker inner loop            es_distributed/es.py:411-426  (theta+v rollout, theta-v rollout, sums / signs / lengths)
  * Policy.rollout               es_distributed/policies.py:378-429 (reset -> ref-batch pass -> act/step until done
                                 or timestep_limit; length counts env steps)
  * slot refill                  gpu_implementation/neuroevolution/concurrent_worker.py:72-125 (running mask, per-slot
                                 cumulative reward/length, finished slots returned to the pool)
"""
from __future__ import annotations

import ctypes as C
from collections import deque
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _ffi as F
from .engine import SlotForward
from .envs import BatchEnv
from .nets import NetSpec


@dataclass
class Unit:
    """G episodes sharing one noise index (G = 2: the +/- pair of es.py:412-421; G = 1: one GA offspring)."""
    noise_idx: int
    scales: Sequence[float]
    theta_idx: int = 0
    noiseless: bool = False    # evaluation episodes (es.py:388-391): no action noise, never sampled for ob statistics


@dataclass
class RolloutResult:
    returns: np.ndarray        # float32 [n_units, G]   es.py:425
    signreturns: np.ndarray    # float32 [n_units, G]   es.py:423
    lengths: np.ndarray        # int32   [n_units, G]   es.py:426
    bcs: Optional[list] = None  # per unit, per member: behaviour characterisation (policies.py:418,429)
    steps: int = 0             # env steps executed (== lengths.sum())
    ticks: int = 0             # forward launches
    ob_sum: Optional[np.ndarray] = None     # float64 [ob_dim]: sum of the observations of the sampled episodes (es.py:358-359)
    ob_sumsq: Optional[np.ndarray] = None
    ob_count: int = 0                       # number of observations in the sums


class _Half:
    def __init__(self, ctx, net, lo, hi, n_ref):
        self.lo, self.hi = lo, hi
        n = hi - lo
        self.sf = SlotForward(ctx, net, n, n_ref=n_ref)
        dev = self.sf.device
        self.stream = torch.cuda.Stream(device=dev)
        self.event = torch.cuda.Event()
        if net.ob_kind == F.OB_ATARI_U8:
            self.obs_dev = torch.zeros(n, 84, 84, 4, dtype=torch.uint8, device=dev)
            self.act_host = torch.zeros(n, dtype=torch.int32).pin_memory()
        else:
            self.obs_dev = torch.zeros(n, net.ob_dim, dtype=torch.float32, device=dev)
            self.act_host = torch.zeros(n, net.n_out, dtype=torch.float32).pin_memory()
        self.noise_idx = np.zeros(n, dtype=np.int64)
        self.scale = np.zeros(n, dtype=np.float32)
        self.theta_idx = np.zeros(n, dtype=np.int32)
        self.active = np.zeros(n, dtype=np.uint8)
        self.unit = np.full(n, -1, dtype=np.int64)       # unit id occupying the slot
        self.member = np.zeros(n, dtype=np.int64)
        self.ret = np.zeros(n, dtype=np.float64)
        self.sret = np.zeros(n, dtype=np.float64)
        self.length = np.zeros(n, dtype=np.int64)
        self.dirty = True
        self.launched = False
        self.fresh = np.zeros(n, dtype=np.uint8)          # slots that start an episode at the next launch
        self.noiseless = np.zeros(n, dtype=bool)          # evaluation episodes: no action noise
        self.save = np.zeros(n, dtype=np.uint8)           # episode sampled for the observation statistics (es.py:356-357)
        self.save_m = 0                                   # number of slots in save_list
        self.save_list = None                             # device int32 [n]: active & sampled slots (built lazily)
        self.ob_sum = self.ob_sumsq = None                # device float64 [ob_dim] (per half: the halves run on two streams)


class RolloutRunner:
    def __init__(self, ctx: F.Context, net: NetSpec, env: BatchEnv, n_slots: int, group: int = 2, pipeline: int = 2,
                 ref_batch: Optional[torch.Tensor] = None):
        assert n_slots % (group * pipeline) == 0, "n_slots must be a multiple of group*pipeline"
        assert env.n_slots >= n_slots
        self.ctx, self.net, self.env, self.n_slots, self.G = ctx, net, env, n_slots, group
        per = n_slots // pipeline
        n_ref = int(ref_batch.shape[0]) if ref_batch is not None else 128
        self.halves = [_Half(ctx, net, i * per, (i + 1) * per, n_ref) for i in range(pipeline)]
        self.ref_batch = ref_batch
        self.use_theta_idx = False
        self.action_fn = None          # optional host map from the network's output rows to environment actions

    # ---------------------------------------------------------------------------------------------------
    def run(self, theta: torch.Tensor, units: List[Unit], timestep_limit: Optional[int] = None, *, ob_mean=None,
            ob_std=None, collect_bc: Optional[str] = None, ac_noise_std: float = 0.0,
            random_stream: Optional[np.random.RandomState] = None, save_obs_prob: float = 0.0) -> RolloutResult:
        """Evaluate every unit once.  ``collect_bc``: None | 'trace' (RAM after every step, ES Atari,
        policies.py:410,418) | 'final' (RAM / position at episode end, policies.py:510,292-299)."""
        G, env = self.G, self.env
        if collect_bc == "trace" and getattr(env, "bc_kind", "trace") != "trace":
            raise NotImplementedError(f"{type(env).__name__} has no RAM trace: its behaviour characterisation is "
                                      f"collect_bc={env.bc_kind!r}")
        n_units = len(units)
        limit = env.max_episode_steps if timestep_limit is None else \
            (timestep_limit if env.max_episode_steps is None else min(timestep_limit, env.max_episode_steps))
        assert limit is not None and limit >= 1
        res = RolloutResult(np.zeros((n_units, G), np.float32), np.zeros((n_units, G), np.float32),
                            np.zeros((n_units, G), np.int32), [[None] * G for _ in range(n_units)] if collect_bc else None)
        self.use_theta_idx = theta.dim() == 2 and theta.shape[0] > 1
        pending = deque(range(n_units))
        remaining = [G] * n_units
        want_obstat = save_obs_prob != 0.0 and self.net.ob_kind == F.OB_VECTOR
        obstat_stream = random_stream if random_stream is not None else np.random.RandomState(0)
        for h in self.halves:
            h.save[:] = 0
            h.save_m = 0
            if want_obstat:
                if h.ob_sum is None:
                    h.ob_sum = torch.zeros(self.net.ob_dim, dtype=torch.float64, device=h.sf.device)
                    h.ob_sumsq = torch.zeros_like(h.ob_sum)
                    h.save_list = torch.zeros(h.hi - h.lo, dtype=torch.int32, device=h.sf.device)
                    h.save_host = torch.zeros(h.hi - h.lo, dtype=torch.int32).pin_memory()
                h.ob_sum.zero_()
                h.ob_sumsq.zero_()
        if collect_bc == "trace":                          # per-slot RAM trace buffers, filled with vectorised writes
            for h in self.halves:
                if getattr(h, "bc_buf", None) is None or h.bc_buf.shape[1] < limit:
                    h.bc_buf = np.zeros((h.hi - h.lo, limit, 128), dtype=np.uint8)
        cur = torch.cuda.current_stream()
        for h in self.halves:
            h.unit[:] = -1
            h.active[:] = 0
            h.launched = False
            h.dirty = True
            h.stream.wait_stream(cur)

        def refill(h: _Half):
            n = h.hi - h.lo
            for u0 in range(0, n, G):
                if not pending:
                    break
                if h.unit[u0] >= 0:
                    continue
                uid = pending.popleft()
                unit = units[uid]
                for g in range(G):
                    s = u0 + g
                    h.unit[s], h.member[s] = uid, g
                    h.noise_idx[s], h.scale[s], h.theta_idx[s] = unit.noise_idx, unit.scales[g], unit.theta_idx
                    h.active[s], h.fresh[s] = 1, 1
                    h.ret[s] = h.sret[s] = 0.0
                    h.length[s] = 0
                    h.noiseless[s] = unit.noiseless
                    # es.py:356-357: each (non-evaluation) episode is sampled with probability calc_obstat_prob
                    h.save[s] = 1 if (want_obstat and not unit.noiseless and obstat_stream.rand() < save_obs_prob) else 0
                env.reset(h.lo + np.arange(u0, u0 + G))
                h.dirty = True

        def launch(h: _Half):
            # torch.cuda.set_stream pair instead of the `with torch.cuda.stream(...)` context manager: the manager's device-index
            # validation costs ~28 us per half-tick (cProfile), a quarter of the host time of a 64-slot half-table
            torch.cuda.set_stream(h.stream)
            try:
                if h.dirty:
                    h.sf.set_slots(h.noise_idx, h.scale, active=h.active,
                                   theta_idx=h.theta_idx if self.use_theta_idx else None)
                    if self.net.needs_ref_batch and h.fresh.any():
                        mask = torch.as_tensor(h.fresh).to(h.sf.device, non_blocking=True)
                        h.sf.vbn_reference_pass(theta, self.ref_batch, active=mask)     # policies.py:399
                    h.fresh[:] = 0
                    if want_obstat:                                  # slot list of the sampled episodes still running
                        loc = np.nonzero(np.logical_and(h.active, h.save))[0].astype(np.int32)
                        h.save_m = len(loc)
                        if h.save_m:
                            h.save_host[:h.save_m] = torch.from_numpy(loc)
                            h.save_list[:h.save_m].copy_(h.save_host[:h.save_m], non_blocking=True)
                    h.dirty = False
                if hasattr(env, "device_obs"):                                           # raw frames -> device preprocess (dne/raw_env.py)
                    h.obs_dev = env.device_obs(h.lo, h.hi)
                else:
                    h.obs_dev.copy_(env.obs_block(h.lo, h.hi), non_blocking=True)       # pinned -> HBM
                if want_obstat and h.save_m:                         # es.py:358-359 on the device, unnormalised observations
                    F.check(F.lib().dne_ob_stat_accumulate(F.ptr(h.obs_dev, torch.float32), self.net.ob_dim,
                                                           F.ptr(h.save_list), h.save_m, F.ptr(h.ob_sum),
                                                           F.ptr(h.ob_sumsq), F.stream_ptr()))
                    res.ob_count += h.save_m
                out = h.sf.forward(theta, h.obs_dev, paired=(G == 2), ob_mean=ob_mean, ob_std=ob_std)
                h.act_host.copy_(out, non_blocking=True)
                h.event.record(h.stream)
            finally:
                torch.cuda.set_stream(cur)
            h.launched = True
            res.ticks += 1

        def finish(h: _Half):
            h.event.synchronize()
            h.launched = False
            loc = np.nonzero(h.active)[0]
            acts = h.act_host.numpy()[loc]
            if self.action_fn is not None:                             # discretised MuJoCo heads: scores -> bin values
                acts = self.action_fn(acts)
            if ac_noise_std != 0.0 and random_stream is not None and acts.dtype != np.int32:
                noisy = ~h.noiseless[loc]                             # evaluation episodes act without noise (es.py:388-391)
                acts = acts + (random_stream.randn(*acts.shape).astype(np.float32) * np.float32(ac_noise_std)) * \
                    noisy[:, None].astype(np.float32)                 # policies.py:204-205
            rew, done = env.step(h.lo + loc, acts)
            h.ret[loc] += rew
            h.sret[loc] += np.sign(rew)
            h.length[loc] += 1
            res.steps += len(loc)
            if collect_bc == "trace":
                h.bc_buf[loc, h.length[loc] - 1] = env.get_ram(h.lo + loc)        # policies.py:410,418
            fin = loc[np.logical_or(done, h.length[loc] >= limit)]
            if len(fin):
                for s in fin:
                    uid, g = int(h.unit[s]), int(h.member[s])
                    res.returns[uid, g] = np.float32(h.ret[s])
                    res.signreturns[uid, g] = np.float32(h.sret[s])
                    res.lengths[uid, g] = h.length[s]
                    if collect_bc == "trace":
                        res.bcs[uid][g] = h.bc_buf[s, :h.length[s]].copy()
                    elif collect_bc == "final":
                        res.bcs[uid][g] = env.get_ram(np.array([h.lo + s]))[0]
                    h.active[s] = 0
                    remaining[uid] -= 1
                    if remaining[uid] == 0:
                        base = (s // G) * G
                        h.unit[base:base + G] = -1
                h.dirty = True

        for h in self.halves:
            refill(h)
            if h.active.any():
                launch(h)
        while any(h.launched for h in self.halves):
            for h in self.halves:
                if not h.launched:
                    continue
                finish(h)
                refill(h)
                if h.active.any():
                    launch(h)
            if hasattr(env, "advance"):
                env.advance()
        for h in self.halves:
            cur.wait_stream(h.stream)
        assert not pending and all(r == 0 for r in remaining)
        if want_obstat:
            res.ob_sum = sum(h.ob_sum for h in self.halves).cpu().numpy()
            res.ob_sumsq = sum(h.ob_sumsq for h in self.halves).cpu().numpy()
        return res


class EpisodeKernelRunner:
    """``RolloutRunner`` for environments whose episodes run entirely on the device (``env.device_episodes``:
    ``dne.envs.CartPoleEnv``, ``AcrobotEnv``, ``MountainCarEnv``, ``PendulumEnv``, ``MazeEnv``): every member of every unit plays its whole episode inside ONE
    launch (``env.launch_episodes``), followed by one host sync for the results.  Same ``run`` signature and
    ``RolloutResult`` as ``RolloutRunner``.

    Members are flattened in (unit, member) order; row ``u*G + g`` starts from row ``u*G + g`` of one
    ``env.initial_states(n_units*G)`` call per ``run``.  When the environment's kernel takes MujocoPolicy's inputs
    (``env.kernel_policy_io``), ``run`` also draws, from ``random_stream``: first one ``rand()`` per non-noiseless member in
    (unit, member) order against ``save_obs_prob`` (the members whose observations go into the statistics), then one
    ``randn(n_noisy, limit, adim)`` of action noise for the non-noiseless members, scaled as ``RolloutRunner`` scales it
    (adim: the action dimensions, ``net.n_out`` for a linear head).

    ``action_bins``: MujocoPolicy's float32 [adim, nb] bin table of a discretised head ('uniform:' / 'custom:'); the kernel
    then takes per dimension the bin of the highest score (numpy's argmax) and acts with its value, as ``action_fn``
    followed by ``RolloutRunner``'s noise would."""

    def __init__(self, ctx: F.Context, net: NetSpec, env: BatchEnv, n_slots: int = 0, group: int = 2, pipeline: int = 1,
                 ref_batch: Optional[torch.Tensor] = None, action_bins=None):
        assert getattr(env, "device_episodes", False), "EpisodeKernelRunner needs an environment with device episodes"
        if net.needs_ref_batch:
            raise NotImplementedError("the episode kernel runs nets without batch norm only")
        self.ctx, self.net, self.env, self.n_slots, self.G = ctx, net, env, n_slots, group
        self.device = torch.device("cuda", ctx.device)
        self.halves = (None,)          # one launch covers every member (drivers read len(halves) as tables per launch)
        self.use_theta_idx = False
        self.action_fn = None          # accepted for interface parity; the kernel's head is the environment's action
        self.action_bins = None
        if action_bins is not None:
            if not env.kernel_policy_io:
                raise NotImplementedError(f"{type(env).__name__}'s episode kernel has no discretised heads")
            tab = np.ascontiguousarray(action_bins, dtype=np.float32)
            if tab.ndim != 2 or tab.shape[0] * tab.shape[1] != net.n_out:
                raise ValueError(f"action_bins {tab.shape} do not match the net's {net.n_out} outputs (adim * n_bins)")
            self.action_bins = tab

    def run(self, theta: torch.Tensor, units: List[Unit], timestep_limit: Optional[int] = None, *, ob_mean=None,
            ob_std=None, collect_bc: Optional[str] = None, ac_noise_std: float = 0.0,
            random_stream: Optional[np.random.RandomState] = None, save_obs_prob: float = 0.0) -> RolloutResult:
        """Evaluate every unit once.  ``collect_bc``: None | 'final' (float64 [env.bc_dim]: the leading components of the
        state after the last step; ``bc_dim`` defaults to ``env.state_dim``)."""
        G, env = self.G, self.env
        if not env.kernel_policy_io:
            if ob_mean is not None or ob_std is not None:
                raise NotImplementedError("the episode kernel does not normalise observations")
        if collect_bc not in (None, "final"):
            raise NotImplementedError(f"collect_bc={collect_bc!r}: the episode kernel records the final state only")
        if not env.kernel_policy_io:
            if save_obs_prob != 0.0:
                raise NotImplementedError("the episode kernel does not sample observation statistics")
            if ac_noise_std != 0.0:
                raise NotImplementedError("the episode kernel acts without action noise")
        n_units = len(units)
        n = n_units * G
        limit = env.max_episode_steps if timestep_limit is None else min(timestep_limit, env.max_episode_steps)
        assert limit is not None and limit >= 1
        res = RolloutResult(np.zeros((n_units, G), np.float32), np.zeros((n_units, G), np.float32),
                            np.zeros((n_units, G), np.int32), [[None] * G for _ in range(n_units)] if collect_bc else None)
        self.use_theta_idx = theta.dim() == 2 and theta.shape[0] > 1
        want_obstat = save_obs_prob != 0.0 and self.net.ob_kind == F.OB_VECTOR
        if want_obstat:
            res.ob_sum = np.zeros(self.net.ob_dim)
            res.ob_sumsq = np.zeros(self.net.ob_dim)
        if n == 0:
            return res
        noise_idx = np.repeat(np.array([u.noise_idx for u in units], dtype=np.int64), G)
        scale = np.array([u.scales[g] for u in units for g in range(G)], dtype=np.float32)
        init = env.initial_states(n)
        dev = self.device
        extra = {}
        if env.kernel_policy_io:
            noisy = ~np.repeat(np.array([u.noiseless for u in units], dtype=bool), G)
            if want_obstat:                   # es.py:356-357, drawn in RolloutRunner's order (before any action noise)
                stream = random_stream if random_stream is not None else np.random.RandomState(0)
                save = np.zeros(n, dtype=bool)
                save[noisy] = stream.rand(int(noisy.sum())) < save_obs_prob     # = one rand() per member, in order
                extra["d_ob_sum"] = torch.empty(n, self.net.ob_dim, dtype=torch.float64, device=dev)
                extra["d_ob_sumsq"] = torch.empty_like(extra["d_ob_sum"])
            if ac_noise_std != 0.0 and random_stream is not None:          # policies.py:204-205, RolloutRunner.finish
                adim = self.net.n_out if self.action_bins is None else self.action_bins.shape[0]
                ac = np.zeros((n, int(limit), adim), dtype=np.float32)
                ac[noisy] = random_stream.randn(int(noisy.sum()), int(limit), adim).astype(np.float32) * \
                    np.float32(ac_noise_std)
                extra["d_ac_noise"] = torch.from_numpy(ac).to(dev)
            if self.action_bins is not None:
                extra["action_bins"] = self.action_bins
            if ob_mean is not None:
                extra["d_ob_mean"] = ob_mean.to(dev, torch.float32).contiguous()
                extra["d_ob_std"] = ob_std.to(dev, torch.float32).contiguous()
        d_idx = torch.from_numpy(noise_idx).to(dev)
        d_scale = torch.from_numpy(scale).to(dev)
        d_row = torch.from_numpy(np.repeat(np.array([u.theta_idx for u in units], dtype=np.int32), G)).to(dev) \
            if self.use_theta_idx else None
        sd = env.state_dim
        d_init = torch.from_numpy(np.ascontiguousarray(init, dtype=np.float64)).to(dev)
        d_ret = torch.empty(n, dtype=torch.float32, device=dev)
        d_sret = torch.empty(n, dtype=torch.float32, device=dev)
        d_len = torch.empty(n, dtype=torch.int32, device=dev)
        d_fin = torch.empty(n, sd, dtype=torch.float64, device=dev) if collect_bc == "final" else None
        theta = theta.contiguous()
        env.launch_episodes(self.ctx, self.net, theta, d_idx, d_scale, d_row, n, d_init, limit, d_ret, d_sret, d_len,
                            d_fin, **extra)
        outs = {"ret": d_ret, "sret": d_sret, "len": d_len, "fin": d_fin,
                "ob_sum": extra.get("d_ob_sum"), "ob_sumsq": extra.get("d_ob_sumsq")}
        host = {}
        for k, d in outs.items():
            if d is not None:
                host[k] = torch.empty(d.shape, dtype=d.dtype, pin_memory=True)
                host[k].copy_(d, non_blocking=True)
        torch.cuda.current_stream().synchronize()                 # the one host sync of the run
        res.returns[:] = host["ret"].numpy().reshape(n_units, G)
        res.signreturns[:] = host["sret"].numpy().reshape(n_units, G)
        res.lengths[:] = host["len"].numpy().reshape(n_units, G)
        res.steps = int(res.lengths.sum())
        res.ticks = 1
        if d_fin is not None:
            fin = host["fin"].numpy().reshape(n_units, G, sd)
            bd = getattr(env, "bc_dim", sd)
            res.bcs = [[fin[u, g, :bd].copy() for g in range(G)] for u in range(n_units)]
        if want_obstat:                       # the flagged members' sums, added in member order
            s_, q_ = host["ob_sum"].numpy(), host["ob_sumsq"].numpy()
            for m in np.nonzero(save)[0]:
                res.ob_sum += s_[m]
                res.ob_sumsq += q_[m]
            res.ob_count = int(res.lengths.ravel()[save].sum())
        return res


def make_runner(ctx: F.Context, net: NetSpec, env: BatchEnv, action_fn=None, action_bins=None, **kw):
    """The rollout runner for ``env``: ``EpisodeKernelRunner`` when its episodes run on the device
    (``env.device_episodes``), the environment's kernel takes ``net`` (``env.episode_net_supported``) and no host
    ``action_fn`` maps the network's output to actions; otherwise the per-tick ``RolloutRunner`` when the environment
    has a host step.  ``action_fn``: the policy's map from output rows to actions (discretised MuJoCo heads), None for
    the identity; an environment without a host step refuses one unless ``action_bins`` comes with it.
    ``action_bins``: the bin table [adim, nb] behind a discretised ``action_fn`` (MujocoPolicy's ``_bin_values``); an
    environment without a host step (the maze) then runs the head in its episode kernel (``EpisodeKernelRunner``), one
    with a host step keeps the per-tick runner with ``action_fn``.  ``kw`` are ``RolloutRunner``'s arguments."""
    device = getattr(env, "device_episodes", False)
    if action_bins is not None:
        if action_fn is None:
            raise ValueError("action_bins comes with the policy's action_fn (the host map of the same head)")
        if device and not env.host_step:
            r = EpisodeKernelRunner(ctx, net, env, action_bins=action_bins, **kw)
            r.action_fn = action_fn
            return r
    if device and action_fn is not None and not env.host_step:
        raise NotImplementedError(f"{type(env).__name__} runs only on its episode kernel, whose head is the action: a "
                                  "discretised ('uniform:' / 'custom:') head runs there only with its bin table "
                                  "(action_bins); otherwise use 'continuous:'")
    if device and ((action_fn is None and env.episode_net_supported(net)) or not env.host_step):
        r = EpisodeKernelRunner(ctx, net, env, **kw)
    else:
        r = RolloutRunner(ctx, net, env, **kw)
    r.action_fn = action_fn
    return r
