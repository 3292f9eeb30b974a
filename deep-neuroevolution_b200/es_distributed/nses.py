"""``es_distributed.nses`` -- NS-ES / NSR-ES (nses.py:12-39,58-316,318-400) on the H100 engine.

Kept semantics: a meta-population of ``novelty_search.population_size`` (theta, optimizer) pairs (nses.py:95-117), an
archive of behaviour characterisations seeded with each member's mean BC (:113-114); every iteration runs one ES
generation on ``theta_dict[curr_parent]`` where each rollout's NOVELTY (mean distance to its k nearest archive
entries, nses.py:22-32) replaces the sign-return slot (:381-384); with ``return_proc_mode = centered_sign_rank`` the
master ranks novelty (:221-222) and NSR averages reward ranks and novelty ranks (:226-228); after the step the new
theta's mean BC is appended (:246-247); the next parent is drawn with probability proportional to novelty (:293-302)
or round-robin (:303-304).

Device design: BCs are RAM traces [t, 128] uint8 (policies.py:410,418), kept last-row padded to the longest episode
of the batch; novelty = dne_knn_novelty (exact integer distances, float64 sqrt) against the archive resident in HBM.
Only ``num_rollouts == 1`` is supported (the reference's ``np.mean`` over ragged traces only works for equal
lengths anyway; configurations/frostbite_ns*.json use 1).
"""
from __future__ import annotations

import ctypes as C
import logging
import time

import numpy as np
import torch

from dne import _ffi as F
from dne import shard
from dne.rollout import Unit, make_runner
from .es import (Config, Result, Task, RunningStat, SharedNoiseTable, default_context, default_noise,   # noqa: F401
                 set_default_noise, setup as _es_setup, _cutoff, _process_returns, get_ref_batch, reference_row)

logger = logging.getLogger(__name__)


class BCArchive:
    """Archive of behaviour characterisations in HBM.  ``kind='trace'``: uint8 RAM sequences [t, 128] (ES Atari,
    policies.py:410,418), last-row padded to a common t_max, with true lengths.  ``kind='vector'``: float64 vectors of one
    length (MujocoPolicy final (x, y) position, policies.py:292-299)."""

    def __init__(self, device, D=128, kind="trace"):
        self.device, self.D, self.kind = device, D, kind
        self.seqs = []                      # host copies (np.uint8 [t, D] / np.float64 [D])
        self._dev = self._len = None
        self._tmax = 0

    def append(self, bc: np.ndarray):
        if self.kind == "vector":
            bc = np.ascontiguousarray(bc, dtype=np.float64).reshape(-1)
            self.D = bc.size
            self.seqs.append(bc)
        else:
            self.seqs.append(np.ascontiguousarray(bc, dtype=np.uint8))
        self._dev = None

    def __len__(self):
        return len(self.seqs)

    @staticmethod
    def pad(seqs, t_max):
        out = np.empty((len(seqs), t_max, seqs[0].shape[1]), dtype=np.uint8)
        for i, s in enumerate(seqs):
            out[i, :len(s)] = s
            out[i, len(s):] = s[-1]
        return out

    def device_view(self, t_max):
        if self._dev is None or self._tmax != t_max:
            self._dev = torch.from_numpy(self.pad(self.seqs, t_max)).to(self.device)
            self._len = torch.tensor([len(s) for s in self.seqs], dtype=torch.int32, device=self.device)
            self._tmax = t_max
        return self._dev, self._len


def compute_novelty_vs_archive(archive: BCArchive, bcs, k: int) -> np.ndarray:
    """nses.py:22-32 for a batch of BC sequences (device k-NN)."""
    dev = archive.device
    if len(bcs) == 0:                       # a rank whose shard of the population is empty (n_pairs < world)
        return np.zeros(0, dtype=np.float32)
    if archive.kind == "vector":
        q, A, D = len(bcs), len(archive), archive.D
        d_bc = torch.from_numpy(np.stack([np.asarray(b, dtype=np.float64).reshape(-1) for b in bcs])).to(dev)
        if archive._dev is None:
            archive._dev = torch.from_numpy(np.stack(archive.seqs)).to(dev)
        nb = C.c_size_t()
        F.check(F.lib().dne_knn_ws_bytes(q, A, C.byref(nb)))
        ws = torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)
        nov = torch.empty(q, dtype=torch.float32, device=dev)
        F.check(F.lib().dne_knn_novelty_vec(F.ptr(d_bc), q, F.ptr(archive._dev), A, D, int(k), F.ptr(nov), F.ptr(ws),
                                            ws.numel(), F.stream_ptr()))
        return nov.cpu().numpy()
    t_max = max(max(len(b) for b in bcs), max(len(s) for s in archive.seqs))
    d_arch, d_alen = archive.device_view(t_max)
    q = len(bcs)
    d_bc = torch.from_numpy(BCArchive.pad(bcs, t_max)).to(dev)
    d_len = torch.tensor([len(b) for b in bcs], dtype=torch.int32, device=dev)
    nb = C.c_size_t()
    F.check(F.lib().dne_knn_ws_bytes(q, len(archive), C.byref(nb)))
    ws = torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)
    nov = torch.empty(q, dtype=torch.float32, device=dev)
    F.check(F.lib().dne_knn_novelty(F.ptr(d_bc), F.ptr(d_len), q, F.ptr(d_arch), F.ptr(d_alen), len(archive), t_max,
                                    archive.D, int(k), F.ptr(nov), F.ptr(ws), ws.numel(), F.stream_ptr()))
    return nov.cpu().numpy()


def choose_bc_mode(env, net) -> str:
    """The behaviour characterisation ``runner.run(collect_bc=...)`` records: the environment's ``bc_kind`` when it sets
    one (``ImageMazeEnv``: 'final', the final (x, y) behind Atari-shaped observations), otherwise per policy family: the
    RAM trace for the Atari policies (policies.py:410,418), the final (x, y) position for MujocoPolicy
    (policies.py:292-299, bc_choice default)."""
    return getattr(env, "bc_kind", None) or ("final" if net.ob_kind == F.OB_VECTOR else "trace")


def run_master(master_redis_cfg, log_dir, exp, *, max_iterations=None, n_slots=256, env=None, noise=None, seed=None,
               on_iteration=None):
    """nses.py:58-316."""
    from .optimizers import SGD, Adam
    from . import tabular_logger as tlogger
    rank, world = shard.dist_info()
    # Multi-GPU (SURVEY 8e): rollout units sharded over the ranks; every rank scores its own BCs against the (replicated)
    # archive and the ranks all_gather (returns, lengths, novelty) -- a few floats per pair instead of the BC traces --
    # then the ES collectives (partial gradient with the global denominator, one all_reduce).  Everything that feeds the
    # archive or the parent choice comes from rank 0 (broadcast), so the replicas cannot drift apart.
    # world == 1 executes exactly the single-GPU statements; tests/test_gpu_multi.py runs world 2 against world 1 on NCCL.
    if rank == 0:
        tlogger.start(log_dir)
    else:
        tlogger.set_quiet(True)
    if noise is not None:
        set_default_noise(noise)
    noise = default_noise()
    ctx = default_context()
    seed = shard.broadcast_seed(seed)
    rs = np.random.RandomState(seed)
    algo_type = exp['algo_type']
    ns = exp['novelty_search']
    pop_size, num_rollouts, k = int(ns['population_size']), int(ns['num_rollouts']), int(ns['k'])
    assert num_rollouts == 1, "only num_rollouts == 1 (see module docstring)"
    config, env, _, policy = _es_setup(exp, single_threaded=False, n_slots=n_slots, env=env, seed=seed)
    P = policy.num_params
    dev = policy.device
    tslimit, incr_thr, incr_ratio, tslimit_max, adaptive = _cutoff(config)
    if policy.needs_ref_batch:
        policy.set_ref_batch(get_ref_batch(env, batch_size=128, rs=np.random.RandomState(seed)))
    runner = make_runner(ctx, policy.net, env, n_slots=n_slots, group=2, pipeline=2 if n_slots % 4 == 0 else 1,
                         ref_batch=policy.ref_batch, **policy.runner_head_kw())
    bc_mode = choose_bc_mode(env, policy.net)
    vector_bc = bc_mode == "final"
    archive = BCArchive(dev, kind="vector" if vector_bc else "trace")
    ob_stat = RunningStat(env.observation_space.shape, eps=1e-2) if policy.needs_ob_stat else None      # nses.py:72-75
    ob_count_this_batch = 0

    def ob_norm():
        if ob_stat is None:
            return None, None
        policy.set_ob_stat(ob_stat.mean, ob_stat.std)
        return policy.ob_mean, policy.ob_std

    def mean_bc(theta):                                    # nses.py:34-39 (one noiseless rollout)
        om, osd = ob_norm()
        res = runner.run(theta, [Unit(0, (0.0, 0.0), noiseless=True)], tslimit_max, collect_bc=bc_mode, ob_mean=om, ob_std=osd)
        return res.bcs[0][0]

    theta_dict, optimizer_dict = {}, {}
    for p in range(pop_size):                              # nses.py:95-117: independent initialisations
        pol_p = type(policy)(env.observation_space, env.action_space, **exp['policy']['args'], seed=seed + 1 + p, ctx=ctx)
        opt = {'sgd': SGD, 'adam': Adam}[exp['optimizer']['type']](pol_p.get_trainable_flat(), ctx=ctx,
                                                                   **exp['optimizer']['args'])
        theta_dict[p], optimizer_dict[p] = opt.device_theta, opt
        archive.append(shard.broadcast_object(mean_bc(opt.device_theta)))

    curr_parent = 0
    episodes_so_far = timesteps_so_far = 0
    tstart = time.time()
    it = 0
    while max_iterations is None or it < max_iterations:
        step_tstart = time.time()
        it += 1
        optimizer = optimizer_dict[curr_parent]
        upd = optimizer._upd
        n_pairs = -(-config.episodes_per_batch // 2)
        idx = np.array([noise.sample_index(rs, P) for _ in range(n_pairs)], dtype=np.int64)
        sig = np.float32(config.noise_stdev)
        units = [Unit(int(i), (sig, -sig)) for i in idx]
        lo, hi = shard.shard_bounds(n_pairs, rank, world)
        om, osd = ob_norm()
        res = runner.run(optimizer.device_theta, units[lo:hi], tslimit, collect_bc=bc_mode, ob_mean=om, ob_std=osd,
                         ac_noise_std=getattr(policy, "ac_noise_std", 0.0),
                         random_stream=np.random.RandomState((seed + 1000 * it + rank) % (2 ** 31)),
                         save_obs_prob=config.calc_obstat_prob if ob_stat is not None else 0.0)
        if ob_stat is not None and config.calc_obstat_prob != 0:                                         # nses.py:196-199
            t = torch.from_numpy(np.concatenate([res.ob_sum, res.ob_sumsq, [float(res.ob_count)]])).to(dev)
            shard.all_reduce_sum_(t)
            tot = t.cpu().numpy()
            Dd = (len(tot) - 1) // 2
            ob_count_this_batch = int(round(tot[-1]))
            if ob_count_this_batch > 0:
                shp = ob_stat.sum.shape
                ob_stat.increment(tot[:Dd].astype(np.float32).reshape(shp), tot[Dd:2 * Dd].astype(np.float32).reshape(shp),
                                  ob_count_this_batch)
        bcs = [res.bcs[u][g] for u in range(hi - lo) for g in range(2)]
        novelty_n2 = compute_novelty_vs_archive(archive, bcs, k).reshape(hi - lo, 2).astype(np.float32)   # nses.py:381-384
        returns_n2, lengths_n2 = res.returns, res.lengths
        if world > 1:
            pack = torch.from_numpy(np.concatenate([returns_n2, lengths_n2.astype(np.float32), novelty_n2], axis=1)).to(dev)
            allr = shard.all_gather_rows(pack, n_pairs).cpu().numpy()
            returns_n2, lengths_n2 = allr[:, 0:2].astype(np.float32), allr[:, 2:4].astype(np.int32)
            novelty_n2 = allr[:, 4:6].astype(np.float32)
        proc = _process_returns(config, upd, torch.from_numpy(returns_n2).to(dev), torch.from_numpy(novelty_n2).to(dev))
        if algo_type == "nsr":                                                                         # nses.py:226-228
            rew_ranks = upd.centered_ranks(torch.from_numpy(returns_n2).to(dev))[0]
            proc = (rew_ranks + proc) / 2.0
        g = upd.gradient(proc[lo:hi].contiguous(), torch.from_numpy(idx[lo:hi]).to(dev), denom=returns_n2.size)
        shard.all_reduce_sum_(g)
        update_ratio, _ = optimizer.update_from_gradient(g, config.l2coeff)
        archive.append(shard.broadcast_object(mean_bc(optimizer.device_theta)))                        # nses.py:246-247
        if adaptive and (lengths_n2 == tslimit).mean() >= incr_thr:
            tslimit = min(int(incr_ratio * tslimit), tslimit_max)
        episodes_so_far += lengths_n2.size
        timesteps_so_far += int(lengths_n2.sum())
        stats = dict(ParentId=curr_parent, EpRewMean=float(returns_n2.mean()), EpRewStd=float(returns_n2.std()),
                     EpLenMean=float(lengths_n2.mean()), NoveltyMean=float(novelty_n2.mean()),
                     Norm=float(torch.square(optimizer.device_theta).sum()), GradNorm=float(torch.square(g).sum()),
                     UpdateRatio=float(update_ratio), EpisodesThisIter=int(lengths_n2.size),
                     EpisodesSoFar=int(episodes_so_far), TimestepsThisIter=int(lengths_n2.sum()),
                     TimestepsSoFar=int(timesteps_so_far), ObCount=int(ob_count_this_batch), ArchiveSize=len(archive),
                     TimeElapsedThisIter=time.time() - step_tstart, TimeElapsed=time.time() - tstart)
        stats = reference_row("nses", stats, world)                                    # the reference's keys, in its order
        if rank == 0:
            for kk, v in stats.items():
                tlogger.record_tabular(kk, v)
            tlogger.dump_tabular()
        if on_iteration is not None:
            on_iteration(it, stats, dict(noise_inds_n=idx, returns_n2=returns_n2, novelty_n2=novelty_n2, g=g, bcs=bcs,
                                         archive=archive, parent=curr_parent, theta=optimizer.device_theta))
        # ---- next parent (nses.py:293-306) ----
        if ns['selection_method'] == "novelty_prob":
            nov = compute_novelty_vs_archive(archive, [mean_bc(theta_dict[p]) for p in range(pop_size)], k).astype(np.float64)
            probs = nov / float(nov.sum()) if nov.sum() > 0 else np.full(pop_size, 1.0 / pop_size)
            curr_parent = int(shard.broadcast_object(int(rs.choice(range(pop_size), 1, p=probs)[0])))
        elif ns['selection_method'] == "round_robin":
            curr_parent = (curr_parent + 1) % pop_size
        else:
            raise NotImplementedError(ns['selection_method'])
    return theta_dict, archive


def run_worker(master_redis_cfg, relay_redis_cfg, noise, *, min_task_runtime=.2, exp=None, **kw):
    """nses.py:318-400: workers are the ranks of the torchrun job (see es.run_worker)."""
    assert isinstance(noise, SharedNoiseTable)
    if exp is None:
        raise RuntimeError("run_worker needs the experiment dict (no redis)")
    return run_master(master_redis_cfg, None, exp, noise=noise, **kw)
