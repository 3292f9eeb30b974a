"""``es_distributed.rs`` -- the reference's random-search driver (rs.py:4-174) on the H100 engine.

Random search evaluates ``episodes_per_batch`` fresh candidates per iteration, each candidate being
``reinitialize(noise[idx])`` (rs.py:112-116 on the master, ga.py:256-260 in the workers it reuses: a GA genome of
length 1), and keeps the best-scoring one as the policy.  On the device that is the GA generation-0 path repeated:
a slot-table full of candidates is materialised with ``dne_ga_materialize(mode)`` (column-normalised noise slice) and
rolled out with one weight row per slot; nothing is perturbed (scale 0).  Multi-GPU: candidates sharded over ranks,
all_gather(returns, lengths); every rank rebuilds the same winner from its seed.
"""
from __future__ import annotations

import logging
import time

import numpy as np
import torch

from dne import shard
from dne.rollout import Unit, make_runner
from .es import SharedNoiseTable, default_context, default_noise, set_default_noise, _cutoff, reference_row   # noqa: F401
from .ga import GenomeCache, setup

logger = logging.getLogger(__name__)


def run_master(master_redis_cfg, log_dir, exp, *, max_iterations=None, n_slots=256, env=None, noise=None, seed=None,
               on_iteration=None):
    """rs.py:4-174 (the ``while True`` loop runs ``max_iterations`` times when given)."""
    from . import tabular_logger as tlogger
    rank, world = shard.dist_info()
    if rank == 0:
        tlogger.start(log_dir)
    else:
        tlogger.set_quiet(True)
    if noise is not None:
        set_default_noise(noise)
    noise = default_noise()
    ctx = default_context()
    seed = shard.broadcast_seed(seed)
    config, env, _, policy = setup(exp, single_threaded=False, n_slots=n_slots, env=env, seed=seed)
    rs = np.random.RandomState(seed)
    P = policy.num_params
    dev = policy.device
    tslimit, incr_thr, incr_ratio, _, adaptive = _cutoff(config)
    cache = GenomeCache(ctx, policy.net, config.noise_stdev, exp.get('ga_mode', 'cpu'))
    runner = make_runner(ctx, policy.net, env, n_slots=n_slots, group=1, pipeline=2 if n_slots % 2 == 0 else 1,
                         **policy.runner_head_kw())
    ob_stat = dict(ob_mean=policy.ob_mean, ob_std=policy.ob_std)            # MujocoPolicy: its fixed statistics
    chunk = torch.empty(n_slots, P, dtype=torch.float32, device=dev)
    best_score, best_seed = float('-inf'), None                   # rs.py:35
    episodes_so_far = timesteps_so_far = 0
    tstart = time.time()
    it = 0
    while max_iterations is None or it < max_iterations:
        step_tstart = time.time()
        it += 1
        if rank == 0:
            tlogger.log('********** Iteration {} **********'.format(it))
        seeds, rets, lens = [], [], []
        num_eps = num_ts = 0
        first = True
        while first or num_eps < config.episodes_per_batch or num_ts < config.timesteps_per_batch:   # rs.py:64
            n_cand = config.episodes_per_batch if first else world * n_slots
            batch = [noise.sample_index(rs, P) for _ in range(n_cand)]
            lo, hi = shard.shard_bounds(n_cand, rank, world)
            r_loc = np.zeros(hi - lo, np.float32)
            l_loc = np.zeros(hi - lo, np.int32)
            for c0 in range(lo, hi, n_slots):
                c1 = min(hi, c0 + n_slots)
                for j in range(c0, c1):
                    cache.materialize((batch[j],), chunk[j - c0])          # theta = reinitialize(noise[seed])
                units = [Unit(0, (0.0,), j - c0) for j in range(c0, c1)]
                res = runner.run(chunk, units, tslimit, **ob_stat)
                r_loc[c0 - lo:c1 - lo], l_loc[c0 - lo:c1 - lo] = res.returns[:, 0], res.lengths[:, 0]
            pack = torch.from_numpy(np.stack([r_loc, l_loc.astype(np.float32)], axis=1)).to(dev)
            allr = shard.all_gather_rows(pack, n_cand).cpu().numpy()
            seeds += batch
            rets.append(allr[:, 0].astype(np.float32))
            lens.append(allr[:, 1].astype(np.int32))
            num_eps += n_cand
            num_ts += int(allr[:, 1].sum())
            first = False
        noise_inds_n = np.asarray(seeds, dtype=np.int64)
        returns_n2 = np.concatenate(rets).reshape(-1, 1)          # rs.py:84-86: one episode per candidate
        lengths_n2 = np.concatenate(lens).reshape(-1, 1)
        episodes_so_far += lengths_n2.size
        timesteps_so_far += int(lengths_n2.sum())

        idx = int(np.argmax(returns_n2))                          # rs.py:112-116 (first max on ties)
        if returns_n2[idx, 0] > best_score:
            best_score, best_seed = float(returns_n2[idx, 0]), int(noise_inds_n[idx])
            theta = torch.empty(P, dtype=torch.float32, device=dev)
            cache.materialize((best_seed,), theta)
            policy.set_trainable_flat(theta)
        if adaptive and (lengths_n2 == tslimit).mean() >= incr_thr:                   # rs.py:118-121
            tslimit = int(incr_ratio * tslimit)
        step_tend = time.time()
        stats = dict(EpRewMax=float(returns_n2.max()), EpRewMean=float(returns_n2.mean()),
                     EpRewStd=float(returns_n2.std()), EpLenMean=float(lengths_n2.mean()),
                     Norm=float(torch.square(policy.device_theta).sum()),
                     EpisodesThisIter=int(lengths_n2.size), EpisodesSoFar=int(episodes_so_far),
                     TimestepsThisIter=int(lengths_n2.sum()), TimestepsSoFar=int(timesteps_so_far),
                     UniqueWorkers=world, TimeElapsedThisIter=step_tend - step_tstart, TimeElapsed=step_tend - tstart)
        stats = reference_row("rs", stats, world)                                      # the reference's keys, in its order
        if rank == 0:
            for k, v in stats.items():
                tlogger.record_tabular(k, v)
            tlogger.dump_tabular()
        if on_iteration is not None:
            on_iteration(it, stats, dict(noise_inds_n=noise_inds_n, returns_n2=returns_n2, lengths_n2=lengths_n2,
                                         best_score=best_score, best_seed=best_seed, theta=policy.device_theta))
        if rank == 0 and log_dir and config.snapshot_freq != 0:                       # rs.py:160-168 (every iteration)
            import os.path as osp
            policy.save(osp.join(log_dir, 'snapshot_iter{:05d}_rew{}.h5'.format(it, int(best_score))))
    return best_seed, best_score


def run_worker(master_redis_cfg, relay_redis_cfg, noise, *, min_task_runtime=.2, exp=None, **kw):
    """rs.py imports the GA worker (``from .ga import *``): a worker is a non-zero rank of the torchrun job."""
    assert isinstance(noise, SharedNoiseTable)
    if exp is None:
        raise RuntimeError("run_worker needs the experiment dict (no redis); launch every rank through "
                           "`python -m es_distributed.main master --algo rs` under torchrun")
    return run_master(master_redis_cfg, None, exp, noise=noise, **kw)
