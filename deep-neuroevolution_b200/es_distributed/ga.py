"""``es_distributed.ga`` -- the reference's GA driver (ga.py:4,33-206,209-284) on the H100 engine, plus the GPU path's
Deep GA options (gpu_implementation/ga.py:123-129,165-204,260-271; configurations/ga_atari_config.json).

Genomes are seed chains (ga.py:252-254): ``[idx0, idx1, ...]``; weights = reinitialize(noise[idx0]) + sigma * sum
noise[idx_k] (ga.py:256-264).  Device design:
  * the ``population_size`` parents' weights are CACHED in HBM ([T, P] floats; 324 MB for T = 20 LargeModels) and an
    offspring is evaluated as  theta[parent] + sigma * noise[new seed]  straight from the slot table -- never
    materialised (the reference GPU path caches parents the same way, models/base.py:127-139);
  * generation 0 (no parents) materialises one chunk of offspring at a time with dne_ga_materialize;
  * selection = dne_ga_truncate (stable descending; ga.py:145-149), elites first (ga.py:136-137);
  * multi-GPU: offspring sharded over ranks, all_gather(fitness); genomes are rebuilt identically on every rank.
Two genome flavours: ``exp['ga_mode'] = 'cpu'`` (default, ga.py: column-normalised init) or ``'gpu'``
(models/base.py:140-146: scale_by init, per-mutation power).
"""
from __future__ import annotations

import ctypes as C
import logging
import time
from collections import namedtuple

import numpy as np
import torch

from dne import _ffi as F
from dne import shard
from dne.rollout import Unit, make_runner
from .es import (Config, Result, Task, RunningStat, SharedNoiseTable, default_context, default_noise,   # noqa: F401
                 set_default_noise, setup as _es_setup, _cutoff, reference_row)

logger = logging.getLogger(__name__)

GATask = namedtuple('GATask', ['params', 'population', 'ob_mean', 'ob_std', 'timestep_limit'])


def setup(exp, single_threaded, n_slots=256, env=None, seed=None):
    """ga.py:7-20."""
    return _es_setup(exp, single_threaded, n_slots=n_slots, env=env, seed=seed)


class GenomeCache:
    """Device cache of materialised parents."""

    def __init__(self, ctx, net, sigma, mode):
        self.ctx, self.net, self.sigma, self.mode = ctx, net, float(sigma), 1 if mode == "cpu" else 0
        self.dev = torch.device("cuda", ctx.device)
        self.std = (C.c_double * len(net.layers))(*net.init_std())
        self.seeds = []                       # list of tuples
        self.theta = None                     # [n, P]

    def materialize(self, seeds, out: torch.Tensor):
        """Full rebuild of one genome into ``out`` (ga.py:256-264 / models/base.py:140-146)."""
        s = torch.tensor(list(seeds), dtype=torch.int64, device=self.dev)
        p = torch.full((len(seeds),), self.sigma, dtype=torch.float32, device=self.dev)
        F.check(F.lib().dne_ga_materialize(self.ctx.handle, C.byref(self.net.desc), F.ptr(s), F.ptr(p), len(seeds),
                                           self.std, self.mode, F.ptr(out), F.stream_ptr()))

    def rebuild(self, new_seeds):
        """New parent set.  A genome already cached is copied; parent+one seed is one mutation of the cached parent
        (the floating-point order is the chain order, identical to a full rebuild); anything else is rebuilt."""
        P = self.net.num_params
        new_theta = torch.empty(len(new_seeds), P, dtype=torch.float32, device=self.dev)
        index = {s: i for i, s in enumerate(self.seeds)}
        for j, s in enumerate(new_seeds):
            s = tuple(s)
            if s in index:
                new_theta[j].copy_(self.theta[index[s]])
            elif len(s) > 1 and s[:-1] in index:
                F.check(F.lib().dne_ga_mutate(self.ctx.handle, F.ptr(self.theta[index[s[:-1]]]), int(s[-1]),
                                              self.sigma, P, F.ptr(new_theta[j]), F.stream_ptr()))
            else:
                self.materialize(s, new_theta[j])
        self.theta, self.seeds = new_theta, [tuple(s) for s in new_seeds]


def run_master(master_redis_cfg, log_dir, exp, *, max_iterations=None, n_slots=256, env=None, noise=None, seed=None,
               on_iteration=None):
    """ga.py:33-206."""
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
    # two selection schemes: the CPU driver's (ga.py:135-158: num_elites + top population_size) and, when the experiment
    # carries the GPU path's keys (configurations/ga_atari_config.json: selection_threshold, validation_threshold,
    # num_validation_episodes), Deep GA with a validation stage (gpu_implementation/ga.py:180-204,260-271)
    deep = 'validation_threshold' in exp
    population_size = exp['selection_threshold'] if deep else exp['population_size']          # ga.py:66
    num_elites = 0 if deep else exp['num_elites']                                              # ga.py:67
    elite = None
    deep_stats, deep_extra = {}, {}
    cache = GenomeCache(ctx, policy.net, config.noise_stdev, exp.get('ga_mode', 'cpu'))
    runner = make_runner(ctx, policy.net, env, n_slots=n_slots, group=1, pipeline=2 if n_slots % 2 == 0 else 1,
                         **policy.runner_head_kw())
    ob_stat = dict(ob_mean=policy.ob_mean, ob_std=policy.ob_std)            # MujocoPolicy: its fixed statistics
    population, population_score = [], np.array([], dtype=np.float32)
    episodes_so_far = timesteps_so_far = 0
    tstart = time.time()
    it = 0
    while max_iterations is None or it < max_iterations:
        step_tstart = time.time()
        it += 1
        if rank == 0:
            tlogger.log('********** Iteration {} **********'.format(it))
        genomes, rets, lens = [], [], []
        num_eps = num_ts = 0
        first = True
        while first or (not deep and (num_eps < config.episodes_per_batch or num_ts < config.timesteps_per_batch)):   # ga.py:94
            # offspring per generation: the CPU driver's episode quota (ga.py:94), or exactly population_size on the
            # GPU path (gpu_implementation/ga.py:165-166)
            n_off = (exp['population_size'] if deep else config.episodes_per_batch) if first else world * n_slots
            parents = [int(rs.randint(len(population))) if len(population) > 0 else -1 for _ in range(n_off)]   # ga.py:251-254
            new_seeds = [noise.sample_index(rs, P) for _ in range(n_off)]
            batch = [(tuple(population[p]) if p >= 0 else ()) + (s,) for p, s in zip(parents, new_seeds)]
            lo, hi = shard.shard_bounds(n_off, rank, world)
            r_loc = np.zeros(hi - lo, np.float32)
            l_loc = np.zeros(hi - lo, np.int32)
            if len(population) > 0:
                units = [Unit(new_seeds[i], (np.float32(config.noise_stdev),), parents[i]) for i in range(lo, hi)]
                res = runner.run(cache.theta, units, tslimit, **ob_stat)
                r_loc[:], l_loc[:] = res.returns[:, 0], res.lengths[:, 0]
            else:
                # generation 0: theta = reinitialize(noise[seed]) per offspring, a slot-table full at a time
                chunk = torch.empty(n_slots, P, dtype=torch.float32, device=dev)
                for c0 in range(lo, hi, n_slots):
                    c1 = min(hi, c0 + n_slots)
                    for j in range(c0, c1):
                        cache.materialize(batch[j], chunk[j - c0])
                    units = [Unit(0, (0.0,), j - c0) for j in range(c0, c1)]
                    res = runner.run(chunk, units, tslimit, **ob_stat)
                    r_loc[c0 - lo:c1 - lo], l_loc[c0 - lo:c1 - lo] = res.returns[:, 0], res.lengths[:, 0]
            pack = torch.from_numpy(np.stack([r_loc, l_loc.astype(np.float32)], axis=1)).to(dev)
            allr = shard.all_gather_rows(pack, n_off).cpu().numpy()
            genomes += batch
            rets.append(allr[:, 0].astype(np.float32))
            lens.append(allr[:, 1].astype(np.int32))
            num_eps += n_off
            num_ts += int(allr[:, 1].sum())
            first = False
        returns = np.concatenate(rets)
        lengths_n2 = np.concatenate(lens)
        episodes_so_far += len(returns)
        timesteps_so_far += int(lengths_n2.sum())

        if deep:
            # ---- Deep GA of the GPU path (gpu_implementation/ga.py:180-204,260-271): stable descending sort, the top
            # validation_threshold (+ last elite) re-evaluated num_validation_episodes times, elite = argmax of the mean
            # validation return, parents = top selection_threshold with the elite forced in ----
            d_fit = torch.from_numpy(returns.astype(np.float32)).to(dev)
            order_t = torch.empty(len(returns), dtype=torch.int32, device=dev)
            F.check(F.lib().dne_ga_truncate(F.ptr(d_fit), len(returns), len(returns), F.ptr(order_t), F.stream_ptr()))   # ga.py:180
            order = order_t.cpu().numpy()
            pop_sorted = [tuple(genomes[i]) for i in order]
            V, n_val = int(exp['validation_threshold']), int(exp['num_validation_episodes'])
            val_pop = pop_sorted[:V]
            if elite is not None:
                val_pop = [elite] + val_pop[:-1]                                            # ga.py:186-188
            val_theta = torch.empty(len(val_pop), P, dtype=torch.float32, device=dev)
            index = {sd: i for i, sd in enumerate(cache.seeds)}
            for j, gnm in enumerate(val_pop):                                               # compute_weights_from_seeds(cache=parents)
                if gnm in index:
                    val_theta[j].copy_(cache.theta[index[gnm]])
                elif len(gnm) > 1 and gnm[:-1] in index:
                    F.check(F.lib().dne_ga_mutate(ctx.handle, F.ptr(cache.theta[index[gnm[:-1]]]), int(gnm[-1]), cache.sigma, P,
                                                  F.ptr(val_theta[j]), F.stream_ptr()))
                else:
                    cache.materialize(gnm, val_theta[j])
            v_units = [Unit(0, (0.0,), j) for j in range(len(val_pop)) for _ in range(n_val)]
            vlo, vhi = shard.shard_bounds(len(v_units), rank, world)
            vres = runner.run(val_theta, v_units[vlo:vhi], tslimit, **ob_stat)
            vpack = torch.from_numpy(np.stack([vres.returns[:, 0], vres.lengths[:, 0].astype(np.float32)], axis=1)).to(dev)
            vall = shard.all_gather_rows(vpack, len(v_units)).cpu().numpy()
            val_returns = vall[:, 0].reshape(len(val_pop), n_val)
            val_means = val_returns.mean(axis=1)
            elite_idx = int(np.argmax(val_means))                                           # ga.py:197
            elite = val_pop[elite_idx]
            Tsel = int(exp['selection_threshold'])
            top = pop_sorted[:Tsel]
            population = top if elite in top else [elite] + top[:Tsel - 1]                  # ga.py:260-271
            score_of = {tuple(genomes[i]): float(returns[i]) for i in order[::-1]}
            population_score = np.array([score_of.get(g, float(val_means[elite_idx])) for g in population], dtype=np.float32)
            timesteps_so_far += int(vall[:, 1].sum())
            cache.rebuild(population)
            policy.set_trainable_flat(cache.theta[population.index(elite)])
            deep_stats = dict(TruncatedPopulationRewMean=float(np.mean([score_of.get(g, np.nan) for g in val_pop])),
                              TruncatedPopulationValidationRewMean=float(val_means.mean()),
                              TruncatedPopulationEliteValidationRewMean=float(val_means.max()),
                              TruncatedPopulationEliteIndex=elite_idx, ValidationTimestepsThisIter=int(vall[:, 1].sum()))
            deep_extra = dict(val_pop=val_pop, val_returns=val_returns, elite=elite, pop_sorted=pop_sorted)
        if not deep:
            # ---- selection (ga.py:135-149): elites first, then this generation's offspring ----
            cand = [tuple(g) for g in population[:num_elites]] + genomes
            fit = np.concatenate([population_score[:num_elites], returns]).astype(np.float32)
            T = min(population_size, len(cand))
            d_fit = torch.from_numpy(fit).to(dev)
            sel = torch.empty(T, dtype=torch.int32, device=dev)
            F.check(F.lib().dne_ga_truncate(F.ptr(d_fit), len(fit), T, F.ptr(sel), F.stream_ptr()))
            sel = sel.cpu().numpy()
            population = [cand[i] for i in sel]
            population_score = fit[sel]
            assert len(population) == T and np.max(fit) == population_score[0]            # ga.py:148-149
            cache.rebuild(population)                                                     # parents for the next generation
            policy.set_trainable_flat(cache.theta[0])                                     # elite (ga.py:151-158)

        if adaptive and (lengths_n2 == tslimit).mean() >= incr_thr:                   # ga.py:161-164
            tslimit = int(incr_ratio * tslimit)
        step_tend = time.time()
        stats = dict(EpRewMax=float(returns.max()), EpRewMean=float(returns.mean()), EpRewStd=float(returns.std()),
                     EpLenMean=float(lengths_n2.mean()), Norm=float(torch.square(cache.theta[0]).sum()),
                     EpisodesThisIter=int(lengths_n2.size), EpisodesSoFar=int(episodes_so_far),
                     TimestepsThisIter=int(lengths_n2.sum()), TimestepsSoFar=int(timesteps_so_far),
                     UniqueWorkers=world, TimeElapsedThisIter=step_tend - step_tstart, TimeElapsed=step_tend - tstart)
        stats.update(deep_stats)
        stats = reference_row("ga", stats, world)                                      # the reference's keys, in its order
        if rank == 0:
            tlogger.log('Elite: {} score: {}'.format(elite if deep else population[0], population_score[0]))
            for k, v in stats.items():
                tlogger.record_tabular(k, v)
            tlogger.dump_tabular()
        if on_iteration is not None:
            on_iteration(it, stats, dict(population=population, population_score=population_score, returns=returns,
                                         genomes=genomes, elite_theta=cache.theta[population.index(elite)] if deep else cache.theta[0],
                                         **deep_extra))
        if rank == 0 and log_dir and config.snapshot_freq != 0:                        # ga.py:198-206 (every iteration)
            import os.path as osp
            policy.save(osp.join(log_dir, 'snapshot_iter{:05d}_rew{}.h5'.format(it, int(population_score[0]))))
    return population, population_score


def run_worker(master_redis_cfg, relay_redis_cfg, noise, *, min_task_runtime=.2, exp=None, **kw):
    """ga.py:209-284: a worker is a non-zero rank of the torchrun job running the same loop."""
    assert isinstance(noise, SharedNoiseTable)
    if exp is None:
        raise RuntimeError("run_worker needs the experiment dict (no redis); launch every rank through "
                           "`python -m es_distributed.main master --algo ga` under torchrun")
    return run_master(master_redis_cfg, None, exp, noise=noise, **kw)
