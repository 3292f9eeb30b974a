"""``es_distributed.es`` -- the reference's ES driver API (es.py:12-23,26-85,125-138,141-353,366-439) on the H100 engine.

Same names, argument meaning and configuration keys: ``Config``, ``Task``, ``Result``, ``RunningStat``,
``SharedNoiseTable``, ``compute_ranks``, ``compute_centered_ranks``, ``setup``, ``run_master``, ``run_worker``.
What changed underneath:
  * no redis: "workers" are the GPU ranks of one torchrun job (or the single process); the master loop and the
    worker loop of the reference run in the same process, one generation = rollouts of this rank's shard of the
    perturbations on its env slots, then all_gather(returns) + all_reduce(partial gradient) over NCCL;
  * theta, Adam state and the noise table never leave HBM; members' weights are never materialised.
``master_redis_cfg`` / ``relay_redis_cfg`` are accepted and ignored.  ``max_iterations`` (new, optional) bounds
the otherwise infinite ``while True`` of es.py:193.
"""
from __future__ import annotations

import logging
import time
from collections import namedtuple

import numpy as np
import torch

from dne import _ffi as F
from dne import shard
from dne.engine import ESUpdate, make_context
from dne.envs import BatchEnv, make_env
from dne.noise import SharedNoiseTable
from dne.rollout import Unit, make_runner

logger = logging.getLogger(__name__)

Config = namedtuple('Config', [
    'l2coeff', 'noise_stdev', 'episodes_per_batch', 'timesteps_per_batch',
    'calc_obstat_prob', 'eval_prob', 'snapshot_freq',
    'return_proc_mode', 'episode_cutoff_mode'
])
Task = namedtuple('Task', ['params', 'ob_mean', 'ob_std', 'ref_batch', 'timestep_limit'])
Result = namedtuple('Result', [
    'worker_id',
    'noise_inds_n', 'returns_n2', 'signreturns_n2', 'lengths_n2',
    'eval_return', 'eval_length',
    'ob_sum', 'ob_sumsq', 'ob_count'
])

# ---- process-wide engine state (one GPU per process) -----------------------------------------------------------
_STATE = {"noise": None, "ctx": None}


def default_noise(count=None) -> SharedNoiseTable:
    if _STATE["noise"] is None:
        _STATE["noise"] = SharedNoiseTable() if count is None else SharedNoiseTable(count=count)
    return _STATE["noise"]


def set_default_noise(noise: SharedNoiseTable):
    _STATE["noise"] = noise
    _STATE["ctx"] = None


def default_context() -> F.Context:
    if _STATE["ctx"] is None:
        _STATE["ctx"] = make_context(torch.cuda.current_device(), default_noise())
    return _STATE["ctx"]


class RunningStat(object):
    """es.py:26-48 (host numpy: a few hundred floats per generation, not on the device path)."""

    def __init__(self, shape, eps):
        self.sum = np.zeros(shape, dtype=np.float32)
        self.sumsq = np.full(shape, eps, dtype=np.float32)
        self.count = eps

    def increment(self, s, ssq, c):
        self.sum += s
        self.sumsq += ssq
        self.count += c

    @property
    def mean(self):
        return self.sum / self.count

    @property
    def std(self):
        return np.sqrt(np.maximum(self.sumsq / self.count - np.square(self.mean), 1e-2))

    def set_from_init(self, init_mean, init_std, init_count):
        self.sum[:] = init_mean * init_count
        self.sumsq[:] = (np.square(init_mean) + np.square(init_std)) * init_count
        self.count = init_count


def _device_ranks(x: np.ndarray):
    import ctypes as C
    dev = torch.device("cuda", torch.cuda.current_device())
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32).ravel()).to(dev)
    cen = torch.empty_like(t)
    ranks = torch.empty(t.numel(), dtype=torch.int32, device=dev)
    F.check(F.lib().dne_centered_rank(F.ptr(t), t.numel(), F.ptr(cen), F.ptr(ranks), F.stream_ptr()))
    return cen, ranks


def compute_ranks(x):
    """es.py:70-78 (stable tie rule), computed by dne_centered_rank."""
    assert x.ndim == 1
    return _device_ranks(x)[1].cpu().numpy().astype(np.int64)


def compute_centered_ranks(x):
    """es.py:81-85."""
    return _device_ranks(x)[0].cpu().numpy().reshape(x.shape)


def itergroups(items, group_size):
    assert group_size >= 1
    group = []
    for x in items:
        group.append(x)
        if len(group) == group_size:
            yield tuple(group)
            del group[:]
    if group:
        yield tuple(group)


def get_ref_batch(env: BatchEnv, batch_size=32, rs=None):
    """es.py:105-113: ``batch_size`` observations collected under random actions (slot 0 of the batched env)."""
    rs = rs or np.random.RandomState(0)
    ref_batch = []
    slot = np.array([0])
    env.reset(slot)
    while len(ref_batch) < batch_size:
        _, done = env.step(slot, env.random_actions(1, rs))
        if hasattr(env, "advance"):
            env.advance()
        ref_batch.append(env.obs_block(0, 1)[0].numpy().copy())
        if done[0]:
            env.reset(slot)
    return ref_batch


def setup(exp, single_threaded, n_slots=256, env=None, seed=None):
    """es.py:125-138: (config, env, sess, policy).  ``sess`` is None (no TensorFlow); ``env`` is a batched env."""
    from . import policies
    config = Config(**exp['config'])
    if env is None:
        extra = {'maze_file': exp['maze_file']} if exp.get('maze_file') else {}
        env = make_env(exp['env_id'], n_slots, seed=0 if seed is None else seed,
                       episode_len=exp.get('synthetic_episode_len'), allow_synthetic=bool(exp.get('allow_synthetic_env')),
                       **extra)
    policy = getattr(policies, exp['policy']['type'])(env.observation_space, env.action_space, **exp['policy']['args'],
                                                     seed=seed)
    return config, env, None, policy


def _cutoff(config):
    """es.py:169-186."""
    m = config.episode_cutoff_mode
    if isinstance(m, int):
        return m, None, None, m, False
    if m.startswith('adaptive:'):
        _, args = m.split(':')
        a0, a1, a2, a3 = args.split(',')
        return int(a0), float(a1), float(a2), float(a3), True
    if m == 'env_default':
        return None, None, None, None, False
    raise NotImplementedError(m)


def _process_returns(config, upd: ESUpdate, returns_n2, signreturns_n2):
    """es.py:281-288 on the device."""
    mode = config.return_proc_mode
    if mode == 'centered_rank':
        return upd.centered_ranks(returns_n2)[0]
    if mode == 'sign':
        return signreturns_n2.to(upd.device, torch.float32)
    if mode == 'centered_sign_rank':
        return upd.centered_ranks(signreturns_n2)[0]
    raise NotImplementedError(mode)


class GenerationStats(dict):
    pass


# The keys the reference's masters log every iteration, in their order (es.py:313-339, ga.py:171-196, nses.py:256-284,
# rs.py; tests/golden/ref_log_keys.json is that list extracted from the reference sources).
REF_ROW_KEYS = {
    "ga": ["EpRewMax", "EpRewMean", "EpRewStd", "EpLenMean", "EvalEpRewMean", "EvalEpRewMedian", "EvalEpRewStd", "EvalEpLenMean",
           "EvalPopRank", "EvalEpCount", "Norm", "EpisodesThisIter", "EpisodesSoFar", "TimestepsThisIter", "TimestepsSoFar",
           "UniqueWorkers", "UniqueWorkersFrac", "ResultsSkippedFrac", "ObCount", "TimeElapsedThisIter", "TimeElapsed"],
    "nses": ["ParentId", "EpRewMean", "EpRewStd", "EpLenMean", "EvalEpRewMean", "EvalEpRewStd", "EvalEpLenMean", "EvalPopRank",
             "EvalEpCount", "Norm", "GradNorm", "UpdateRatio", "EpisodesThisIter", "EpisodesSoFar", "TimestepsThisIter",
             "TimestepsSoFar", "UniqueWorkers", "UniqueWorkersFrac", "ResultsSkippedFrac", "ObCount", "TimeElapsedThisIter",
             "TimeElapsed"],
}
REF_ROW_KEYS["rs"] = list(REF_ROW_KEYS["ga"])
_ROW_DEFAULTS = dict(EvalEpRewMean=float("nan"), EvalEpRewMedian=float("nan"), EvalEpRewStd=float("nan"),
                     EvalEpLenMean=float("nan"), EvalPopRank=float("nan"), EvalEpCount=0, UniqueWorkersFrac=1.0,
                     ResultsSkippedFrac=0.0, ObCount=0)


def reference_row(kind, stats, world=1):
    """``stats`` as the row the reference's master of this algorithm logs: every reference key, in the reference's order, then
    this engine's extra keys.  Keys without a counterpart here get the reference's own "nothing happened" value (no evaluation
    episodes this iteration: NaN statistics and EvalEpCount 0; no stale results; one 'worker' per rank)."""
    d = dict(_ROW_DEFAULTS, UniqueWorkers=world)
    d.update(stats)
    out = {k: d[k] for k in REF_ROW_KEYS[kind]}
    out.update({k: v for k, v in stats.items() if k not in out})
    return out


def vine_export_cloud(root, iteration, bc_vectors):
    """es_modified.py:179-199 ``master_extract_cloud``: one row per offspring episode in
    ``<root>/snapshots/snapshot_gen_{it:04}/snapshot_offspring_{it:04}.dat`` = final BC row, fitness, length, noise index,
    policy seed, sign -- the per-generation point cloud the reference's visual_inspector reads.
    ``bc_vectors``: iterable of (bc [t, D] or [D], fitness, length, noise_idx, policy_seed, sign) (es_modified.py:505-512)."""
    import csv
    import os
    path = os.path.join(root, "snapshots", "snapshot_gen_{:04}".format(int(iteration)))
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "snapshot_offspring_{:04}.dat".format(int(iteration))), 'w+') as f:
        writer = csv.writer(f, delimiter=' ')
        for bc_vec, fitness, length, noise_idx, policy_seed, sign in bc_vectors:
            last = np.asarray(bc_vec)
            last = last[-1] if last.ndim > 1 else last
            writer.writerow(np.hstack((last, fitness, length, noise_idx, policy_seed, sign)))
    return path


def vine_export_parent(root, iteration, eval_bc_vecs, eval_rets, noise_stdev, policy=None, ref_batch=None):
    """es_modified.py:140-177 ``master_extract_parent``: the parent's snapshot (+ pickled reference batch) and the
    evaluation episode whose return is closest to the mean as ``snapshot_parent_{it:04}.dat`` (final BC row, fitness,
    length, seed, noise_stdev)."""
    import csv
    import os
    import pickle
    path = os.path.join(root, "snapshots", "snapshot_gen_{:04}".format(int(iteration)))
    os.makedirs(path, exist_ok=True)
    if policy is not None:
        policy.save(os.path.join(path, "snapshot_parent_{:04d}.h5".format(iteration)))
    if ref_batch is not None:
        with open(os.path.join(path, "snapshot_parent_{:04d}_rb.p".format(iteration)), "wb") as f:
            pickle.dump(ref_batch, f)
    if not len(eval_rets):
        return path
    rets = np.asarray(eval_rets)
    idx = int((np.abs(rets - int(np.mean(rets)))).argmin())                    # es_modified.py:165-167
    bc_vec, fitness, length, seed = eval_bc_vecs[idx]
    last = np.asarray(bc_vec)
    last = last[-1] if last.ndim > 1 else last
    with open(os.path.join(path, "snapshot_parent_{:04}.dat".format(int(iteration))), 'w+') as f:
        csv.writer(f, delimiter=' ').writerow(np.hstack((last, fitness, length, seed, noise_stdev)))
    return path


class TrainingState(object):
    """gpu_implementation/es.py:40-83,155-162,278-283: everything a run needs to continue after a restart -- iteration and
    timestep counters, the (adaptive) timestep limit, theta, the optimizer's moments and step count, the observation
    statistics and the noise-index stream -- pickled to ``<log_dir>/snapshot.pkl`` after every iteration and picked up by the
    next ``run_master`` on the same ``log_dir``.  Arrays are host numpy copies (the device state is rebuilt from them)."""

    FILE = 'snapshot.pkl'

    def __init__(self, exp):
        self.exp = exp
        self.it = 0
        self.timesteps_so_far = 0
        self.episodes_so_far = 0
        self.time_elapsed = 0.0
        self.tslimit = None
        self.theta = None
        self.optimizer = None          # dict(kind, t, m, v)
        self.ob_stat = None            # dict(sum, sumsq, count)
        self.rs_state = None           # np.random.RandomState.get_state() of the noise-index stream

    def capture(self, optimizer, ob_stat, rs):
        upd = optimizer._upd
        self.theta = upd.theta.cpu().numpy()
        self.optimizer = dict(kind=upd.kind, t=int(upd.t), v=upd.v.cpu().numpy(),
                              m=None if upd.m is None else upd.m.cpu().numpy())
        self.ob_stat = None if ob_stat is None else dict(sum=ob_stat.sum.copy(), sumsq=ob_stat.sumsq.copy(), count=ob_stat.count)
        self.rs_state = rs.get_state()

    def restore(self, optimizer, ob_stat, rs):
        upd = optimizer._upd
        assert upd.kind == self.optimizer['kind'] and upd.P == self.theta.size
        upd.theta.copy_(torch.from_numpy(self.theta))
        upd.v.copy_(torch.from_numpy(self.optimizer['v']))
        if upd.m is not None:
            upd.m.copy_(torch.from_numpy(self.optimizer['m']))
        upd.t = int(self.optimizer['t'])
        upd.ctx.theta_epoch = getattr(upd.ctx, "theta_epoch", 0) + 1
        if ob_stat is not None and self.ob_stat is not None:
            ob_stat.sum[:], ob_stat.sumsq[:], ob_stat.count = self.ob_stat['sum'], self.ob_stat['sumsq'], self.ob_stat['count']
        rs.set_state(self.rs_state)

    def save(self, log_dir):
        import os
        import pickle
        os.makedirs(log_dir, exist_ok=True)
        tmp = os.path.join(log_dir, self.FILE + '.tmp')
        with open(tmp, 'wb') as f:
            pickle.dump(self, f)
        os.replace(tmp, os.path.join(log_dir, self.FILE))

    @classmethod
    def load(cls, log_dir):
        import os
        import pickle
        with open(os.path.join(log_dir, cls.FILE), 'rb') as f:
            return pickle.load(f)


def run_master(master_redis_cfg, log_dir, exp, *, max_iterations=None, n_slots=256, env=None, noise=None, seed=None,
               on_iteration=None):
    """es.py:141-353.  Every rank of the job calls this (rank 0 logs); returns the final flat theta (numpy) once
    ``max_iterations`` generations are done."""
    from .optimizers import SGD, Adam
    from . import tabular_logger as tlogger
    rank, world = shard.dist_info()
    if rank == 0:
        logger.info('run_master: {}'.format({'log_dir': log_dir, 'exp': exp}))
        tlogger.start(log_dir)
    else:
        tlogger.set_quiet(True)
    if noise is not None:
        set_default_noise(noise)
    noise = default_noise()
    ctx = default_context()
    seed = shard.broadcast_seed(seed)
    config, env, _, policy = setup(exp, single_threaded=False, n_slots=n_slots, env=env, seed=seed)
    theta = policy.get_trainable_flat()
    optimizer = {'sgd': SGD, 'adam': Adam}[exp['optimizer']['type']](theta, ctx=ctx, **exp['optimizer']['args'])
    policy.bind_theta(optimizer.device_theta)
    upd: ESUpdate = optimizer._upd
    rs = np.random.RandomState(seed)          # identical on every rank: same noise-index stream (bit-exact bookkeeping)
    P = policy.num_params

    ob_stat = None
    if policy.needs_ob_stat:
        ob_stat = RunningStat(env.observation_space.shape, eps=1e-2)           # es.py:155-158
    ref_batch = None
    if policy.needs_ref_batch:
        ref_batch = get_ref_batch(env, batch_size=128, rs=np.random.RandomState(seed))   # es.py:160-162
        policy.set_ref_batch(ref_batch)

    tslimit, incr_tslimit_threshold, tslimit_incr_ratio, tslimit_max, adaptive_tslimit = _cutoff(config)
    vine = bool(exp.get('vine_export'))        # es_modified.py: per-generation BC point clouds for the visual inspector
    group = 2
    runner = make_runner(ctx, policy.net, env, n_slots=n_slots, group=group,
                         pipeline=2 if n_slots % 4 == 0 else 1, ref_batch=policy.ref_batch, **policy.runner_head_kw())

    episodes_so_far = timesteps_so_far = 0
    tstart = time.time()
    it = 0
    # resume (gpu_implementation/es.py:155-162): a snapshot.pkl in log_dir continues that run; written after every
    # iteration when exp['save_training_state'] is set (rank 0 writes, every rank of a restarted job reads the same file)
    state = TrainingState(exp)
    keep_state = bool(exp.get('save_training_state')) and bool(log_dir)
    if keep_state:
        try:
            state = TrainingState.load(log_dir)
            state.restore(optimizer, ob_stat, rs)
            it, timesteps_so_far, episodes_so_far = state.it, state.timesteps_so_far, state.episodes_so_far
            if state.tslimit is not None:
                tslimit = state.tslimit
            if rank == 0:
                tlogger.log('Loaded iteration {} from {}'.format(state.it, log_dir))
        except FileNotFoundError:
            pass
    while max_iterations is None or it < max_iterations:
        step_tstart = time.time()
        it += 1
        if rank == 0:
            tlogger.log('********** Iteration {} **********'.format(it))
        ob_mean = ob_std = None
        if policy.needs_ob_stat:
            policy.set_ob_stat(ob_stat.mean, ob_stat.std)                       # es.py:382-383 (task.ob_mean/std)
            ob_mean, ob_std = policy.ob_mean, policy.ob_std

        noise_inds, returns, signreturns, lengths = [], [], [], []
        eval_rets, eval_lens = [], []
        num_eps = num_ts = 0
        ob_count_this_batch = 0
        ob_acc = None
        vine_cloud, vine_eval = [], []
        ticks_this_iter = 0
        first = True
        # es.py:230: collect until BOTH quotas are met.  First batch = ceil(episodes_per_batch/2) pairs; if the
        # timestep quota is still short, keep adding world*n_slots/2 pairs at a time.
        while first or num_eps < config.episodes_per_batch or num_ts < config.timesteps_per_batch:
            n_pairs = -(-config.episodes_per_batch // 2) if first else world * n_slots // 2
            n_eval = int(rs.binomial(n_pairs, config.eval_prob)) if (first and config.eval_prob > 0) else 0
            idx = np.array([noise.sample_index(rs, P) for _ in range(n_pairs)], dtype=np.int64)      # es.py:412
            sig = np.float32(config.noise_stdev)
            units = [Unit(int(i), (sig, -sig)) for i in idx] + \
                    [Unit(0, (0.0, 0.0), noiseless=True) for _ in range(-(-n_eval // 2))]        # es.py:388-391
            lo, hi = shard.shard_bounds(len(units), rank, world)
            # the worker-side random stream (es.py:372: action noise, ob-stat sampling) is separate from the seeded
            # noise-index stream, so the index sequence never depends on episode lengths or the rank count
            res = runner.run(optimizer.device_theta, units[lo:hi], tslimit, ob_mean=ob_mean, ob_std=ob_std,
                             collect_bc="final" if vine else None,
                             ac_noise_std=getattr(policy, "ac_noise_std", 0.0),
                             random_stream=np.random.RandomState((seed + 1000 * it + rank) % (2 ** 31)),
                             save_obs_prob=config.calc_obstat_prob if policy.needs_ob_stat else 0.0)
            if policy.needs_ob_stat and config.calc_obstat_prob != 0:                # es.py:260-263
                acc = np.concatenate([res.ob_sum, res.ob_sumsq, [float(res.ob_count)]])
                ob_acc = acc if ob_acc is None else ob_acc + acc
            ticks_this_iter += res.ticks
            if vine:                       # es_modified.py:505-512: (bc, return, length, noise_idx, policy_seed, sign) per episode
                mine = [(res.bcs[u][g], float(res.returns[u, g]), int(res.lengths[u, g]),
                         int(units[lo + u].noise_idx), 0, 1 if g == 0 else -1, lo + u >= n_pairs)
                        for u in range(hi - lo) for g in range(2)]
                for part in (shard.all_gather_object(mine) if world > 1 else [mine]):
                    vine_cloud += [p[:6] for p in part if not p[6]]
                    vine_eval += [(p[0], p[1], p[2], 0) for p in part if p[6]][:max(0, n_eval - len(vine_eval))]
            dev = upd.device
            pack = torch.from_numpy(np.concatenate([res.returns, res.signreturns, res.lengths.astype(np.float32)],
                                                   axis=1)).to(dev)
            allr = shard.all_gather_rows(pack, len(units)).cpu().numpy()
            r_all, s_all, l_all = allr[:, 0:2], allr[:, 2:4], allr[:, 4:6].astype(np.int32)
            noise_inds.append(idx)
            returns.append(r_all[:n_pairs]); signreturns.append(s_all[:n_pairs]); lengths.append(l_all[:n_pairs])
            if n_eval:
                eval_rets += list(r_all[n_pairs:].ravel()[:n_eval])
                eval_lens += list(l_all[n_pairs:].ravel()[:n_eval])
            num_eps += 2 * n_pairs
            num_ts += int(l_all[:n_pairs].sum())
            first = False

        noise_inds_n = np.concatenate(noise_inds)
        returns_n2 = np.concatenate(returns).astype(np.float32)
        signreturns_n2 = np.concatenate(signreturns).astype(np.float32)
        lengths_n2 = np.concatenate(lengths)
        episodes_so_far += lengths_n2.size + len(eval_lens)
        timesteps_so_far += int(lengths_n2.sum()) + int(np.sum(eval_lens))
        assert noise_inds_n.shape[0] == returns_n2.shape[0] == lengths_n2.shape[0]

        # ---- update (es.py:281-301) on the device ----
        dev = upd.device
        proc = _process_returns(config, upd, torch.from_numpy(returns_n2).to(dev), torch.from_numpy(signreturns_n2).to(dev))
        n = len(noise_inds_n)
        lo, hi = shard.shard_bounds(n, rank, world)
        d_idx = torch.from_numpy(noise_inds_n[lo:hi]).to(dev)
        g = upd.gradient(proc[lo:hi].contiguous(), d_idx, denom=returns_n2.size)      # partial over this rank's indices
        shard.all_reduce_sum_(g)                                                      # 4*P bytes over NVLink
        update_ratio, _ = optimizer.update_from_gradient(g, config.l2coeff)           # es.py:298

        # ---- observation statistics (es.py:260-263): every worker's (sum, sumsq, count) added into the running stat ----
        if ob_acc is not None:
            t = torch.from_numpy(ob_acc).to(dev)
            shard.all_reduce_sum_(t)
            tot = t.cpu().numpy()
            D = (len(tot) - 1) // 2
            ob_count_this_batch = int(round(tot[-1]))
            if ob_count_this_batch > 0:
                shp = ob_stat.sum.shape
                ob_stat.increment(tot[:D].astype(np.float32).reshape(shp), tot[D:2 * D].astype(np.float32).reshape(shp),
                                  ob_count_this_batch)

        if adaptive_tslimit and (lengths_n2 == tslimit).mean() >= incr_tslimit_threshold:   # es.py:308-311
            old = tslimit
            tslimit = min(int(tslimit_incr_ratio * tslimit), tslimit_max)
            logger.info('Increased timestep limit from {} to {}'.format(old, tslimit))

        step_tend = time.time()
        stats = GenerationStats(
            EpRewMean=float(returns_n2.mean()), EpRewStd=float(returns_n2.std()), EpLenMean=float(lengths_n2.mean()),
            EvalEpRewMean=np.nan if not eval_rets else float(np.mean(eval_rets)),
            EvalEpRewMedian=np.nan if not eval_rets else float(np.median(eval_rets)),
            EvalEpRewStd=np.nan if not eval_rets else float(np.std(eval_rets)),
            EvalEpLenMean=np.nan if not eval_rets else float(np.mean(eval_lens)),
            EvalPopRank=np.nan if not eval_rets else float(
                np.searchsorted(np.sort(returns_n2.ravel()), eval_rets).mean() / returns_n2.size),
            EvalEpCount=len(eval_rets),
            Norm=float(torch.square(optimizer.device_theta).sum()), GradNorm=float(torch.square(g).sum()),
            UpdateRatio=float(update_ratio),
            EpisodesThisIter=int(lengths_n2.size), EpisodesSoFar=int(episodes_so_far),
            TimestepsThisIter=int(lengths_n2.sum()), TimestepsSoFar=int(timesteps_so_far),
            UniqueWorkers=world, UniqueWorkersFrac=1.0, ResultsSkippedFrac=0.0, ObCount=ob_count_this_batch,
            TimeElapsedThisIter=step_tend - step_tstart, TimeElapsed=step_tend - tstart)
        if rank == 0:
            for k, v in stats.items():
                tlogger.record_tabular(k, v)
            tlogger.dump_tabular()
        if on_iteration is not None:
            on_iteration(it, stats, dict(noise_inds_n=noise_inds_n, returns_n2=returns_n2, lengths_n2=lengths_n2,
                                         signreturns_n2=signreturns_n2, g=g, theta=optimizer.device_theta,
                                         forward_launches=ticks_this_iter, ob_stat=ob_stat,
                                         slots_per_launch=n_slots // len(runner.halves)))
        if vine and rank == 0 and log_dir:                                                # es_modified.py:140-199
            vine_export_cloud(log_dir, it, vine_cloud)
            vine_export_parent(log_dir, it, vine_eval, [e[1] for e in vine_eval], config.noise_stdev)
        if keep_state:                                                                    # gpu_implementation/es.py:278-283
            state.it, state.timesteps_so_far, state.episodes_so_far = it, timesteps_so_far, episodes_so_far
            state.tslimit, state.time_elapsed = tslimit, step_tend - tstart
            state.capture(optimizer, ob_stat, rs)
            if rank == 0:
                state.save(log_dir)
            shard.barrier()
        if rank == 0 and log_dir and config.snapshot_freq != 0 and it % config.snapshot_freq == 0:   # es.py:345-353
            import os.path as osp
            filename = osp.join(log_dir, 'snapshot_iter{:05d}_rew{}.h5'.format(
                it, np.nan if not eval_rets else int(np.mean(eval_rets))))
            policy.save(filename)
            tlogger.log('Saved snapshot {}'.format(filename))
    return optimizer.theta


def run_worker(master_redis_cfg, relay_redis_cfg, noise, *, min_task_runtime=.2, exp=None, **kw):
    """es.py:366-439.  In this engine a "worker" is a non-zero rank of the torchrun job: it runs the same loop as
    the master on its shard of the population (NCCL replaces the redis relay)."""
    assert isinstance(noise, SharedNoiseTable)
    if exp is None:
        raise RuntimeError("run_worker needs the experiment dict (there is no redis to fetch it from); "
                           "launch every rank through `python -m es_distributed.main master` under torchrun")
    return run_master(master_redis_cfg, None, exp, noise=noise, **kw)
