"""GPU tests of the reference-facing drivers (es_distributed.{es,ga,nses}.run_master) on BASELINE.json configs[0]-
style plumbing runs: the reference's configuration dictionaries drive the engine, and every generation's bookkeeping
and update is re-derived by the oracle from the same (noise indices, returns)."""
import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from oracle import oracle as O                 # noqa: E402
from dne.envs import SyntheticAtariEnv          # noqa: E402
from dne.noise import SharedNoiseTable          # noqa: E402

NOISE_COUNT = 6_000_000
FROSTBITE_ES = {      # configurations/frostbite_es.json (reference), population scaled down like BASELINE.json configs[0]
    "config": {"calc_obstat_prob": 0.0, "episodes_per_batch": 16, "eval_prob": 0.1, "l2coeff": 0.005,
               "noise_stdev": 0.005, "snapshot_freq": 0, "timesteps_per_batch": 10, "return_proc_mode": "centered_rank",
               "episode_cutoff_mode": 5000},
    "env_id": "FrostbiteNoFrameskip-v4",
    "optimizer": {"args": {"stepsize": 0.01}, "type": "adam"},
    "policy": {"args": {}, "type": "ESAtariPolicy"},
}
FROSTBITE_GA = {      # configurations/frostbite_ga.json
    "config": {"calc_obstat_prob": 0.0, "episodes_per_batch": 12, "eval_prob": 0.0, "l2coeff": 0.005,
               "noise_stdev": 0.005, "snapshot_freq": 0, "timesteps_per_batch": 10, "return_proc_mode": "centered_rank",
               "episode_cutoff_mode": 5000},
    "population_size": 4, "num_elites": 1, "env_id": "FrostbiteNoFrameskip-v4",
    "policy": {"args": {"nonlin_type": "relu"}, "type": "GAAtariPolicy"},
}
FROSTBITE_NSR = {     # configurations/frostbite_nsres.json
    "config": {"calc_obstat_prob": 0.0, "episodes_per_batch": 8, "eval_prob": 0.0, "l2coeff": 0.005, "noise_stdev": 0.02,
               "snapshot_freq": 0, "timesteps_per_batch": 10, "return_proc_mode": "centered_sign_rank",
               "episode_cutoff_mode": 5000},
    "env_id": "FrostbiteNoFrameskip-v4", "algo_type": "nsr",
    "novelty_search": {"k": 3, "population_size": 2, "num_rollouts": 1, "selection_method": "novelty_prob"},
    "optimizer": {"args": {"stepsize": 0.01}, "type": "adam"},
    "policy": {"args": {}, "type": "ESAtariPolicy"},
}


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def noise(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device="cuda:0")


def test_reference_config_files_parse_unchanged():
    """The reference's own configuration keys are the ones the drivers read (no renamed / extra required keys)."""
    from es_distributed.es import Config
    ref = {"config": {"calc_obstat_prob": 0.0, "episodes_per_batch": 5000, "eval_prob": 0.01, "l2coeff": 0.005,
                      "noise_stdev": 0.005, "snapshot_freq": 20, "timesteps_per_batch": 10000,
                      "return_proc_mode": "centered_rank", "episode_cutoff_mode": 5000}}
    cfg = Config(**ref["config"])
    assert cfg.episodes_per_batch == 5000 and cfg.episode_cutoff_mode == 5000


def test_es_run_master_generation_matches_oracle(noise, host_noise, tmp_path):
    from es_distributed import es as ES
    env = SyntheticAtariEnv(8, episode_len=(3, 9), seed=3)
    log = []
    theta_before = {}

    def on_it(it, stats, extra):
        log.append((it, dict(stats), {k: (v.clone() if hasattr(v, "clone") else np.array(v)) for k, v in extra.items()
                                      if k in ("noise_inds_n", "returns_n2", "lengths_n2", "g", "theta")}))
    ES.set_default_noise(noise)
    # capture theta0 by seeding the policy the same way run_master does
    theta_final = ES.run_master({"unix_socket_path": None}, str(tmp_path), json.loads(json.dumps(FROSTBITE_ES)),
                                max_iterations=2, n_slots=8, env=env, noise=noise, seed=11, on_iteration=on_it)
    assert len(log) == 2 and theta_final.dtype == np.float32 and theta_final.shape == (1009058,)
    net = O.make_net("ESAtariPolicy")
    P = net.num_params
    from es_distributed import policies
    pol = policies.ESAtariPolicy(env.observation_space, env.action_space, seed=11)
    theta = pol.get_trainable_flat()
    adam = O.Adam(theta, 0.01)
    for it, stats, ex in log:
        idx, ret = ex["noise_inds_n"], ex["returns_n2"]
        assert idx.dtype == np.int64 and ret.shape == (len(idx), 2) and ret.dtype == np.float32
        assert len(idx) >= 8 and ex["lengths_n2"].min() >= 3 and ex["lengths_n2"].max() <= 9
        assert (idx >= 0).all() and (idx <= NOISE_COUNT - P).all()
        assert stats["EpisodesThisIter"] == ret.size and stats["TimestepsThisIter"] == int(ex["lengths_n2"].sum())
        g, ratio, new_theta = O.es_generation_update(adam.theta, adam, host_noise, idx, ret, 0.005)
        got_g = ex["g"].cpu().numpy()
        assert np.abs(got_g - g).max() <= 1e-5 * np.abs(g).max()
        np.testing.assert_allclose(ex["theta"].cpu().numpy(), new_theta, rtol=0, atol=2e-7)
        assert stats["UpdateRatio"] == pytest.approx(float(ratio), rel=1e-4)
    np.testing.assert_allclose(theta_final, adam.theta, rtol=0, atol=2e-7)
    assert os.path.exists(os.path.join(str(tmp_path), "log.txt"))


def test_ga_run_master_bookkeeping(noise, host_noise, tmp_path):
    from es_distributed import ga as GA
    env = SyntheticAtariEnv(8, episode_len=4, seed=5, num_actions=6)
    log = []
    GA.set_default_noise(noise)
    pop, score = GA.run_master(None, str(tmp_path), json.loads(json.dumps(FROSTBITE_GA)), max_iterations=3, n_slots=8,
                               env=env, noise=noise, seed=2,
                               on_iteration=lambda it, st, ex: log.append((it, st, {k: (v.clone() if hasattr(v, "clone") else v)
                                                                                    for k, v in ex.items()})))
    assert len(pop) == 4 and len(score) == 4 and len(log) == 3
    net = O.make_net("GAAtariPolicy", num_actions=6)
    prev_pop, prev_score = [], np.array([], dtype=np.float32)
    for it, st, ex in log:
        genomes, returns = ex["genomes"], ex["returns"]
        assert len(genomes) == 12 and all(1 <= len(g) <= it for g in genomes)     # a chain grows by one seed per generation it survives
        if it > 1:
            assert all(tuple(g[:-1]) in [tuple(p) for p in prev_pop] for g in genomes)   # parent drawn from the population
        cand = [tuple(p) for p in prev_pop[:1]] + [tuple(g) for g in genomes]        # ga.py:136-140 (elite first)
        fit = np.concatenate([prev_score[:1], returns]).astype(np.float32)
        sel = O.ga_truncate(fit, 4)
        assert [tuple(p) for p in ex["population"]] == [cand[i] for i in sel]
        np.testing.assert_array_equal(ex["population_score"], fit[sel])
        assert ex["population_score"][0] == fit.max()                               # ga.py:149
        elite = O.ga_materialize_cpu(net, host_noise, list(ex["population"][0]), 0.005)
        np.testing.assert_allclose(ex["elite_theta"].cpu().numpy(), elite, rtol=1e-6, atol=1e-9)
        prev_pop, prev_score = ex["population"], ex["population_score"]


def test_rs_run_master_keeps_best_candidate(noise, host_noise, tmp_path):
    """rs.py:112-116: the policy becomes reinitialize(noise[idx]) of the best-scoring candidate seen so far."""
    from es_distributed import rs as RS
    env = SyntheticAtariEnv(8, episode_len=4, seed=6, num_actions=6)
    log = []
    RS.set_default_noise(noise)
    best_seed, best_score = RS.run_master(None, str(tmp_path), json.loads(json.dumps(FROSTBITE_GA)), max_iterations=3,
                                          n_slots=8, env=env, noise=noise, seed=3,
                                          on_iteration=lambda it, st, ex: log.append((it, st, dict(ex, theta=ex["theta"].clone()))))
    assert len(log) == 3
    net = O.make_net("GAAtariPolicy", num_actions=6)
    run_best, run_seed = -np.inf, None
    for it, st, ex in log:
        r, idx = ex["returns_n2"], ex["noise_inds_n"]
        assert r.shape == ex["lengths_n2"].shape == (len(idx), 1) and len(idx) == 12 and r.dtype == np.float32
        assert np.all(ex["lengths_n2"] == 4) and st["EpisodesThisIter"] == 12
        j = int(np.argmax(r))
        if r[j, 0] > run_best:
            run_best, run_seed = float(r[j, 0]), int(idx[j])
        assert ex["best_score"] == run_best and ex["best_seed"] == run_seed
        want = O.ga_reinitialize(net, host_noise[run_seed:run_seed + net.num_params])
        np.testing.assert_allclose(ex["theta"].cpu().numpy(), want, rtol=1e-6, atol=1e-9)
    assert (best_seed, best_score) == (run_seed, run_best)


def test_nsr_run_master_novelty_and_update(noise, host_noise, tmp_path):
    from es_distributed import nses as NS
    env = SyntheticAtariEnv(8, episode_len=(3, 7), seed=9)
    log = []
    NS.set_default_noise(noise)
    NS.run_master(None, str(tmp_path), json.loads(json.dumps(FROSTBITE_NSR)), max_iterations=2, n_slots=8, env=env,
                  noise=noise, seed=4, on_iteration=lambda it, st, ex: log.append((it, st, dict(ex, g=ex["g"].clone()), len(ex["archive"]))))
    assert len(log) == 2
    for it, st, ex, arch_len in log:
        assert arch_len == 2 + it                                                     # nses.py:113-114, 246-247
        arch = ex["archive"].seqs[:arch_len - 1]                                     # archive as the rollouts saw it
        nov = np.array([O.compute_novelty_vs_archive(arch, b, 3) for b in ex["bcs"]], dtype=np.float32).reshape(-1, 2)
        np.testing.assert_allclose(ex["novelty_n2"], nov, rtol=1e-6)
        proc = O.nsr_blend(ex["returns_n2"], nov)                                     # nses.py:221-228
        g = O.es_gradient(proc, host_noise, ex["noise_inds_n"], 1009058)
        assert np.abs(ex["g"].cpu().numpy() - g).max() <= 1e-5 * np.abs(g).max()


HUMANOID_ES = {       # configurations/humanoid.json (reference) -- population / batch sizes scaled down
    "config": {"calc_obstat_prob": 0.5, "episodes_per_batch": 24, "eval_prob": 0.2, "l2coeff": 0.005, "noise_stdev": 0.02,
               "snapshot_freq": 0, "timesteps_per_batch": 10, "return_proc_mode": "centered_rank",
               "episode_cutoff_mode": "env_default"},
    "env_id": "Humanoid-v1",
    "optimizer": {"args": {"stepsize": 0.01}, "type": "adam"},
    "policy": {"args": {"ac_bins": "continuous:", "ac_noise_std": 0.01, "connection_type": "ff", "hidden_dims": [256, 256],
                        "nonlin_type": "tanh"}, "type": "MujocoPolicy"},
}


def test_es_humanoid_ob_stat_plumbing_matches_running_stat(noise, tmp_path):
    """es.py:356-363,260-263,304-305: episodes sampled with calc_obstat_prob contribute (sum o, sum o^2, count) of the
    observations fed to the policy; the master adds them into RunningStat and next iteration's rollouts normalise with the
    new mean / std.  The environment here records every observation block it hands out, so the oracle RunningStat can be
    rebuilt independently of the device accumulation: the set of sampled episodes is recovered from the counts."""
    from es_distributed import es as ES
    from dne.envs import SyntheticVectorEnv

    class Recorder(SyntheticVectorEnv):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            self.blocks = {}          # (lo, hi) -> observation block handed to the next forward
            self.fed = []             # (slot, obs vector) for every env step, in order

        def obs_block(self, lo, hi):
            blk = super().obs_block(lo, hi)
            self.blocks[(lo, hi)] = (lo, blk.clone().numpy())
            return blk

        def step(self, slots, actions):
            slots = np.asarray(slots)
            for (lo, hi), (l0, blk) in self.blocks.items():
                m = (slots >= lo) & (slots < hi)
                for s in slots[m]:
                    self.fed.append((int(s), blk[s - l0].copy()))
            return super().step(slots, actions)

    env = Recorder(8, episode_len=5, seed=4)
    snaps = []

    def on_it(it, stats, extra):
        st = extra["ob_stat"]
        snaps.append((it, stats["ObCount"], st.sum.copy(), st.sumsq.copy(), float(st.count), len(env.fed)))
    ES.set_default_noise(noise)
    ES.run_master(None, str(tmp_path), json.loads(json.dumps(HUMANOID_ES)), max_iterations=3, n_slots=8, env=env,
                  noise=noise, seed=5, on_iteration=on_it)
    assert len(snaps) == 3
    orc = O.RunningStat((376,), eps=1e-2)
    fed_prev = 0
    total = 0
    for it, ob_count, s_sum, s_sumsq, s_count, n_fed in snaps:
        fed = env.fed[fed_prev:n_fed]
        fed_prev = n_fed
        # episodes are 5 steps long: an episode is sampled as a whole, so the count is a multiple of 5 and with
        # prob 0.5 over >= 24 episodes some but not all episodes are sampled
        assert ob_count % 5 == 0 and 0 < ob_count < len(fed)
        total += ob_count
        assert s_count == pytest.approx(1e-2 + total)
        # the device sums must equal the sums over SOME set of whole episodes of this generation: check through the
        # totals' consistency with per-dimension bounds, then exactly through the mean of the sampled observations
        allv = np.stack([v for _, v in fed]).astype(np.float64)
        assert np.all(np.abs(s_sum) <= np.abs(allv).sum(axis=0) + 1.0)
    # exact check: rerun with probability 1 -> every observation fed counts
    env2 = Recorder(8, episode_len=5, seed=4)
    cfg = json.loads(json.dumps(HUMANOID_ES))
    cfg["config"]["calc_obstat_prob"] = 1.0
    cfg["config"]["eval_prob"] = 0.0
    snaps2 = []
    ES.run_master(None, str(tmp_path), cfg, max_iterations=2, n_slots=8, env=env2, noise=noise, seed=5,
                  on_iteration=lambda it, stats, extra: snaps2.append(
                      (stats["ObCount"], extra["ob_stat"].sum.copy(), extra["ob_stat"].sumsq.copy(),
                       float(extra["ob_stat"].count), extra["ob_stat"].mean.copy(), extra["ob_stat"].std.copy(), len(env2.fed))))
    orc = O.RunningStat((376,), eps=1e-2)
    prev = 0
    for ob_count, s_sum, s_sumsq, s_count, s_mean, s_std, n_fed in snaps2:
        obs = np.stack([v for _, v in env2.fed[prev:n_fed]])
        prev = n_fed
        assert ob_count == len(obs)
        orc.increment(obs.sum(axis=0), np.square(obs).sum(axis=0), len(obs))                 # es.py:358-359
        assert s_count == pytest.approx(orc.count)
        np.testing.assert_allclose(s_sum, orc.sum, rtol=1e-5, atol=1e-4)
        np.testing.assert_allclose(s_sumsq, orc.sumsq, rtol=1e-5, atol=1e-4)
        np.testing.assert_allclose(s_mean, orc.mean, rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(s_std, orc.std, rtol=1e-4, atol=1e-5)


def test_deep_ga_validation_and_elite_selection(noise, host_noise, tmp_path):
    """gpu_implementation/ga.py:180-204,260-271 (configurations/ga_atari_config.json keys): fitness-sorted population, the top
    validation_threshold (+ last elite) re-evaluated num_validation_episodes times, elite = argmax of the mean validation
    return, parents = top selection_threshold with the elite forced in -- every step re-derived by the oracle from the
    returns the driver reports."""
    from es_distributed import ga as GA
    from es_distributed import es as ES
    exp = {"config": {"calc_obstat_prob": 0.0, "episodes_per_batch": 12, "eval_prob": 0.0, "l2coeff": 0.005, "noise_stdev": 0.002,
                      "snapshot_freq": 0, "timesteps_per_batch": 10, "return_proc_mode": "centered_rank", "episode_cutoff_mode": 5000},
           "env_id": "FrostbiteNoFrameskip-v4", "ga_mode": "gpu", "policy": {"args": {}, "type": "GAAtariPolicy"},
           "population_size": 12, "selection_threshold": 4, "validation_threshold": 3, "num_validation_episodes": 5,
           "num_test_episodes": 2, "mutation_power": 0.002}
    env = SyntheticAtariEnv(8, episode_len=(3, 9), seed=5)
    log = []
    ES.set_default_noise(noise)
    GA.run_master(None, str(tmp_path), json.loads(json.dumps(exp)), max_iterations=3, n_slots=8, env=env, noise=noise, seed=3,
                  on_iteration=lambda it, stats, extra: log.append((it, dict(stats), extra)))
    assert len(log) == 3
    elite = None
    for it, stats, ex in log:
        fit = np.asarray(ex["returns"], dtype=np.float32)
        genomes = [tuple(g) for g in ex["genomes"]]
        assert len(genomes) == 12
        order = O.ga_truncate(fit, len(fit))                                    # stable descending (ga.py:180)
        pop_sorted = [genomes[i] for i in order]
        assert pop_sorted == ex["pop_sorted"]
        val_pop = O.deep_ga_validation_population(pop_sorted, elite, 3)
        assert val_pop == ex["val_pop"]
        assert ex["val_returns"].shape == (3, 5)
        new_elite, means = O.deep_ga_elite(val_pop, list(ex["val_returns"]))
        assert new_elite == ex["elite"] and stats["TruncatedPopulationEliteIndex"] == int(np.argmax(means))
        parents = O.deep_ga_parents(pop_sorted, new_elite, 4)
        assert parents == [tuple(g) for g in ex["population"]]
        assert new_elite in parents and len(parents) == 4
        assert all(1 <= len(g) <= it for g in genomes)                            # offspring = one mutation of a cached parent
        elite = new_elite


def test_es_training_state_resume_is_bit_identical(noise, tmp_path):
    """gpu_implementation/es.py:155-162,278-283: snapshot.pkl (theta, optimizer moments + step count, counters, the
    noise-index stream) after every iteration; a restarted run_master on the same log_dir continues exactly where the first
    one stopped: 1 iteration + restart + 1 iteration == 2 iterations, bit for bit (deterministic environment)."""
    from es_distributed import es as ES
    from dne.envs import DeterministicAtariEnv
    exp = json.loads(json.dumps(FROSTBITE_ES))
    exp["policy"]["type"] = "GAAtariPolicy"
    exp["config"]["eval_prob"] = 0.0
    exp["save_training_state"] = True
    ES.set_default_noise(noise)

    def run(log_dir, iters):
        return ES.run_master(None, str(log_dir), json.loads(json.dumps(exp)), max_iterations=iters, n_slots=8,
                             env=DeterministicAtariEnv(8, episode_len=6, seed=3), noise=noise, seed=11)
    straight = run(tmp_path / "a", 2)
    run(tmp_path / "b", 1)
    st = ES.TrainingState.load(str(tmp_path / "b"))
    assert st.it == 1 and st.optimizer["t"] == 1 and st.theta.shape == straight.shape
    resumed = run(tmp_path / "b", 2)
    np.testing.assert_array_equal(resumed, straight)
    assert ES.TrainingState.load(str(tmp_path / "b")).it == 2


def test_raw_frame_env_device_pipeline_matches_reference_wrappers():
    """dne/raw_env.py: emulators on a host thread pool + max / gray / Pillow-exact 84x84 warp / frame stack on the device
    against the reference's wrapper chain restated on the CPU (atari_wrappers.py:86-107 MaxAndSkipEnv, :129-142 WarpFrame,
    :167-180 FrameStack) fed with the SAME emulator frames: bit-exact uint8 stacks after resets and steps."""
    from dne.raw_env import SyntheticEmulator, RawFrameAtariEnv
    n = 6
    env = RawFrameAtariEnv([SyntheticEmulator(100 + s, frames=40) for s in range(n)], noop_max=3, seed=1, device="cuda:0")
    twin = [SyntheticEmulator(100 + s, frames=40) for s in range(n)]            # CPU replica of every emulator
    rs_noop = np.random.RandomState(1)
    stacks = np.zeros((n, 84, 84, 4), dtype=np.uint8)

    def cpu_reset(slots):
        noops = rs_noop.randint(1, 4, size=len(slots))
        for s, k in zip(slots, noops):
            f = twin[s].reset()
            for _ in range(k):
                _, over, f = twin[s].act(0)
                if over:
                    f = twin[s].reset()
            twin[s].last = f
            stacks[s] = O.warp_frame_cpu(f)[:, :, None]                           # FrameStack._reset: first frame x 4

    def cpu_step(slots, actions):
        for s, a in zip(slots, actions):
            prev = cur = twin[s].last
            for _ in range(4):
                _, over, f = twin[s].act(int(a))
                prev, cur = cur, f
                if over:
                    break
            twin[s].last = cur
            w = O.warp_frame_cpu(np.maximum(prev, cur))                           # MaxAndSkipEnv + WarpFrame
            stacks[s, :, :, :3] = stacks[s, :, :, 1:]
            stacks[s, :, :, 3] = w
    all_slots = np.arange(n)
    env.reset(all_slots)
    cpu_reset(all_slots)
    np.testing.assert_array_equal(env.device_obs(0, n).cpu().numpy(), stacks)
    rs = np.random.RandomState(2)
    for t in range(5):
        acts = rs.randint(0, 18, size=n)
        env.step(all_slots, acts)
        cpu_step(all_slots, acts)
        if t == 2:                                                                # mid-run reset of two slots
            env.reset(np.array([1, 4]))
            cpu_reset([1, 4])
        np.testing.assert_array_equal(env.device_obs(0, n).cpu().numpy(), stacks)


def test_es_run_master_on_raw_frame_env(noise, tmp_path):
    """The ES driver end to end on raw frames: thread-pool emulators, device preprocess, tensor-core forward, update."""
    from es_distributed import es as ES
    from dne.raw_env import make_synthetic_raw_env
    exp = json.loads(json.dumps(FROSTBITE_ES))
    exp["policy"]["type"] = "GAAtariPolicy"
    exp["config"].update(eval_prob=0.0, episodes_per_batch=8, episode_cutoff_mode=6)
    ES.set_default_noise(noise)
    env = make_synthetic_raw_env(8, seed=2, frames=400, noop_max=2, device="cuda:0")
    log = []
    theta = ES.run_master(None, str(tmp_path), exp, max_iterations=2, n_slots=8, env=env, noise=noise, seed=4,
                          on_iteration=lambda it, stats, extra: log.append(dict(stats)))
    assert len(log) == 2 and np.isfinite(theta).all()
    assert log[0]["EpLenMean"] == 6 and log[1]["TimestepsSoFar"] == 2 * 8 * 6


def test_mujoco_discretised_action_heads():
    """policies.py:116-119,166-190: 'uniform:N' and 'custom:...' heads -- a dense layer to adim*num_bins scores, per action
    dimension the argmax bin, mapped to evenly spaced / listed values rescaled to [low, high]."""
    from dne.envs import Box
    from es_distributed import policies
    ob, ac = Box(-np.inf, np.inf, (5,)), Box(np.array([-0.4, -1.0, 0.0], np.float32), np.array([0.4, 1.0, 2.0], np.float32))
    kw = dict(ac_noise_std=0.0, nonlin_type="tanh", hidden_dims=[8], connection_type="ff")
    pu = policies.MujocoPolicy(ob, ac, ac_bins="uniform:5", **kw)
    assert pu.net.n_out == 3 * 5
    scores = np.zeros((2, 3, 5), np.float32)
    scores[0, 0, 4] = scores[0, 1, 0] = scores[0, 2, 2] = 1.0
    scores[1, :, 1] = 1.0
    a = pu.action_fn(scores.reshape(2, 15))
    np.testing.assert_allclose(a[0], [0.4, -1.0, 1.0], rtol=1e-6)
    np.testing.assert_allclose(a[1], [-0.4 + 0.25 * 0.8, -1.0 + 0.25 * 2.0, 0.5], rtol=1e-6)
    pc = policies.MujocoPolicy(ob, ac, ac_bins="custom:-1,-0.5,0,1", **kw)
    assert pc.net.n_out == 3 * 4
    a = pc.action_fn(np.eye(4, dtype=np.float32)[[1, 3, 0]].reshape(1, 12))
    np.testing.assert_allclose(a[0], [-0.2, 1.0, 0.0], rtol=1e-6)


def test_bench_without_warmup_prints_line_and_dumps_seeded_outputs(tmp_path):
    """bench.py at a tiny size with --warmup 0 (the e2e window opens before run_master's first iteration) prints its one
    JSON line; the timed region's kernel launches scale with --steps (two timed generations launch exactly twice what one
    does); --dump-outputs writes the last generation's arrays (float32, <= 64 MB, actions = argmax of the dumped logits);
    a second run with the same arguments sees the same inputs and computes the same outputs."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

    def bench(steps, d):
        out = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", "0",
                              "--pop", "8", "--episode-len", "20", "--noise-count", str(NOISE_COUNT), "--no-cpu-baseline",
                              "--dump-outputs", str(d)], capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-3000:]
        line = json.loads(out.stdout.strip().splitlines()[-1])
        assert line["steps"] == steps and line["warmup"] == 0 and line["value"] > 0 and line["e2e"]["value"] > 0
        return line, {k: np.load(d / f"{k}.npy") for k in ("theta", "grad", "returns", "logits", "actions")}

    one, _ = bench(1, tmp_path / "d1")
    two, a = bench(2, tmp_path / "d2")
    again, b = bench(2, tmp_path / "d3")
    assert one["gpu_launches"] > 0 and two["gpu_launches"] == 2 * one["gpu_launches"]
    assert a["theta"].shape == (4052658,) and a["grad"].shape == (4052658,) and a["returns"].shape == (4, 2)
    assert a["logits"].shape == (8, 18) and a["actions"].shape == (8,)
    assert all(v.dtype == np.float32 for v in a.values()) and sum(v.nbytes for v in a.values()) <= 64 << 20
    np.testing.assert_array_equal(a["actions"], np.argmax(a["logits"], axis=1))
    assert np.abs(a["grad"]).max() > 0
    for k in a:
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)
