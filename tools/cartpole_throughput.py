"""CartPole-v1 (or Acrobot-v1 / MountainCar-v0) throughput of the fused episode kernel at the es_gym_config population
(needs an H100).

    python tools/cartpole_throughput.py [--env CartPole-v1] [--gens 45] [--launches 50] [--out FILE.json]

Population: 5000 episodes per generation = 2500 antithetic pairs plus the 1 % evaluation share (eval_prob 0.01 of the
2500 pairs: 25 episodes, run as 13 noiseless pairs), SimpleClassifier, noise_stdev 0.02, the 500-step limit.
Reports, from one process:
  * the kernel time of dne_cartpole_episodes (CUDA events over --launches back-to-back launches after 3 warm-up launches)
    and env-steps/s (the steps those launches executed / kernel time), for the initial weights and for the weights after
    --gens generations of configurations/cartpole_es.json (longer episodes);
  * the generation wall-clock of es_distributed.es.run_master on that configuration (median over generations 2..gens);
  * the card's name and power limit, read in the same run.
--env Acrobot-v1 / MountainCar-v0 runs the same population of SimpleClassifier members (3 actions) through
dne_discrete_episodes at the task's time limit, the trained weights coming from --gens generations of
configurations/acrobot_es.json (ES) / mountaincar_ga.json (GA, the elite's weights).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-neuroevolution_b200")]

import numpy as np   # noqa: E402
import torch         # noqa: E402

from dne import _ffi as F                        # noqa: E402
from dne import nets                             # noqa: E402
from dne.envs import AcrobotEnv, CartPoleEnv, MountainCarEnv   # noqa: E402
from es_distributed import es as ES              # noqa: E402
from es_distributed import ga as GA              # noqa: E402
from es_distributed import policies              # noqa: E402

CONFIGS = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations")
# env id -> (environment, DNE_EPISODE_* id, configuration, ob_dim, actions)
TASKS = {"CartPole-v1": (CartPoleEnv, F.EPISODE_CARTPOLE, "cartpole_es.json", 4, 2),
         "Acrobot-v1": (AcrobotEnv, F.EPISODE_ACROBOT, "acrobot_es.json", 6, 3),
         "MountainCar-v0": (MountainCarEnv, F.EPISODE_MOUNTAINCAR, "mountaincar_ga.json", 2, 3)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def time_kernel(ctx, net, theta, n_pairs, n_eval_pairs, launches, seed=0, env_id="CartPole-v1"):
    """CUDA-event time of `launches` dne_cartpole_episodes (dne_discrete_episodes for the other tasks) launches over one
    generation's members."""
    env_cls, episode_env = TASKS[env_id][:2]
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(seed)
    P = net.num_params
    n = 2 * (n_pairs + n_eval_pairs)
    pidx = rs.randint(0, ES.default_noise().count - P + 1, size=n_pairs)
    idx = np.concatenate([np.repeat(pidx, 2), np.zeros(2 * n_eval_pairs, np.int64)]).astype(np.int64)
    scale = np.concatenate([np.tile([0.02, -0.02], n_pairs), np.zeros(2 * n_eval_pairs)]).astype(np.float32)
    init = env_cls(n, seed=seed).initial_states(n)
    limit = env_cls(1).max_episode_steps
    th = theta.contiguous()
    d_idx, d_sc = torch.from_numpy(idx).to(dev), torch.from_numpy(scale).to(dev)
    d_init = torch.from_numpy(init).to(dev)
    d_ret = torch.empty(n, dtype=torch.float32, device=dev)
    d_len = torch.empty(n, dtype=torch.int32, device=dev)

    def launch():
        if env_id == "CartPole-v1":
            F.check(F.lib().dne_cartpole_episodes(ctx.handle, C.byref(net.desc), F.ptr(th), F.ptr(d_idx), F.ptr(d_sc), None,
                                                  n, F.ptr(d_init), 500, F.ptr(d_ret), F.ptr(d_len), None, F.stream_ptr()))
        else:
            F.check(F.lib().dne_discrete_episodes(ctx.handle, episode_env, C.byref(net.desc), F.ptr(th), F.ptr(d_idx),
                                                  F.ptr(d_sc), None, n, F.ptr(d_init), limit, F.ptr(d_ret), F.ptr(d_len),
                                                  None, F.stream_ptr()))
    for _ in range(3):
        launch()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        launch()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / launches
    steps = int(d_len.sum().item())                    # every launch runs the same episodes (deterministic)
    return {"members": n, "launches": launches, "kernel_ms": ms, "steps_per_launch": steps,
            "mean_length": steps / n, "env_steps_per_s": steps / (ms * 1e-3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--env", choices=sorted(TASKS), default="CartPole-v1")
    ap.add_argument("--gens", type=int, default=45)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    out = {"card": card()}
    env_cls, _, config, ob_dim, n_act = TASKS[args.env]
    if args.env != "CartPole-v1":
        out["env"] = args.env
    with open(os.path.join(CONFIGS, config)) as f:
        exp = json.load(f)
    exp["config"]["snapshot_freq"] = 0
    # the es_gym_config population: 5000 episodes, a 1 % evaluation share
    n_pairs = 5000 // 2
    n_eval_pairs = -(-int(round(n_pairs * 0.01)) // 2)
    ctx = ES.default_context()
    net = nets.make_net("SimpleClassifier", num_actions=n_act, ob_dim=ob_dim)
    env = env_cls(8, seed=0)
    pol = policies.SimpleClassifierPolicy(env.observation_space, env.action_space, seed=0)
    out["kernel_initial_theta"] = time_kernel(ctx, net, pol.device_theta, n_pairs, n_eval_pairs, args.launches,
                                              env_id=args.env)

    gens = []

    def on_it(it, st, ex):
        gens.append((st["TimeElapsedThisIter"], st.get("EpLenMean", 0.0), st.get("EpisodesThisIter", 0),
                     st.get("EvalEpCount", 0)))
        if "elite_theta" in ex:
            out["_elite"] = ex["elite_theta"].clone()
    if "population_size" in exp:                                   # the GA configuration
        GA.run_master(None, None, exp, max_iterations=args.gens, env=env, seed=0, on_iteration=on_it)
        theta = out.pop("_elite")
    else:
        theta = ES.run_master(None, None, exp, max_iterations=args.gens, env=env, seed=0, on_iteration=on_it)
    theta = theta if torch.is_tensor(theta) else torch.from_numpy(theta).cuda()
    out["kernel_trained_theta"] = time_kernel(ctx, net, theta, n_pairs, n_eval_pairs, args.launches, env_id=args.env)
    out["generations"] = [{"seconds": g[0], "ep_len_mean": g[1], "episodes": g[2], "eval_episodes": g[3]} for g in gens]
    out["generation_wallclock_s_median"] = float(np.median([g[0] for g in gens[1:]])) if len(gens) > 1 else gens[0][0]
    out["generation_wallclock_s_last"] = gens[-1][0]
    out["card_after"] = card()
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
