"""Pendulum-v1 throughput of the fused episode kernel (needs an H100).

    python tools/pendulum_throughput.py [--launches 50] [--gens 10] [--per-tick-members 256] [--hidden 256 256]
                                        [--cluster {0,2,4,8}] [--ac-bins uniform:5] [--out FILE.json]

Reports, from one process, for configurations/pendulum_es.json (MujocoPolicy, 200-step episodes; --hidden replaces its
hidden_dims, e.g. the reference's humanoid [256, 256]):
  * the kernel time of dne_pendulum_episodes (CUDA events over --launches back-to-back launches after 3 warm-up launches,
    with observation statistics, action noise and per-member observation sums) and env-steps/s, at the config's
    population and at about 5000 members;
  * the generation wall-clock of es_distributed.es.run_master on that configuration (median over generations 2..gens);
  * the per-tick RolloutRunner stepping the host PendulumEnv against EpisodeKernelRunner on the same members,
    alternated (three rounds each, wall-clock per run() including its host sync);
  * at the config's population, the wall-clock of one EpisodeKernelRunner.run() with statistics sampling and action
    noise, and of its host-side action-noise draw (randn + float32 scaling + copy to the device) alone (medians of 5);
  * the card's name and power limit, read in the same run.
The kernel is dne_pendulum_episodes when the net fits one CTA, otherwise dne_pendulum_cluster_episodes at the automatic
cluster size, as PendulumEnv launches it; --cluster forces the cluster entry at that size (0: automatic), and the kernel
results then also report its geometry (cluster size, threads and shared bytes per CTA, resident members).  --gens 0
skips the generation and the runner costs, --per-tick-members 0 the per-tick comparison.
--ac-bins (a MujocoPolicy head, e.g. uniform:5) also times dne_pendulum_binned_episodes for the same hidden sizes and
members (binned_kernel_*), beside the continuous kernel, and the per-tick RolloutRunner with the policy's host action_fn
against EpisodeKernelRunner(action_bins=...) (binned_per_tick_vs_kernel).
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-neuroevolution_b200")]

import numpy as np   # noqa: E402
import torch         # noqa: E402

from dne import _ffi as F                        # noqa: E402
from dne.envs import PendulumEnv                 # noqa: E402
from dne.rollout import EpisodeKernelRunner, RolloutRunner, Unit   # noqa: E402
from es_distributed import es as ES              # noqa: E402
from es_distributed import policies              # noqa: E402

CONFIG = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations", "pendulum_es.json")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def time_kernel(ctx, net, theta, n, launches, seed=0, cluster=None, bins=None):
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(seed)
    P, T = net.num_params, 200
    n -= n % 2
    idx = np.repeat(rs.randint(0, ES.default_noise().count - P + 1, size=n // 2), 2).astype(np.int64)
    scale = np.tile([0.02, -0.02], n // 2).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)          # noqa: E731
    d_idx, d_sc, d_init = t(idx), t(scale), t(PendulumEnv(n, seed=seed, pin=False).initial_states(n))
    d_mean, d_std = t(np.zeros(3, np.float32)), t(np.array([0.7, 0.7, 3.0], np.float32))
    d_ac = t((rs.randn(n, T, 1) * 0.01).astype(np.float32))
    d_ret, d_sret = torch.empty(n, device=dev), torch.empty(n, device=dev)
    d_len = torch.empty(n, dtype=torch.int32, device=dev)
    d_s, d_q = torch.empty(n, 3, dtype=torch.float64, device=dev), torch.empty(n, 3, dtype=torch.float64, device=dev)
    th = theta.contiguous()

    args = (C.byref(net.desc), F.ptr(th), F.ptr(d_idx), F.ptr(d_sc), None, n, F.ptr(d_init), T, F.ptr(d_mean),
            F.ptr(d_std), F.ptr(d_ac), F.ptr(d_ret), F.ptr(d_sret), F.ptr(d_len), None, F.ptr(d_s), F.ptr(d_q))
    if bins is not None:
        tab = np.ascontiguousarray(bins, dtype=np.float32)
    elif cluster is None and F.lib().dne_pendulum_net_supported(C.byref(net.desc)) != 0:
        cluster = 0                                   # PendulumEnv's choice for a net too wide for one CTA

    def launch():
        if bins is not None:                          # one CTA when the member fits one, as PendulumEnv launches it
            F.check(F.lib().dne_pendulum_binned_episodes(ctx.handle, *args, tab.ctypes.data_as(C.c_void_p),
                                                         tab.shape[1], cluster or 0, F.stream_ptr()))
        elif cluster is None:
            F.check(F.lib().dne_pendulum_episodes(ctx.handle, *args, F.stream_ptr()))
        else:
            F.check(F.lib().dne_pendulum_cluster_episodes(ctx.handle, *args, cluster, F.stream_ptr()))
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
    res = {"members": n, "launches": launches, "kernel_ms": ms, "env_steps_per_s": n * T / (ms * 1e-3)}
    if cluster is not None and bins is None:
        res["cluster_geometry"] = F.cluster_geometry("pendulum", net.desc, cluster)
    return res


def per_tick_vs_kernel(ctx, net, theta, n, rounds=3, pol=None):
    """pol: a discretised-head policy, whose bins the kernel runner takes and whose action_fn the per-tick one."""
    rs = np.random.RandomState(1)
    units = [Unit(int(rs.randint(0, ES.default_noise().count - net.num_params)), (0.02, -0.02)) for _ in range(n // 2)]
    mean, std = torch.zeros(3, device="cuda"), torch.tensor([0.7, 0.7, 3.0], device="cuda")
    runners = {"kernel": EpisodeKernelRunner(ctx, net, PendulumEnv(n, seed=2), group=2,
                                             action_bins=None if pol is None else pol._bin_values),
               "per_tick": RolloutRunner(ctx, net, PendulumEnv(n, seed=2), n, group=2, pipeline=2)}
    runners["per_tick"].action_fn = None if pol is None else pol.action_fn
    out = {k: [] for k in runners}
    for name, r in runners.items():                     # warm-up
        r.run(theta, units, None, ob_mean=mean, ob_std=std)
    for _ in range(rounds):
        for name, r in runners.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r.run(theta, units, None, ob_mean=mean, ob_std=std)
            out[name].append(time.perf_counter() - t0)
    res = {"members": n, "steps_per_run": n * 200}
    for k, v in out.items():
        res[k + "_s"] = v
        res[k + "_env_steps_per_s"] = n * 200 / float(np.median(v))
    res["speedup"] = float(np.median(out["per_tick"]) / np.median(out["kernel"]))
    return res


def runner_costs(ctx, net, theta, n_pairs, reps=5):
    rs = np.random.RandomState(3)
    units = [Unit(int(rs.randint(0, ES.default_noise().count - net.num_params)), (0.05, -0.05)) for _ in range(n_pairs)]
    mean, std = torch.zeros(3, device="cuda"), torch.tensor([0.7, 0.7, 3.0], device="cuda")
    r = EpisodeKernelRunner(ctx, net, PendulumEnv(8, seed=2), group=2)
    run_s, draw_s = [], []
    for i in range(reps + 1):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r.run(theta, units, None, ob_mean=mean, ob_std=std, ac_noise_std=0.01,
              random_stream=np.random.RandomState(i), save_obs_prob=0.01)
        run_s.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        a = np.random.RandomState(i).randn(2 * n_pairs, 200, 1).astype(np.float32) * np.float32(0.01)
        torch.from_numpy(a).to("cuda")
        torch.cuda.synchronize()
        draw_s.append(time.perf_counter() - t0)
    return {"members": 2 * n_pairs, "run_ms_median": 1e3 * float(np.median(run_s[1:])),
            "action_noise_draw_ms_median": 1e3 * float(np.median(draw_s[1:]))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--per-tick-members", type=int, default=256)
    ap.add_argument("--hidden", type=int, nargs="+", default=None, help="hidden_dims instead of the config's")
    ap.add_argument("--cluster", type=int, choices=(0, 2, 4, 8), default=None,
                    help="force dne_pendulum_cluster_episodes at this cluster size (0: automatic) in the kernel timings")
    ap.add_argument("--ac-bins", default=None, help="also time this discretised head (e.g. uniform:5)")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    out = {"card": card()}
    with open(CONFIG) as f:
        exp = json.load(f)
    exp["config"]["snapshot_freq"] = 0
    if args.hidden:
        exp["policy"]["args"]["hidden_dims"] = args.hidden
        out["hidden_dims"] = args.hidden
    cfg = exp["config"]
    ctx = ES.default_context()
    env = PendulumEnv(8, seed=0)
    pol = policies.MujocoPolicy(env.observation_space, env.action_space, seed=0, **exp["policy"]["args"])
    n_cfg = cfg["episodes_per_batch"] + 2 * -(-int(round(cfg["episodes_per_batch"] // 2 * cfg["eval_prob"])) // 2)
    out["kernel_config_population"] = time_kernel(ctx, pol.net, pol.device_theta, n_cfg, args.launches,
                                                  cluster=args.cluster)
    out["kernel_5000"] = time_kernel(ctx, pol.net, pol.device_theta, 5000, args.launches, cluster=args.cluster)
    if args.gens > 0:
        gens = []
        ES.run_master(None, None, exp, max_iterations=args.gens, env=env, seed=0,
                      on_iteration=lambda it, st, ex: gens.append(st["TimeElapsedThisIter"]))
        out["generation_wallclock_s_median"] = float(np.median(gens[1:])) if len(gens) > 1 else gens[0]
        out["runner_costs"] = runner_costs(ctx, pol.net, pol.device_theta, cfg["episodes_per_batch"] // 2)
    if args.per_tick_members > 0:
        out["per_tick_vs_kernel"] = per_tick_vs_kernel(ctx, pol.net, pol.device_theta, args.per_tick_members)
    if args.ac_bins:
        out["ac_bins"] = args.ac_bins
        bp = policies.MujocoPolicy(env.observation_space, env.action_space, seed=0,
                                   **dict(exp["policy"]["args"], ac_bins=args.ac_bins))
        for key, n in (("binned_kernel_config_population", n_cfg), ("binned_kernel_5000", 5000)):
            out[key] = time_kernel(ctx, bp.net, bp.device_theta, n, args.launches, cluster=args.cluster,
                                   bins=bp._bin_values)
        if args.per_tick_members > 0:
            out["binned_per_tick_vs_kernel"] = per_tick_vs_kernel(ctx, bp.net, bp.device_theta, args.per_tick_members,
                                                                  pol=bp)
    out["card_after"] = card()
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
