"""Hard-maze throughput of the continuous episode kernel (needs an H100).

    python tools/maze_throughput.py [--launches 20] [--gens 10] [--hidden 256 256] [--cluster {0,2,4,8}]
                                    [--ac-bins uniform:10] [--out FILE.json]

Reports, from one process, for configurations/hardmaze_nses.json (MujocoPolicy, 400-step episodes; --hidden replaces its
hidden_dims, e.g. the reference's humanoid [256, 256]):
  * the kernel time of dne_maze_episodes (CUDA events over --launches back-to-back launches after 3 warm-up launches,
    with observation statistics, action noise and per-member observation sums) and env-steps/s, at the config's
    population (episodes_per_batch) and at 5000 members;
  * the generation wall-clock of es_distributed.nses.run_master on that configuration (median over generations
    2..gens);
  * the card's name and power limit, read in the same run.
The kernel is dne_maze_episodes when the net fits one CTA, otherwise dne_maze_cluster_episodes at the automatic cluster
size, as MazeEnv launches it; --cluster forces the cluster entry at that size (0: automatic), and the result then also
reports its geometry (cluster size, threads and shared bytes per CTA, resident members).  --gens 0 skips the generation.
--ac-bins (a MujocoPolicy head, e.g. uniform:10 or custom:-1,0,1) also times dne_maze_binned_episodes for the same
hidden sizes and members (binned_kernel_*), beside the continuous kernel; the generation then runs with that head.
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
from dne.envs import MazeEnv                     # noqa: E402
from es_distributed import es as ES              # noqa: E402
from es_distributed import nses as NS            # noqa: E402
from es_distributed import policies              # noqa: E402

CONFIG = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations", "hardmaze_nses.json")
T = 400


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def time_kernel(ctx, net, theta, n, launches, seed=0, cluster=None, bins=None):
    dev = torch.device("cuda", 0)
    rs = np.random.RandomState(seed)
    P = net.num_params
    n -= n % 2
    env = MazeEnv(n)
    idx = np.repeat(rs.randint(0, ES.default_noise().count - P + 1, size=n // 2), 2).astype(np.int64)
    scale = np.tile([0.05, -0.05], n // 2).astype(np.float32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)          # noqa: E731
    d_idx, d_sc, d_init = t(idx), t(scale), t(env.initial_states(n))
    d_mean, d_std = t(np.zeros(11, np.float32)), t(np.full(11, 0.5, np.float32))
    d_ac = t((rs.randn(n, T, 2) * 0.01).astype(np.float32))
    d_ret, d_sret = torch.empty(n, device=dev), torch.empty(n, device=dev)
    d_len = torch.empty(n, dtype=torch.int32, device=dev)
    d_fin = torch.empty(n, 7, dtype=torch.float64, device=dev)
    d_s, d_q = torch.empty(n, 11, dtype=torch.float64, device=dev), torch.empty(n, 11, dtype=torch.float64, device=dev)
    th = theta.contiguous()

    args = (C.byref(env.desc), C.byref(net.desc), F.ptr(th), F.ptr(d_idx), F.ptr(d_sc), None, n, F.ptr(d_init), T,
            F.ptr(d_mean), F.ptr(d_std), F.ptr(d_ac), F.ptr(d_ret), F.ptr(d_sret), F.ptr(d_len), F.ptr(d_fin), F.ptr(d_s),
            F.ptr(d_q))
    if bins is not None:
        tab = np.ascontiguousarray(bins, dtype=np.float32)
    elif cluster is None and F.lib().dne_maze_net_supported(C.byref(net.desc)) != 0:
        cluster = 0                                   # MazeEnv's choice for a net too wide for one CTA

    def launch():
        if bins is not None:                          # one CTA when the member fits one, as MazeEnv launches it
            F.check(F.lib().dne_maze_binned_episodes(ctx.handle, *args, tab.ctypes.data_as(C.c_void_p), tab.shape[1],
                                                     cluster or 0, F.stream_ptr()))
        elif cluster is None:
            F.check(F.lib().dne_maze_episodes(ctx.handle, *args, F.stream_ptr()))
        else:
            F.check(F.lib().dne_maze_cluster_episodes(ctx.handle, *args, cluster, F.stream_ptr()))
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
        res["cluster_geometry"] = F.cluster_geometry("maze", net.desc, cluster)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--gens", type=int, default=10)
    ap.add_argument("--hidden", type=int, nargs="+", default=None, help="hidden_dims instead of the config's")
    ap.add_argument("--cluster", type=int, choices=(0, 2, 4, 8), default=None,
                    help="force dne_maze_cluster_episodes at this cluster size (0: automatic)")
    ap.add_argument("--ac-bins", default=None, help="also time this discretised head (e.g. uniform:10)")
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
    ctx = ES.default_context()
    env = MazeEnv(8)
    pol = policies.MujocoPolicy(env.observation_space, env.action_space, seed=0, **exp["policy"]["args"])
    out["kernel_config_population"] = time_kernel(ctx, pol.net, pol.device_theta, exp["config"]["episodes_per_batch"],
                                                  args.launches, cluster=args.cluster)
    out["kernel_5000"] = time_kernel(ctx, pol.net, pol.device_theta, 5000, args.launches, cluster=args.cluster)
    if args.ac_bins:
        exp["policy"]["args"]["ac_bins"] = out["ac_bins"] = args.ac_bins
        bp = policies.MujocoPolicy(env.observation_space, env.action_space, seed=0, **exp["policy"]["args"])
        for key, n in (("binned_kernel_config_population", exp["config"]["episodes_per_batch"]),
                       ("binned_kernel_5000", 5000)):
            out[key] = time_kernel(ctx, bp.net, bp.device_theta, n, args.launches, cluster=args.cluster,
                                   bins=bp._bin_values)
    if args.gens > 0:
        gens = []
        NS.run_master(None, None, exp, max_iterations=args.gens, seed=0,
                      on_iteration=lambda it, st, ex: gens.append(st["TimeElapsedThisIter"]))
        out["generation_wallclock_s_median"] = float(np.median(gens[1:])) if len(gens) > 1 else gens[0]
    out["card_after"] = card()
    print(json.dumps(out, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
