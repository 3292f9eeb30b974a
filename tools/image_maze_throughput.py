"""Per-tick runner throughput on the image hard maze against the synthetic Atari stand-in (needs an H100).

    python tools/image_maze_throughput.py [--slots 256] [--policy LargeModelPolicy] [--out FILE.json]

One process, for each environment (ImageHardMaze-v0, then SyntheticAtariEnv with the same 9 actions and 400-step
episodes): dne.rollout.RolloutRunner at `--slots` slots (two half-tables, GA units of one member) plays one 400-step
episode per slot after a warm-up run, and reports
  * env-steps/s over the timed run (host clock, the run ends in a device synchronise);
  * ms per tick (one forward of each half-table, wall clock / ticks * 2);
  * the environment step's host time per half-tick: ImageMazeEnv.step is an upload, the step-and-render launch, the copy
    back and the stream synchronise; SyntheticAtariEnv.step is host numpy.  The rest of a tick is the forward and the
    runner's own host work;
  * the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-neuroevolution_b200")]

import numpy as np   # noqa: E402
import torch         # noqa: E402

from dne.envs import ImageMazeEnv, SyntheticAtariEnv    # noqa: E402
from dne.rollout import RolloutRunner, Unit             # noqa: E402
from es_distributed import es as ES                     # noqa: E402
from es_distributed import policies                     # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def measure(env, policy, n_slots, seed=0):
    step_s = [0.0, 0]
    inner = env.step

    def timed_step(slots, actions):
        t0 = time.perf_counter()
        out = inner(slots, actions)
        step_s[0] += time.perf_counter() - t0
        step_s[1] += 1
        return out
    env.step = timed_step
    runner = RolloutRunner(ES.default_context(), policy.net, env, n_slots, group=1, pipeline=2)
    P = policy.num_params
    rs = np.random.RandomState(seed)
    units = [Unit(int(rs.randint(0, ES.default_noise().count - P)), (np.float32(0.005),)) for _ in range(n_slots)]
    theta = policy.device_theta
    runner.run(theta, units, 20)                                  # warm-up: every shape of the timed run
    torch.cuda.synchronize()
    step_s[:] = [0.0, 0]
    t0 = time.perf_counter()
    res = runner.run(theta, units, 400)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return {"env": type(env).__name__, "slots": n_slots, "steps": int(res.steps), "ticks": int(res.ticks),
            "wall_s": round(wall, 4), "env_steps_per_s": round(res.steps / wall, 1),
            "ms_per_tick": round(wall / res.ticks * 2 * 1e3, 4),
            "env_step_ms_per_half_tick": round(step_s[0] / max(step_s[1], 1) * 1e3, 4),
            "env_step_share": round(step_s[0] / wall, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=256)
    ap.add_argument("--policy", default="LargeModelPolicy")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    ES.default_noise()                                           # the drivers' default table
    envs = [ImageMazeEnv(a.slots), SyntheticAtariEnv(a.slots, num_actions=9, episode_len=400, seed=1)]
    policy = getattr(policies, a.policy)(envs[0].observation_space, envs[0].action_space, seed=0)
    out = {"card": card(), "policy": a.policy, "results": [measure(e, policy, a.slots) for e in envs]}
    print(json.dumps(out, indent=1))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
