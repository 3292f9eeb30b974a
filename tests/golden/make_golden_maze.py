"""Writes tests/golden/ref_maze.npz from the reference's own maze code, through oracle/_ref/maze_ref (oracle/maze_ref.cpp,
built by __graft_entry__.build() when the reference checkout is present).

    python tests/golden/make_golden_maze.py

Arrays (float32 unless noted):
  reset_obs [11]                      the observation of the reset state
  step_in [N, 9], step_out [N, 19]    single steps on the hard maze: (x, y, heading, speed, ang_vel, collide, t, a0, a1)
                                      -> (x, y, heading, speed, ang_vel, collide, t, reward, obs[11])
  sticky_in / sticky_out              the same on the hard maze with its collision flag set (collisions stick)
  ep_actions [E, 400, 2]              open-loop action sequences from the reset state
  ep_out [E, 400, 19]                 per step, the 19 outputs above
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
MAZE = os.path.join(HERE, "hard_maze.txt")
DRIVER = os.path.join(ROOT, "oracle", "_ref", "maze_ref")
T = 400


def run(maze, mode, data, *extra):
    p = subprocess.run([DRIVER, maze, mode, *extra], input=np.ascontiguousarray(data, np.float32).tobytes(),
                       capture_output=True, check=True)
    return np.frombuffer(p.stdout, np.float32)


def walls():
    tok = open(MAZE).read().split()
    n = int(tok[2])
    return np.array([float(t) for t in tok[10:10 + 4 * n]]).reshape(n, 4)


def single_step_inputs(rs):
    W = walls()
    rows = []

    def add(x, y, h, sp, av, col, t, a0, a1):
        rows.append([x, y, h, sp, av, col, t, a0, a1])

    # random states inside the maze's bounding box, actions around [-0.5, 0.5] and beyond
    for _ in range(2000):
        add(rs.uniform(0, 200), rs.uniform(0, 210), rs.uniform(0, 360), rs.uniform(-3, 3), rs.uniform(-3, 3), 0,
            rs.randint(0, T), rs.normal(0, 0.4), rs.normal(0, 0.4))
    # wall contact: the next position lands about one radius (8) from a wall, at its ends too
    for _ in range(800):
        ax, ay, bx, by = W[rs.randint(len(W))]
        u = rs.choice([rs.uniform(0, 1), rs.uniform(-0.05, 0.0), rs.uniform(1.0, 1.05)])
        px, py = ax + u * (bx - ax), ay + u * (by - ay)
        nrm = np.array([-(by - ay), bx - ax]) / np.hypot(bx - ax, by - ay) * rs.choice([-1, 1])
        d = 8.0 + rs.choice([0.0, 1e-5, -1e-5, 1e-3, -1e-3, rs.uniform(-1, 1)])
        h = rs.uniform(0, 360)
        sp = rs.uniform(-3, 3)
        hr = h / 180.0 * 3.1415926
        x, y = px + d * nrm[0] - np.cos(hr) * sp, py + d * nrm[1] - np.sin(hr) * sp
        add(x, y, h, sp, rs.uniform(-3, 3), 0, rs.randint(0, T), sp / 6.0, rs.normal(0, 0.3))
    # grazing rays: a rangefinder parallel (or nearly) to a wall
    sensors = (-90.0, -45.0, 0.0, 45.0, 90.0, -180.0)
    for _ in range(500):
        ax, ay, bx, by = W[rs.randint(len(W))]
        wall_deg = np.degrees(np.arctan2(by - ay, bx - ax))
        h = (wall_deg - rs.choice(sensors) + rs.choice([0.0, 180.0]) + rs.choice([0.0, 1e-4, -1e-4, 1e-2])) % 360.0
        u = rs.uniform(-0.2, 1.2)
        off = rs.choice([0.0, 1e-3, -1e-3, 0.5, -0.5, 9.0])
        nrm = np.array([-(by - ay), bx - ax]) / np.hypot(bx - ax, by - ay)
        add(ax + u * (bx - ax) + off * nrm[0], ay + u * (by - ay) + off * nrm[1], h, 0.0, 0.0, 0, 0, 0.0, 0.0)
    # heading near 0 / 360 with turns across the wrap
    for _ in range(300):
        h = rs.choice([0.0, 1e-6, 1e-3, 0.1, 359.9, 359.999, 360.0 - 1e-5, 360.0, 360.1, -1e-3])
        av = rs.choice([-3.0, -0.2, -1e-3, 0.0, 1e-3, 0.2, 3.0])
        add(rs.uniform(20, 180), rs.uniform(20, 190), h, rs.uniform(-3, 3), av, 0, rs.randint(0, T),
            rs.choice([-0.5, -0.0333, 0.0, 0.0333, 0.5, rs.normal(0, 0.3)]), rs.normal(0, 0.3))
    # speed and turn at their clamps, rate limits exactly at +-0.2, actions outside [-0.5, 0.5]
    for _ in range(400):
        sp, av = rs.choice([-3.0, -2.9, -2.95, 2.9, 2.95, 3.0]), rs.choice([-3.0, -2.9, 2.9, 3.0, 0.1])
        a0 = rs.choice([-5.0, -1.0, -0.6, -0.5, 0.5, 0.6, 1.0, 5.0, av / 6.0 + 0.2 / 6.0, rs.normal(0, 1)])
        a1 = rs.choice([-5.0, -1.0, -0.6, -0.5, 0.5, 0.6, 1.0, 5.0, sp / 6.0 - 0.2 / 6.0, rs.normal(0, 1)])
        add(rs.uniform(20, 180), rs.uniform(20, 190), rs.uniform(0, 360), sp, av, 0, rs.randint(0, T), a0, a1)
    # the reward step (t 399 -> 400), and past it
    for _ in range(300):
        add(rs.uniform(0, 200), rs.uniform(0, 210), rs.uniform(0, 360), rs.uniform(-3, 3), rs.uniform(-3, 3), 0,
            rs.choice([398, 399, 400, 450]), rs.normal(0, 0.4), rs.normal(0, 0.4))
    # NaN and infinity in the actions and in the state; a collided hero
    nan, inf = np.nan, np.inf
    for a0, a1 in ((nan, 0.1), (0.1, nan), (nan, nan), (inf, -inf), (-inf, 0.2)):
        for t in (0, 399):
            add(rs.uniform(40, 160), rs.uniform(40, 160), rs.uniform(0, 360), 1.0, 0.5, 0, t, a0, a1)
    for x, y, h, sp, av in ((nan, 100.0, 10.0, 1.0, 0.0), (100.0, nan, 10.0, 1.0, 0.0), (100.0, 100.0, nan, 1.0, 0.0),
                            (100.0, 100.0, 10.0, nan, 0.0), (100.0, 100.0, 10.0, 1.0, nan), (inf, 100.0, 10.0, 1.0, 0.0)):
        for t in (0, 399):
            add(x, y, h, sp, av, 0, t, 0.1, 0.1)
    for _ in range(40):
        add(rs.uniform(0, 200), rs.uniform(0, 210), rs.uniform(0, 360), rs.uniform(-3, 3), rs.uniform(-3, 3), 1,
            rs.choice([0, 399]), rs.normal(0, 0.4), rs.normal(0, 0.4))
    return np.array(rows, np.float32)


def episode_actions(rs, E=32):
    acts = []
    for e in range(E):
        kind = e % 8
        if kind == 0:                       # white noise
            a = rs.normal(0, 0.3, (T, 2))
        elif kind == 1:                     # smooth (AR(1)) wandering
            a = np.zeros((T, 2))
            for t in range(1, T):
                a[t] = 0.95 * a[t - 1] + rs.normal(0, 0.08, 2)
        elif kind == 2:                     # full speed ahead, a fixed turn: runs into walls and hugs them
            a = np.tile([rs.uniform(-0.1, 0.1), 0.5], (T, 1))
        elif kind == 3:                     # full speed with saturated, out-of-range turns that switch
            a = np.tile([rs.choice([-2.0, 2.0]), 1.5], (T, 1))
            a[rs.randint(0, T, 20), 0] *= -1
        elif kind == 4:                     # reverse into the walls
            a = np.tile([rs.normal(0, 0.05), -0.5], (T, 1)) + rs.normal(0, 0.02, (T, 2))
        elif kind == 5:                     # spinning in place across the heading wrap
            a = np.tile([rs.choice([-0.5, 0.5]), 0.0], (T, 1))
        elif kind == 6:                     # bang-bang
            a = rs.choice([-0.5, 0.5], (T, 2))
        else:                               # smooth, with a NaN action partway
            a = np.cumsum(rs.normal(0, 0.05, (T, 2)), axis=0).clip(-0.6, 0.6)
            if e == 7:
                a[rs.randint(100, 300), rs.randint(2)] = np.nan
        acts.append(a)
    return np.array(acts, np.float32)


def main():
    if not os.path.exists(DRIVER):
        sys.exit(f"{DRIVER} not built: run __graft_entry__.build() with the reference checkout present")
    rs = np.random.RandomState(20260)
    out = {"reset_obs": run(MAZE, "reset", np.zeros(0))}
    step_in = single_step_inputs(rs)
    out["step_in"], out["step_out"] = step_in, run(MAZE, "step", step_in).reshape(-1, 19)
    with tempfile.TemporaryDirectory() as d:
        sticky = os.path.join(d, "sticky_maze.txt")
        with open(sticky, "w") as f:
            f.write("1\n" + open(MAZE).read().split("\n", 1)[1])
        sticky_in = step_in[np.r_[800:1600, 0:200]]       # the wall-contact states, and some random ones
        out["sticky_in"], out["sticky_out"] = sticky_in, run(sticky, "step", sticky_in).reshape(-1, 19)
    acts = episode_actions(rs)
    out["ep_actions"], out["ep_out"] = acts, run(MAZE, "episode", acts, str(T)).reshape(len(acts), T, 19)
    path = os.path.join(HERE, "ref_maze.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {len(step_in)} single steps, {len(acts)} episodes, {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    main()
