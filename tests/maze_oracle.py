"""Scalar referee of the hard maze (DESIGN.md 3.7): the reference's single-precision C++ (gym_tensorflow/maze/maze.h and
tf_maze.cpp's step) restated operation by operation in numpy float32 scalars, with Python floats where the C++ promotes
to double, and glibc's own cosf / sinf / atanf / sqrtf / cos / sin through ctypes.  numpy's float32 transcendentals are
not used: they differ from glibc's by an ulp on some arguments.  tests/test_maze_host.py checks it bit for bit against
tests/golden/ref_maze.npz, written by the reference's code itself (oracle/maze_ref.cpp).

State: (x, y, heading, speed, ang_vel) float32, ``collide`` (bool), ``t`` (steps taken)."""
import ctypes as C
import ctypes.util
import math
import os
from typing import NamedTuple

import numpy as np

_m = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
for _name, _t in (("cosf", C.c_float), ("sinf", C.c_float), ("atanf", C.c_float), ("sqrtf", C.c_float),
                  ("cos", C.c_double), ("sin", C.c_double)):
    getattr(_m, _name).restype = _t
    getattr(_m, _name).argtypes = [_t]

f32 = np.float32
MAZE_STEPS = 400
RADIUS = f32(8.0)
RANGE = f32(100.0)
RANGEFINDER_ANGLES = (-90.0, -45.0, 0.0, 45.0, 90.0, -180.0)
RADAR = ((315.0, 405.0), (45.0, 135.0), (135.0, 225.0), (225.0, 315.0))
FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hard_maze.txt")


def cosf(v):
    return f32(_m.cosf(float(v)))


def sinf(v):
    return f32(_m.sinf(float(v)))


def atanf(v):
    return f32(_m.atanf(float(v)))


def sqrtf(v):
    return f32(_m.sqrtf(float(v)))


def deg2rad(angle):
    """``angle/180.0*3.1415926`` in double, stored to float."""
    return f32(float(angle) / 180.0 * 3.1415926)


class Maze(NamedTuple):
    disable: bool
    steps: int
    start: tuple
    heading: float
    goal: tuple
    poi: tuple
    walls: np.ndarray             # float32 [n, 4]: ax, ay, bx, by


def load_maze(path=FIXTURE) -> Maze:
    tok = open(path).read().split()
    disable, steps, n = int(tok[0]), int(tok[1]), int(tok[2])
    v = [float(t) for t in tok[3:]]
    walls = np.array(v[7:7 + 4 * n], dtype=np.float32).reshape(n, 4)
    assert walls.shape == (n, 4)
    return Maze(bool(disable), steps, (f32(v[0]), f32(v[1])), v[2], (f32(v[3]), f32(v[4])), (f32(v[5]), f32(v[6])), walls)


class State(NamedTuple):
    x: np.float32
    y: np.float32
    heading: np.float32
    speed: np.float32
    ang_vel: np.float32
    collide: bool
    t: int


def reset_state(maze: Maze) -> State:
    """``Character::reset``: the start location, heading / speed / angular velocity 0."""
    return State(maze.start[0], maze.start[1], f32(0), f32(0), f32(0), False, 0)


def _distance(ax, ay, bx, by):
    """``Point(a).distance(b)``."""
    dx = bx - ax
    dy = by - ay
    return sqrtf(dx * dx + dy * dy)


def _rotate(px, py, angle, cx, cy):
    """``Point::rotate(angle, c)``."""
    rad = deg2rad(angle)
    ox, oy = px - cx, py - cy
    return cosf(rad) * ox - sinf(rad) * oy + cx, sinf(rad) * ox + cosf(rad) * oy + cy


def intersect(wall, cx, cy, dx_, dy_):
    """``Line::intersection`` of the wall (A, B) with the segment C -> D: (found, r, s, px, py)."""
    ax, ay, bx, by = (f32(v) for v in wall)
    rtop = (ay - cy) * (dx_ - cx) - (ax - cx) * (dy_ - cy)
    rbot = (bx - ax) * (dy_ - cy) - (by - ay) * (dx_ - cx)
    stop = (ay - cy) * (bx - ax) - (ax - cx) * (by - ay)
    sbot = (bx - ax) * (dy_ - cy) - (by - ay) * (dx_ - cx)
    if rbot == 0 or sbot == 0:
        return False, None, None, None, None
    r = rtop / rbot
    s = stop / sbot
    if r > 0 and r < 1 and s > 0 and s < 1:
        return True, r, s, ax + r * (bx - ax), ay + r * (by - ay)
    return False, r, s, None, None


def line_distance(wall, nx, ny):
    """``Line::distance(n)``."""
    ax, ay, bx, by = (f32(v) for v in wall)
    utop = (nx - ax) * (bx - ax) + (ny - ay) * (by - ay)
    ubot = _distance(ax, ay, bx, by)
    ubot = ubot * ubot
    if ubot == 0.0:
        return f32(0.0)
    u = utop / ubot
    if u < 0 or u > 1:
        d1 = _distance(ax, ay, nx, ny)
        d2 = _distance(bx, by, nx, ny)
        return d1 if d1 < d2 else d2
    return _distance(ax + u * (bx - ax), ay + u * (by - ay), nx, ny)


def rangefinders(maze: Maze, x, y, heading, detail=None):
    """The 6 ranges (``update_rangefinders``).  ``detail``: a list that receives, per sensor, the (r, s) of every wall
    whose rbot is nonzero, for the discrete-event margins of tests/test_gpu_maze.py."""
    out = []
    for ang in RANGEFINDER_ANGLES:
        rad = deg2rad(ang)
        px, py = _rotate(x + cosf(rad) * RANGE, y + sinf(rad) * RANGE, heading, x, y)
        rng = RANGE
        rs_ = []
        for w in maze.walls:
            found, r, s, ix, iy = intersect(w, x, y, px, py)
            if r is not None:
                rs_.append((r, s))
            if found:
                d = _distance(ix, iy, x, y)
                if d < rng:
                    rng = d
        out.append(rng)
        if detail is not None:
            detail.append(rs_)
    return out


def radar_angle(maze: Maze, x, y, heading):
    """``update_radar_gen``'s angle of the goal in the navigator's frame (``Point::angle``), float32 degrees."""
    tx, ty = _rotate(maze.goal[0], maze.goal[1], -heading, x, y)
    tx, ty = tx - x, ty - y
    if tx == 0.0:
        return f32(90.0) if ty > 0.0 else f32(270.0)
    ang = f32(float(atanf(ty / tx)) / 3.1415926 * 180.0)
    return ang if tx > 0.0 else f32(float(ang) + 180.0)


def radar(angle):
    out = []
    for a1, a2 in RADAR:
        hit = (angle >= a1 and angle < a2) or (float(angle) + 360.0 >= a1 and float(angle) + 360.0 < a2)
        out.append(f32(1.0) if hit else f32(0.0))
    return out


def observation(maze: Maze, x, y, heading, detail=None):
    """``generate_neural_inputs``: float32 [11] = bias 1, the 6 ranges / 100, the 4 goal-radar sectors."""
    with np.errstate(all="ignore"):
        rng = rangefinders(maze, f32(x), f32(y), f32(heading), detail)
        return np.array([1.0] + [v / RANGE for v in rng] + radar(radar_angle(maze, f32(x), f32(y), f32(heading))),
                        dtype=np.float32)


def collides(maze: Maze, x, y):
    """``collide_lines(loc, radius)``."""
    return any(line_distance(w, x, y) < RADIUS for w in maze.walls)


def distance_to_target(maze: Maze, x, y):
    d = _distance(x, y, maze.goal[0], maze.goal[1])
    return f32(500.0) if math.isnan(d) else d


def step(maze: Maze, s: State, a0, a1):
    """One ``MazeEnvironment::step``: (next State, float32 reward)."""
    with np.errstate(all="ignore"):
        o1, o2 = f32(float(f32(a0)) + 0.5), f32(0.5 + float(f32(a1)))
        o1 = f32(1.0) if o1 > 1.0 else o1
        o1 = f32(0.0) if o1 < 0.0 else o1
        o2 = f32(1.0) if o2 > 1.0 else o2
        o2 = f32(0.0) if o2 < 0.0 else o2
        d_ang = f32((float(o1) - 0.5) * 6.0) - s.ang_vel
        d_speed = f32((float(o2) - 0.5) * 6.0) - s.speed
        d_ang = f32(0.2) if float(d_ang) >= 0.2 else d_ang              # float vs double 0.2: compared in double
        d_ang = f32(-0.2) if float(d_ang) <= -0.2 else d_ang
        d_speed = f32(0.2) if float(d_speed) >= 0.2 else d_speed
        d_speed = f32(-0.2) if float(d_speed) <= -0.2 else d_speed
        ang_vel, speed = s.ang_vel + d_ang, s.speed + d_speed
        speed = f32(3.0) if speed > 3.0 else speed
        speed = f32(-3.0) if speed < -3.0 else speed
        ang_vel = f32(3.0) if ang_vel > 3.0 else ang_vel
        ang_vel = f32(-3.0) if ang_vel < -3.0 else ang_vel
        # Update(): the velocity from the heading before the turn, in double
        h = float(s.heading) / 180.0 * 3.1415926
        vx, vy = f32(_m.cos(h) * float(speed)), f32(_m.sin(h) * float(speed))
        heading = s.heading + ang_vel
        heading = heading - f32(360) if heading > 360 else heading
        heading = heading + f32(360) if heading < 0 else heading
        nx, ny = vx + s.x, vy + s.y
        x, y, collide = s.x, s.y, s.collide
        if not collide and not collides(maze, nx, ny):
            x, y = nx, ny
        elif maze.disable:
            collide = True
        t = s.t + 1
        reward = -distance_to_target(maze, x, y) if t >= MAZE_STEPS else f32(0.0)
        return State(x, y, heading, speed, ang_vel, collide, t), f32(reward)


def episode(maze: Maze, actions, s: State = None):
    """Open loop from ``s`` (default the reset state): per step (State, reward, observation after the step)."""
    s = reset_state(maze) if s is None else s
    out = []
    for a0, a1 in actions:
        s, r = step(maze, s, a0, a1)
        out.append((s, r, observation(maze, s.x, s.y, s.heading)))
    return out
