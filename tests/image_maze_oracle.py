"""Referee of the image hard maze (DESIGN.md 3.10): the rendering rule of csrc/image_maze_kernels.cu as numpy float32
operations in the kernel's order (vectorised over the pixels: every element still sees the same IEEE single-precision
operations, each rounded, no fused multiply-add), and the step through tests/maze_oracle.py.

Frames are uint8 [84, 84] (row = y); a stack is uint8 [84, 84, 4] with the newest frame last."""
import numpy as np

import maze_oracle as M

f32 = np.float32
RES = 84
DEFAULT_ACTIONS = np.array([(t, s) for t in (-0.5, 0.0, 0.5) for s in (-0.5, 0.0, 0.5)], dtype=np.float32)
# heading_dir's constants, parsed from the kernel's literals
DEG = f32("0.0174532925")
S3, S5, S7 = f32("-0.166666667"), f32("0.00833333333"), f32("-0.000198412698")
C2, C4, C6 = f32("-0.5"), f32("0.0416666667"), f32("-0.00138888889")


def geometry(walls):
    """(x0, y0, upp, half): the walls' lower bounds, maze units per pixel, half a pixel."""
    w = np.asarray(walls, dtype=np.float32)
    xs, ys = w[:, [0, 2]], w[:, [1, 3]]
    x0, x1, y0, y1 = f32(xs.min()), f32(xs.max()), f32(ys.min()), f32(ys.max())
    ex, ey = f32(x1 - x0), f32(y1 - y0)
    ext = ex if ex > ey else ey
    upp = f32(ext / f32(RES))
    return x0, y0, upp, f32(upp * f32(0.5))


def centres(geom):
    """float32 [84, 84] x and y of every pixel centre."""
    x0, y0, upp, _ = geom
    k = np.arange(RES, dtype=np.float32) + f32(0.5)
    cx, cy = x0 + k * upp, y0 + k * upp                       # each a rounded product, then a rounded sum
    return np.broadcast_to(cx[None, :], (RES, RES)), np.broadcast_to(cy[:, None], (RES, RES))


def line_distance(wall, nx, ny):
    """maze_oracle.line_distance (Line::distance) over arrays of points, branch by branch."""
    ax, ay, bx, by = (f32(v) for v in wall)
    with np.errstate(all="ignore"):
        bax, bay = f32(bx - ax), f32(by - ay)
        utop = (nx - ax) * bax + (ny - ay) * bay
        ubot = M._distance(ax, ay, bx, by)
        ubot = f32(ubot * ubot)
        if ubot == 0.0:
            return np.zeros_like(nx)
        u = utop / ubot
        d1 = np.sqrt((nx - ax) * (nx - ax) + (ny - ay) * (ny - ay))
        d2 = np.sqrt((nx - bx) * (nx - bx) + (ny - by) * (ny - by))
        px, py = ax + u * bax, ay + u * bay
        d3 = np.sqrt((nx - px) * (nx - px) + (ny - py) * (ny - py))
        return np.where((u < 0) | (u > 1), np.where(d1 < d2, d1, d2), d3).astype(np.float32)


def background(maze):
    """uint8 [84, 84]: 255 where a wall is within half a pixel of the centre."""
    geom = geometry(maze.walls)
    cx, cy = centres(geom)
    wall = np.zeros((RES, RES), dtype=bool)
    for w in maze.walls:
        wall |= line_distance(w, cx, cy) <= geom[3]
    return np.where(wall, 255, 0).astype(np.uint8)


def heading_dir(h):
    """(hx, hy): the kernel's quadrant reduction and polynomials."""
    h = f32(h)
    with np.errstate(all="ignore"):
        q = f32(np.floor(h / f32(90.0)))
        f = f32(h - f32(f32(90.0) * q))
        x = f32(f * DEG)
        x2 = f32(x * x)
        s = x * (f32(1.0) + x2 * (S3 + x2 * (S5 + x2 * S7)))          # float32 scalars throughout
        c = f32(1.0) + x2 * (C2 + x2 * (C4 + x2 * C6))
    k = int(q) & 3 if (q == q and abs(q) < 1e6) else 0
    return [(c, s), (-s, c), (-c, -s), (s, -c)][k]


def frame(maze, bg, x, y, heading, geom=None):
    """uint8 [84, 84]: the background with the navigator drawn at (x, y, heading)."""
    geom = geometry(maze.walls) if geom is None else geom
    cx, cy = centres(geom)
    dx, dy = cx - f32(x), cy - f32(y)
    hx, hy = heading_dir(heading)
    with np.errstate(all="ignore"):
        inside = (dx * dx + dy * dy) <= f32(64.0)
        front = (dx * hx + dy * hy) > f32(0.0)
    out = bg.copy()
    out[inside & front] = 64
    out[inside & ~front] = 128
    return out


def push(stack, fr):
    """The frame stack after a step: planes 1..3 move to 0..2, the new frame is plane 3."""
    return np.concatenate([stack[:, :, 1:], fr[:, :, None]], axis=2)


def fill(fr):
    """The frame stack after a reset: four copies of the first frame."""
    return np.repeat(fr[:, :, None], 4, axis=2)


def step(maze, s, action, table=DEFAULT_ACTIONS):
    """One step of discrete action `action`: (next maze_oracle.State, float32 reward, done)."""
    a0, a1 = table[int(action)]
    n, r = M.step(maze, s, a0, a1)
    return n, r, n.t >= M.MAZE_STEPS
