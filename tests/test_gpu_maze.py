"""GPU tests of the hard maze on the continuous episode kernel (dne_maze_episodes), its runner and the drivers on it.

Referees:
* the kernel itself: one launch of 400 steps equals 400 chained one-step launches bit for bit;
* every transition of those chained launches against tests/maze_oracle.py (the reference's float32 C++ restated, glibc's
  transcendentals; pinned bit for bit to the reference's own code by tests/test_maze_host.py) under the same action.
  The actions are exact: a zero-weight linear net outputs its bias, and the action noise carries the action sequence.
  The kernel and the referee run the same IEEE float32 / double operations, so heading, speed, angular velocity, the
  step count and the collision flag must agree exactly.  They differ only through the transcendentals, by CUDA's
  documented maximum errors (cosf, sinf, atanf: 2 ulp; double cos / sin: 2 ulp) against glibc's (below 1 ulp):
  - x, y: vx = fl32(cos(h) * speed) is computed in double; CUDA's and glibc's cos differ by at most 3 double ulps, so the
    float32 vx differs by at most one float32 ulp of |vx| <= 3 (2^-22), and the position by that plus one ulp of itself;
  - the rangefinders: cosf / sinf of the heading differ by at most 3 float32 ulps (3 * 2^-24 on values below 1), which
    turns a ray projected 100 units out by at most delta = 100 * 2 * 3 * 2^-24 = 3.6e-5 units, an angle of 3.6e-7 rad;
    the range moves by at most 2 * range * angle / sin(incidence), plus the roundings of the intersection, 16 float32
    ulps of the range / sin(incidence);
  - the goal radar: the sector is decided on an angle whose error is below 1e-4 degrees;
  - the reward: -|goal - position|, within the position's bound times sqrt(2) plus 2 ulps.
  A transition is excluded only where a discrete event lies within that error: a wall distance within 1e-3 of the
  radius, a ray whose intersection parameters r or s lie within 1e-3 of 0 or 1 or which meets a wall at sin(incidence) <
  1e-2, or a radar angle within 1e-3 degrees of a sector edge.  The clamps, the rate limits and the heading wrap are
  decided on exactly computed values and are never excluded.
* the head: a one-step launch from rest at heading 0 (whose observation the kernel computes exactly: cosf(0) = 1,
  sinf(0) = 0, the rays' directions come from the host C library) reveals the head's output through the new angular
  velocity and speed; it is checked against the float64 forward referee of tests/test_gpu_dense_paths.py.
"""
import ctypes as C
import json
import math
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from oracle import oracle as O                     # noqa: E402
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import maze_oracle as M                            # noqa: E402
from test_gpu_dense_paths import U, member, normalise, referee   # noqa: E402  (the float64 forward referee)
from dne import _ffi as F                          # noqa: E402
from dne import nets                               # noqa: E402
from dne.engine import make_context                # noqa: E402
from dne.envs import MazeEnv, make_env             # noqa: E402
from dne.noise import SharedNoiseTable             # noqa: E402
from dne.rollout import EpisodeKernelRunner, Unit, make_runner   # noqa: E402

NOISE_COUNT = 2_000_000
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations")
f32 = np.float32
MAZE = M.load_maze()
# generations within which hardmaze_nses.json (seed 0) must play a noiseless episode ending within 10 of the goal
LEARN_MAX_GENERATIONS = 280          # reached after 140 on an H100 (twice that)
LEARN_RADIUS = 10.0


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def noise(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device="cuda:0")


@pytest.fixture(scope="module")
def ctx(noise):
    return make_context(0, noise)


def _net(hidden=(64, 64), act=F.ACT_TANH, n_out=2, ob_dim=11):
    dims = [ob_dim] + list(hidden)
    layers = [nets._dense(dims[i], dims[i + 1], act=act) for i in range(len(hidden))]
    layers.append(nets._dense(dims[-1], n_out, act=F.ACT_NONE))
    return nets._finish(nets.NetSpec("maze", layers, F.OB_VECTOR, ob_dim))


def _cuda(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(DEV)


def _launch(ctx, net, theta, idx, scale, rows, init, T, ob_mean=None, ob_std=None, ac_noise=None, stats=True,
            desc=None):
    """dne_maze_episodes on numpy inputs -> dict of numpy outputs (and 'rc')."""
    n = len(idx)
    k = max(n, 1)
    d = dict(ret=torch.full((k,), -1.0, dtype=torch.float32, device=DEV),
             sret=torch.full((k,), -1.0, dtype=torch.float32, device=DEV),
             len=torch.full((k,), -1, dtype=torch.int32, device=DEV),
             fin=torch.full((k, 7), -7.0, dtype=torch.float64, device=DEV))
    if stats:
        d["s"] = torch.full((k, 11), -7.0, dtype=torch.float64, device=DEV)
        d["q"] = torch.full((k, 11), -7.0, dtype=torch.float64, device=DEV)
    args = [_cuda(theta, np.float32), _cuda(idx, np.int64), _cuda(scale, np.float32),
            None if rows is None else _cuda(rows, np.int32), _cuda(init, np.float64),
            None if ob_mean is None else _cuda(ob_mean, np.float32), None if ob_std is None else _cuda(ob_std, np.float32),
            None if ac_noise is None else _cuda(ac_noise, np.float32)]
    rc = F.lib().dne_maze_episodes(
        ctx.handle, C.byref(desc if desc is not None else MazeEnv(1).desc), C.byref(net.desc), F.ptr(args[0]),
        F.ptr(args[1]), F.ptr(args[2]), F.ptr(args[3]), n, F.ptr(args[4]), int(T), F.ptr(args[5]), F.ptr(args[6]),
        F.ptr(args[7]), F.ptr(d["ret"]), F.ptr(d["sret"]), F.ptr(d["len"]), F.ptr(d["fin"]), F.ptr(d.get("s")),
        F.ptr(d.get("q")), F.stream_ptr())
    torch.cuda.synchronize()
    out = {key: v.cpu().numpy()[:n] for key, v in d.items()}
    out["rc"] = rc
    return out


def _mixed(rs, P, n=512, n_rows=4):
    """± pairs on row 0, unpaired scales, GA members on rows of a [n_rows, P] matrix, noiseless (scale 0) members."""
    n_pair, n_un, n_zero = n // 4, n // 8, n // 8
    n_ga = n - 2 * n_pair - n_un - n_zero
    hi = NOISE_COUNT - P + 1
    idx = np.concatenate([np.repeat(rs.randint(0, hi, n_pair), 2), rs.randint(0, hi, n_un), rs.randint(0, hi, n_zero),
                          rs.randint(0, hi, n_ga)]).astype(np.int64)
    scale = np.concatenate([np.tile([0.1, -0.1], n_pair), rs.choice([0.05, 0.3, -0.5], n_un), np.zeros(n_zero),
                            rs.choice([0.05, -0.1], n_ga)]).astype(np.float32)
    rows = np.concatenate([np.zeros(2 * n_pair + n_un + n_zero), rs.randint(0, n_rows, n_ga)]).astype(np.int32)
    return idx, scale, rows


def _inits(rs, n):
    """The reset state for half the members, random open positions (t = 0) for the rest."""
    s = MazeEnv(1).initial_states(n)
    k = n // 2
    pos = []
    while len(pos) < k:
        x, y = rs.uniform(10, 190), rs.uniform(10, 195)
        if not M.collides(MAZE, f32(x), f32(y)):
            pos.append((f32(x), f32(y)))
    s[k:, 0:2] = np.array(pos, dtype=np.float64)
    s[k:, 2] = rs.uniform(0, 360, n - k).astype(f32)
    return s


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stats,noisy", [(True, True), (False, False), (True, False), (False, True)])
def test_one_launch_equals_chained_one_step_launches(ctx, stats, noisy):
    net = _net()
    P, T = net.num_params, 400
    rs = np.random.RandomState(1 + 2 * stats + noisy)
    theta = (rs.randn(4, P) * 0.3).astype(np.float32)
    idx, scale, rows = _mixed(rs, P)
    n = len(idx)
    init = _inits(rs, n)
    mean, std = ((rs.randn(11) * 0.1).astype(np.float32), rs.uniform(0.3, 1.0, 11).astype(np.float32)) if stats else \
        (None, None)
    acn = (rs.randn(n, T, 2) * 0.2).astype(np.float32) if noisy else None
    if noisy:
        acn[scale == 0] = 0.0
    full = _launch(ctx, net, theta, idx, scale, rows, init, T, mean, std, acn, stats=stats)
    assert full["rc"] == 0 and (full["len"] == T).all()
    st = init.copy()
    ret, sret = np.zeros(n), np.zeros(n)
    s, q = np.zeros((n, 11)), np.zeros((n, 11))
    for t in range(T):
        one = _launch(ctx, net, theta, idx, scale, rows, st, 1, mean, std, None if acn is None else acn[:, t:t + 1],
                      stats=stats)
        assert one["rc"] == 0
        st = one["fin"]
        ret += one["ret"].astype(np.float64)
        sret += one["sret"].astype(np.float64)
        if stats:
            s += one["s"]
            q += one["q"]
    assert full["fin"].tobytes() == st.tobytes()
    assert full["ret"].tobytes() == ret.astype(np.float32).tobytes()
    assert full["sret"].tobytes() == sret.astype(np.float32).tobytes()
    if stats:
        assert full["s"].tobytes() == s.tobytes() and full["q"].tobytes() == q.tobytes()
    assert (full["fin"][:, 5] == 400).all() and (full["ret"] < 0).all()
    moved = np.hypot(full["fin"][:, 0] - init[:, 0], full["fin"][:, 1] - init[:, 1])
    print(f"members that moved more than 20 units: {(moved > 20).sum()} of {n}")
    assert (moved > 20).sum() > n // 4
    again = _launch(ctx, net, theta, idx, scale, rows, init, T, mean, std, acn, stats=stats)
    for key in ("ret", "sret", "fin") + (("s", "q") if stats else ()):
        assert again[key].tobytes() == full[key].tobytes()      # bit-identical reruns


# ---- transitions against the referee ----------------------------------------------------------------------------------
ULP = lambda v: float(np.spacing(f32(abs(v))))             # noqa: E731
DELTA_RAY = 100 * 2 * 3 * 2.0 ** -24                       # projected-point error of a rangefinder (units)
EDGES = (45.0, 135.0, 225.0, 315.0, 360.0, 405.0, 0.0)


def _sin_incidence(heading, sensor, wall):
    rad = math.radians(float(heading) + sensor)
    dx, dy = math.cos(rad), math.sin(rad)
    wx, wy = float(wall[2] - wall[0]), float(wall[3] - wall[1])
    return abs(dx * wy - dy * wx) / math.hypot(wx, wy)


def _ob_bounds(s):
    """(observation bound [11], excluded?) at state s (x, y, heading)."""
    detail = []
    M.rangefinders(MAZE, f32(s[0]), f32(s[1]), f32(s[2]), detail)
    rng = M.rangefinders(MAZE, f32(s[0]), f32(s[1]), f32(s[2]))
    bnd = np.zeros(11)
    for i, sensor in enumerate(M.RANGEFINDER_ANGLES):
        for r, s_ in detail[i]:
            if min(abs(r), abs(r - 1), abs(s_), abs(s_ - 1)) < 1e-3:
                return bnd, True
        sin_min = 1.0
        for w in MAZE.walls:
            found, r, s_, _, _ = M.intersect(w, f32(s[0]), f32(s[1]), *_ray_end(s, sensor))
            if found:
                sin_min = min(sin_min, _sin_incidence(s[2], sensor, w))
        if sin_min < 1e-2:
            return bnd, True
        R = float(rng[i])
        bnd[1 + i] = (2 * R * DELTA_RAY / 100 + 16 * ULP(R)) / sin_min / 100 + 2 * ULP(R / 100)
    ang = float(M.radar_angle(MAZE, f32(s[0]), f32(s[1]), f32(s[2])))
    if not math.isnan(ang) and min(abs(ang - e) for e in EDGES + tuple(e - 360 for e in EDGES)) < 1e-3:
        return bnd, True
    return bnd, False


def _ray_end(s, sensor):
    rad = M.deg2rad(sensor)
    return M._rotate(f32(s[0]) + M.cosf(rad) * M.RANGE, f32(s[1]) + M.sinf(rad) * M.RANGE, f32(s[2]), f32(s[0]),
                     f32(s[1]))


def _referee_step(s, a, mutate=None):
    st = M.State(f32(s[0]), f32(s[1]), f32(s[2]), f32(s[3]), f32(s[4]), bool(s[6] != 0), int(s[5]))
    n, r = M.step(MAZE, st, a[0], a[1])
    if mutate == "heading_first":          # vx / vy formed from the heading after the turn
        h = float(n.heading) / 180.0 * 3.1415926
        n = n._replace(x=f32(M._m.cos(h) * float(n.speed)) + st.x, y=f32(M._m.sin(h) * float(n.speed)) + st.y)
    elif mutate == "no_rate_limit":        # interpret_outputs without the +-0.2 rate limits
        o = [min(max(float(f32(float(f32(v)) + 0.5)), 0.0), 1.0) for v in a]
        n = n._replace(ang_vel=f32(min(max(float(f32((o[0] - 0.5) * 6.0)), -3.0), 3.0)),
                       speed=f32(min(max(float(f32((o[1] - 0.5) * 6.0)), -3.0), 3.0)))
    return n, r


def _zero_net_theta(net):
    return np.zeros((1, net.num_params), np.float32)


def test_transitions_against_referee(ctx):
    """Chained one-step launches of exact open-loop actions; every transition against the referee's step."""
    net = _net(hidden=())                          # linear head, zero weights and bias: the action is the noise slice
    rs = np.random.RandomState(7)
    n, T = 96, 120
    init = _inits(rs, n)
    acts = np.zeros((n, T, 2), np.float32)
    for m in range(n):
        kind = m % 6
        if kind == 0:
            acts[m] = rs.normal(0, 0.3, (T, 2))
        elif kind == 1:
            acts[m] = np.tile([rs.uniform(-0.1, 0.1), 0.5], (T, 1))          # full speed into the walls
        elif kind == 2:
            acts[m] = rs.choice([-2.0, -0.5, 0.5, 2.0], (T, 2))              # saturated, out of range
        elif kind == 3:
            acts[m] = np.tile([0.5, rs.uniform(-0.1, 0.1)], (T, 1))          # spinning across the heading wrap
        elif kind == 4:
            acts[m] = np.cumsum(rs.normal(0, 0.05, (T, 2)), axis=0).clip(-0.6, 0.6)
        else:
            acts[m] = np.tile([rs.normal(0, 0.05), -0.5], (T, 1))            # reverse into the walls
    init[::8, 5] = 400 - T // 2                                               # the reward step falls inside the window
    theta = _zero_net_theta(net)
    idx, scale = np.zeros(n, np.int64), np.zeros(n, np.float32)
    st, states, rewards, obs_sums = init.copy(), [init.copy()], [], []
    for t in range(T):
        one = _launch(ctx, net, theta, idx, scale, None, st, 1, None, None, acts[:, t:t + 1])
        assert one["rc"] == 0
        st = one["fin"]
        states.append(st.copy())
        rewards.append(one["ret"].copy())
        obs_sums.append(one["s"].copy())          # the observation the step's forward saw: the state before the step
    checked = excluded = 0
    worst = 0.0
    mut = {"heading_first": 0, "no_rate_limit": 0}
    for t in range(T):
        for m in range(0, n, 2 if t % 2 else 1):
            s0, s1 = states[t][m], states[t + 1][m]
            a = acts[m, t]
            obnd, ex = _ob_bounds(s0)
            ref_ob = M.observation(MAZE, s0[0], s0[1], s0[2])
            ref, r = _referee_step(s0, a)
            near_wall = any(abs(float(M.line_distance(w, *_next_pos(s0, ref))) - 8.0) < 1e-3 for w in MAZE.walls)
            if ex or near_wall:
                excluded += 1
                continue
            checked += 1
            got_ob = obs_sums[t][m].astype(np.float32)
            assert np.all(np.abs(got_ob.astype(np.float64) - ref_ob) <= obnd), (t, m, got_ob, ref_ob, obnd)
            assert s1[2] == ref.heading and s1[3] == ref.speed and s1[4] == ref.ang_vel, (t, m, s1, ref)
            assert s1[5] == ref.t and bool(s1[6]) == ref.collide
            px = ULP(3.0) + ULP(max(abs(s1[0]), abs(float(ref.x))))
            py = ULP(3.0) + ULP(max(abs(s1[1]), abs(float(ref.y))))
            ex_, ey_ = abs(s1[0] - float(ref.x)), abs(s1[1] - float(ref.y))
            assert ex_ <= px and ey_ <= py, (t, m, s1, ref)
            rb = math.sqrt(2) * max(px, py) + 2 * ULP(r)
            assert abs(float(rewards[t][m]) - float(r)) <= rb, (t, m, rewards[t][m], r)
            worst = max(worst, ex_ / px, ey_ / py)
            for name in mut:
                mref, _ = _referee_step(s0, a, name)
                mut[name] += int(abs(s1[0] - float(mref.x)) > px or abs(s1[1] - float(mref.y)) > py or
                                 s1[3] != mref.speed or s1[4] != mref.ang_vel)
    print(f"transitions: {checked} checked, {excluded} excluded; worst position error / bound {worst:.3g}; "
          f"mutants rejected {mut}")
    assert checked > 0.8 * (checked + excluded)
    for name, k in mut.items():
        assert k > checked // 2, f"the bound does not reject the '{name}' mutant on most transitions ({k} of {checked})"


def _next_pos(s0, ref):
    """The position the step tried (the referee's unmoved state keeps s0's)."""
    st = M.State(f32(s0[0]), f32(s0[1]), f32(s0[2]), f32(s0[3]), f32(s0[4]), False, int(s0[5]))
    h = float(st.heading) / 180.0 * 3.1415926
    return (f32(M._m.cos(h) * float(ref.speed)) + st.x, f32(M._m.sin(h) * float(ref.speed)) + st.y)


@pytest.mark.parametrize("hidden,act", [((64, 64), F.ACT_TANH), ((32,), F.ACT_RELU), ((200, 100), F.ACT_TANH)])
def test_head_against_float64_referee(ctx, host_noise, hidden, act):
    net = _net(hidden, act)
    P = net.num_params
    rs = np.random.RandomState(23)
    theta = (rs.randn(2, P) * 0.02).astype(np.float32)
    idx, scale, rows = _mixed(rs, P, n=128, n_rows=2)
    scale *= np.float32(0.1)
    n = len(idx)
    init = _inits(rs, n)
    init[:, 2:5] = 0.0                                             # heading 0, at rest
    mean, std = (rs.randn(11) * 0.1).astype(np.float32), rs.uniform(0.3, 1.0, 11).astype(np.float32)
    got = _launch(ctx, net, theta, idx, scale, rows, init, 1, mean, std)
    assert got["rc"] == 0
    bad = 0
    for m in range(n):
        o = M.observation(MAZE, init[m, 0], init[m, 1], 0.0)
        np.testing.assert_array_equal(got["s"][m], o.astype(np.float64))       # the exact observation at heading 0
        w, wm = member(theta, int(rows[m]), host_noise, int(idx[m]), scale[m], P)
        y, e = referee(net, w, wm, normalise(o[None, :], mean, std)[0])
        # new ang_vel = fl(fl(fl(a + 0.5) - 0.5) * 6) while |6a| < 0.2: a is recovered within 2^-25 + 6 ulps of the result
        for j, col in ((0, 4), (1, 3)):
            v = float(got["fin"][m, col])
            if abs(v) >= 0.2:
                continue
            bnd = e[j] + 2.0 ** -25 + 6 * ULP(v) / 6 + 2 * U * abs(y[j])
            bad += int(abs(v / 6.0 - y[j]) > bnd)
    assert bad == 0


# ---- contract, runner, drivers ----------------------------------------------------------------------------------------
def test_contract(ctx):
    net = _net()
    L = F.lib()
    assert L.dne_maze_net_supported(C.byref(net.desc)) == 0
    assert L.dne_maze_net_supported(C.byref(_net((1024,)).desc)) == 0
    unsup = {"ob_dim": _net(ob_dim=3), "n_out": _net(n_out=1), "conv": nets.make_net("Model", num_actions=2),
             "hidden act": _net(act=F.ACT_NONE), "wide": _net((256, 256))}
    th = torch.zeros(net.num_params, device=DEV)
    d_idx = torch.zeros(4, dtype=torch.int64, device=DEV)
    d_sc = torch.zeros(4, device=DEV)
    d_init = torch.zeros(4, 7, dtype=torch.float64, device=DEV)
    d_ret, d_sret = torch.full((4,), -1.0, device=DEV), torch.full((4,), -1.0, device=DEV)
    d_len = torch.full((4,), -1, dtype=torch.int32, device=DEV)

    def call(n_, T, net_=net, desc=None):
        return L.dne_maze_episodes(ctx.handle, C.byref(desc if desc is not None else MazeEnv(1).desc),
                                   C.byref(net_.desc), F.ptr(th), F.ptr(d_idx), F.ptr(d_sc), None, n_, F.ptr(d_init), T,
                                   None, None, None, F.ptr(d_ret), F.ptr(d_sret), F.ptr(d_len), None, None, None,
                                   F.stream_ptr())
    for what, bad in unsup.items():
        assert call(4, 10, bad) == -4, what
        assert L.dne_last_error().decode().startswith("dne_maze_episodes"), what
        assert L.dne_maze_net_supported(C.byref(bad.desc)) == -4, what
    for T in (0, 401, -1):
        assert call(4, T) == -1, T
    big = F.MazeDesc(n_walls=65)
    assert call(4, 10, desc=big) == -1 and "n_walls" in L.dne_last_error().decode()
    assert call(4, 10, desc=F.MazeDesc(n_walls=-1)) == -1
    assert call(4, 400) == 0
    torch.cuda.synchronize()
    assert (d_len == 400).all()


def test_runner_matches_direct_launch_and_make_runner(ctx):
    net = _net()
    P = net.num_params
    rs = np.random.RandomState(12)
    theta = torch.from_numpy((rs.randn(3, P) * 0.3).astype(np.float32)).to(DEV)
    units = [Unit(int(rs.randint(0, NOISE_COUNT - P)), (0.05, -0.05), theta_idx=i % 3) for i in range(40)] + \
            [Unit(0, (0.0, 0.0), theta_idx=1, noiseless=True) for _ in range(3)]
    mean, std = torch.from_numpy(rs.randn(11).astype(np.float32) * 0.1), torch.from_numpy(rs.uniform(0.5, 1, 11)
                                                                                            .astype(np.float32))
    env = make_env("maze", 4)
    r = make_runner(ctx, net, env, n_slots=4, group=2)
    assert isinstance(r, EpisodeKernelRunner)
    with pytest.raises(NotImplementedError, match="continuous"):
        make_runner(ctx, net, env, n_slots=4, group=2, action_fn=lambda a: a)
    res = r.run(theta, units, None, ob_mean=mean, ob_std=std, collect_bc="final", ac_noise_std=0.01,
                random_stream=np.random.RandomState(77), save_obs_prob=0.3)
    n = 2 * len(units)
    init = env.initial_states(n)
    idx = np.repeat([u.noise_idx for u in units], 2)
    scale = np.array([s for u in units for s in u.scales], np.float32)
    rows = np.repeat([u.theta_idx for u in units], 2)
    noisy = scale != 0
    stream = np.random.RandomState(77)
    save = np.zeros(n, bool)
    for m in np.nonzero(noisy)[0]:
        save[m] = stream.rand() < 0.3
    acn = np.zeros((n, 400, 2), np.float32)
    acn[noisy] = stream.randn(int(noisy.sum()), 400, 2).astype(np.float32) * np.float32(0.01)
    d = _launch(ctx, net, theta.cpu().numpy(), idx, scale, rows, init, 400, mean.numpy(), std.numpy(), acn)
    np.testing.assert_array_equal(res.returns.ravel(), d["ret"])
    np.testing.assert_array_equal(res.signreturns.ravel(), d["sret"])
    np.testing.assert_array_equal(res.lengths.ravel(), d["len"])
    bcs = np.stack([b for u in res.bcs for b in u])
    assert bcs.shape == (n, 2) and bcs.dtype == np.float64
    np.testing.assert_array_equal(bcs, d["fin"][:, :2])
    assert res.ob_count == 400 * int(save.sum())
    short = r.run(theta, units[:4], 100)                          # a truncated episode pays 0
    assert (short.returns == 0).all() and (short.lengths == 100).all()


def _exp(name, **over):
    with open(os.path.join(CONFIGS, name)) as f:
        exp = json.load(f)
    exp["config"].update(snapshot_freq=0, **over)
    return exp


def test_drivers_complete_on_maze(noise, tmp_path):
    from es_distributed import es as ES
    from es_distributed import ga as GA
    from es_distributed import nses as NS
    from es_distributed import policies
    from es_distributed import rs as RS
    ES.set_default_noise(noise)
    log = []
    exp = _exp("hardmaze_es.json", episodes_per_batch=16)
    exp["maze_file"] = M.FIXTURE
    ES.run_master(None, None, exp, max_iterations=1, n_slots=8, noise=noise, seed=3,
                  on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 1 and log[0]["returns_n2"].shape == (8, 2) and (log[0]["lengths_n2"] == 400).all()
    assert (log[0]["returns_n2"] < 0).all()
    for algo in ("ns", "nsr"):
        nlog = []
        exp = _exp("hardmaze_nses.json", episodes_per_batch=16)
        exp.update(algo_type=algo)
        exp["novelty_search"].update(population_size=2)
        NS.set_default_noise(noise)
        _, archive = NS.run_master(None, str(tmp_path / algo), exp, max_iterations=2, n_slots=8, noise=noise, seed=2,
                                   on_iteration=lambda it, st, ex: nlog.append(ex))
        assert len(nlog) == 2 and all(np.asarray(b).shape == (2,) for b in nlog[0]["bcs"])
        assert np.isfinite(nlog[-1]["novelty_n2"]).all() and len(archive) == 4
    glog = []
    exp = _exp("hardmaze_es.json", episodes_per_batch=12)
    exp.update(population_size=4, num_elites=1)
    GA.set_default_noise(noise)
    GA.run_master(None, str(tmp_path / "ga"), exp, max_iterations=2, n_slots=8, noise=noise, seed=5,
                  on_iteration=lambda it, st, ex: glog.append(ex))
    assert len(glog) == 2 and all((ex["returns"] < 0).all() for ex in glog)
    rlog = []
    RS.set_default_noise(noise)
    RS.run_master(None, str(tmp_path / "rs"), _exp("hardmaze_es.json", episodes_per_batch=16), max_iterations=1,
                  n_slots=8, noise=noise, seed=3, on_iteration=lambda it, st, ex: rlog.append(ex))
    assert len(rlog) == 1 and rlog[0]["returns_n2"].shape == (16, 1)
    env = MazeEnv(2)
    pol = policies.MujocoPolicy(env.observation_space, env.action_space, seed=1, **_exp("hardmaze_es.json")["policy"]["args"])
    rews, t, bc = pol.rollout(env, timestep_limit=400, random_stream=np.random.RandomState(0))
    assert rews.shape == (1,) and rews[0] < 0 and t == 400 and bc.shape == (2,)


# ------------------------------------------------------------------------------------------------------------------------
class _Reached(Exception):
    pass


def test_ns_learns_hard_maze(noise):
    """hardmaze_nses.json (NS-ES) at seed 0 plays a noiseless episode that ends within 10 units of the goal (the reference's
    reachgoal) within LEARN_MAX_GENERATIONS.  Every generation appends the final (x, y) of the updated parent's noiseless
    episode to the archive; that is the episode checked."""
    from es_distributed import nses as NS
    exp = _exp("hardmaze_nses.json")
    NS.set_default_noise(noise)
    best = []

    def on_it(it, stats, extra):
        x, y = extra["archive"].seqs[-1]
        best.append(math.hypot(x - 31.0, y - 20.0))
        if best[-1] < LEARN_RADIUS:
            raise _Reached(it)
    with pytest.raises(_Reached) as e:
        NS.run_master(None, None, exp, max_iterations=LEARN_MAX_GENERATIONS, noise=noise, seed=0, on_iteration=on_it)
    print(f"NS reached the goal after {e.value.args[0]} generations (distances {[round(b) for b in best[::10]]})")
