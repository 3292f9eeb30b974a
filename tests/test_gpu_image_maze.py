"""GPU tests of the image hard maze (dne_image_maze_*, dne.envs.ImageMazeEnv) against tests/image_maze_oracle.py.

* The background and the rendered frames equal the referee's bit for bit: the rendering rule is float32 arithmetic with
  explicit roundings and no transcendental.
* The dynamics are dne_maze_episodes' device code, whose only difference from tests/maze_oracle.py is CUDA's double
  cos / sin against glibc's in the velocity (at most a few double ulps, tests/test_gpu_maze.py); rounded to float32 that
  changes the position only where the double product lies within those ulps of a float32 rounding boundary, about one
  step in 2^27.  So whole episodes of every action are compared bit for bit.
* End to end, RolloutRunner on ImageMazeEnv against the same runner on HostImageMaze, a host twin built from the referee:
  identical observations give identical forwards, so returns, lengths and final positions must be identical."""
import ctypes as C
import json
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
import image_maze_oracle as IO                     # noqa: E402
import maze_oracle as M                            # noqa: E402
from dne import _ffi as F                          # noqa: E402
from dne.engine import make_context                # noqa: E402
from dne.envs import BatchEnv, Box, Discrete, ImageMazeEnv, make_env   # noqa: E402
from dne.noise import SharedNoiseTable             # noqa: E402
from dne.rollout import RolloutRunner, Unit          # noqa: E402

NOISE_COUNT = 6_000_000
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations")
f32 = np.float32
MAZE = M.load_maze()
BG = IO.background(MAZE)
GEOM = IO.geometry(MAZE.walls)


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def noise(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device="cuda:0")


@pytest.fixture(scope="module")
def ctx(noise):
    return make_context(0, noise)


def _state_tuple(row):
    return M.State(f32(row[0]), f32(row[1]), f32(row[2]), f32(row[3]), f32(row[4]), bool(row[6] != 0), int(row[5]))


def _random_states(rs, n):
    """float64 [n, 7] states whose navigators sit near walls, at and past the frame's edges, in the open, at every
    heading quadrant and its edges, some collided."""
    x0, y0, upp, _ = (float(v) for v in GEOM)
    ext = 84 * upp
    s = np.zeros((n, 7))
    for m in range(n):
        kind = m % 4
        if kind == 0:                              # within 6..10 units of a point of a wall
            w = MAZE.walls[rs.randint(len(MAZE.walls))]
            u = rs.uniform()
            ang = rs.uniform(0, 2 * np.pi)
            r = rs.uniform(6, 10)
            x, y = w[0] + u * (w[2] - w[0]) + r * np.cos(ang), w[1] + u * (w[3] - w[1]) + r * np.sin(ang)
        elif kind == 1:                            # near an edge of the frame, inside or outside it
            x, y = rs.uniform(x0 - 10, x0 + ext + 10), rs.uniform(y0 - 10, y0 + ext + 10)
            if rs.rand() < 0.5:
                x = rs.choice([x0, x0 + ext]) + rs.uniform(-9, 9)
            else:
                y = rs.choice([y0, y0 + ext]) + rs.uniform(-9, 9)
        else:
            x, y = rs.uniform(x0, x0 + ext), rs.uniform(y0, y0 + ext)
        h = rs.choice([0.0, 90.0, 180.0, 270.0, 360.0]) if m % 7 == 0 else rs.uniform(0, 360)
        s[m, :3] = f32(x), f32(y), f32(h)
        s[m, 3:5] = f32(rs.uniform(-3, 3)), f32(rs.uniform(-3, 3))
        s[m, 5] = rs.randint(0, 400)
        s[m, 6] = float(m % 5 == 0)
    return s


def _reset(desc, bg, init, slots, state, stack):
    d_init = torch.from_numpy(np.ascontiguousarray(init)).to(DEV)
    d_slots = torch.from_numpy(np.asarray(slots, np.int32)).to(DEV)
    return F.lib().dne_image_maze_reset(C.byref(desc), F.ptr(bg), F.ptr(d_init), F.ptr(d_slots), len(slots),
                                        F.ptr(state), F.ptr(stack), F.stream_ptr())


# ---- kernels against the referee ---------------------------------------------------------------------------------------
def test_background_matches_referee():
    env = ImageMazeEnv(1)
    got = env._bufs()["background"].cpu().numpy()
    assert got.tobytes() == BG.tobytes()


def test_frames_match_referee():
    """2400 states through dne_image_maze_reset: all four planes of each stack are the referee's frame, bit for bit."""
    env = ImageMazeEnv(1)
    bg = env._bufs()["background"]
    rs = np.random.RandomState(5)
    n = 2400
    init = _random_states(rs, n)
    slots = rs.permutation(n)
    state = torch.full((n, 7), -1.0, dtype=torch.float64, device=DEV)
    stack = torch.zeros(n, 84, 84, 4, dtype=torch.uint8, device=DEV)
    assert _reset(env.desc, bg, init, slots, state, stack) == 0
    got_state, got = state.cpu().numpy(), stack.cpu().numpy()
    np.testing.assert_array_equal(got_state[slots], init)
    bad = []
    drawn = 0
    for e in range(n):
        want = IO.frame(MAZE, BG, init[e, 0], init[e, 1], init[e, 2], GEOM)
        drawn += int((want != BG).any())
        if got[slots[e]].tobytes() != IO.fill(want).tobytes():
            bad.append(e)
    assert not bad, f"{len(bad)} frames differ, first state {init[bad[0]]}"
    assert drawn > n // 2                           # most navigators lie inside the frame


def test_step_contract():
    env = ImageMazeEnv(2)
    b = env._bufs()
    L = F.lib()
    tab = env.action_table.ctypes.data_as(C.c_void_p)
    d = torch.zeros(4, dtype=torch.int32, device=DEV)
    args = (F.ptr(d), F.ptr(d), 1, F.ptr(b["state"]), F.ptr(b["stack"]), F.ptr(b["rew"]), F.ptr(b["done"]), None,
            F.stream_ptr())
    assert L.dne_image_maze_step(C.byref(env.desc), F.ptr(b["background"]), tab, 9, *args) == 0
    assert L.dne_image_maze_step(C.byref(env.desc), F.ptr(b["background"]), tab, 33, *args) == -1
    assert L.dne_image_maze_step(C.byref(env.desc), F.ptr(b["background"]), None, 9, *args) == -1
    assert L.dne_image_maze_step(C.byref(F.MazeDesc(n_walls=0)), F.ptr(b["background"]), tab, 9, *args) == -1
    assert L.dne_image_maze_background(C.byref(F.MazeDesc(n_walls=65)), F.ptr(b["background"]), F.stream_ptr()) == -1
    assert "walls" in L.dne_last_error().decode()
    point = F.MazeDesc(n_walls=1)                   # one wall of zero length spans no area
    assert L.dne_image_maze_background(C.byref(point), F.ptr(b["background"]), F.stream_ptr()) == -1
    torch.cuda.synchronize()
    env.reset([0, 1])
    with pytest.raises(ValueError, match="action index"):
        env.step([0], [9])
    with pytest.raises(ValueError, match="actions for"):
        env.step([0, 1], [1])


def test_episodes_of_every_action_match_referee():
    """36 slots, 400 steps: slots 0..8 repeat one action each, the rest play random action sequences, some slots are
    reset mid-episode.  Every step's reward, done flag and position, the final states and the full frame stacks after
    every step equal the referee's."""
    n, T = 36, 400
    env = ImageMazeEnv(n)
    rs = np.random.RandomState(11)
    acts = np.concatenate([np.tile(np.arange(9)[:, None], (1, T)), rs.randint(0, 9, (n - 9, T))]).astype(np.int64)
    env.reset(np.arange(n))
    ref_s = [M.reset_state(MAZE)] * n
    ref_stack = [IO.fill(IO.frame(MAZE, BG, MAZE.start[0], MAZE.start[1], 0.0, GEOM))] * n
    stack = env.device_obs(0, n).cpu().numpy()
    assert all(stack[m].tobytes() == ref_stack[m].tobytes() for m in range(n))
    ep_t = np.zeros(n, np.int64)
    dones = 0
    for t in range(T + 150):
        live = np.nonzero(ep_t < T)[0]
        if len(live) == 0:
            break
        if t == 150:                               # restart a few slots mid-episode: the next frames come after a reset
            again = np.array([3, 17, 30])
            env.reset(again)
            for m in again:
                ref_s[m] = M.reset_state(MAZE)
                ref_stack[m] = IO.fill(IO.frame(MAZE, BG, MAZE.start[0], MAZE.start[1], 0.0, GEOM))
                ep_t[m] = 0
            live = np.nonzero(ep_t < T)[0]
        a = acts[live, ep_t[live]]
        rew, done = env.step(live, a)
        pos = env.get_ram(live)
        got = env.device_obs(0, n).cpu().numpy()
        for k, m in enumerate(live):
            ref_s[m], r, d = IO.step(MAZE, ref_s[m], a[k])
            ref_stack[m] = IO.push(ref_stack[m], IO.frame(MAZE, BG, ref_s[m].x, ref_s[m].y, ref_s[m].heading, GEOM))
            assert rew[k] == r and done[k] == d, (t, m, rew[k], r)
            assert pos[k, 0] == ref_s[m].x and pos[k, 1] == ref_s[m].y, (t, m, pos[k], ref_s[m])
            assert got[m].tobytes() == ref_stack[m].tobytes(), (t, m)
            dones += int(d)
        ep_t[live] += 1
    assert dones == n                              # the restarted slots' first episodes never ended
    fin = env._bufs()["state"].cpu().numpy()
    for m in range(n):
        assert _state_tuple(fin[m]) == ref_s[m], m
    moved = [np.hypot(float(s.x) - 36.0, float(s.y) - 184.0) for s in ref_s]
    assert sum(d > 20 for d in moved) > n // 3


# ---- the runner against a host twin ------------------------------------------------------------------------------------
class HostImageMaze(BatchEnv):
    """The image maze on the host: the referee's step and frames into a pinned observation table."""

    def __init__(self, n_slots):
        self.n_slots = n_slots
        self.observation_space = Box(0, 255, (84, 84, 4), dtype=np.uint8)
        self.action_space = Discrete(9)
        self.max_episode_steps = 400
        self.states = [M.reset_state(MAZE)] * n_slots
        self.obs = torch.zeros(n_slots, 84, 84, 4, dtype=torch.uint8).pin_memory()

    def reset(self, slots):
        for s in np.asarray(slots, np.int64):
            self.states[s] = M.reset_state(MAZE)
            self.obs[int(s)] = torch.from_numpy(IO.fill(IO.frame(MAZE, BG, MAZE.start[0], MAZE.start[1], 0.0, GEOM)))

    def step(self, slots, actions):
        rew, done = np.zeros(len(slots), np.float32), np.zeros(len(slots), bool)
        for k, (s, a) in enumerate(zip(np.asarray(slots, np.int64), np.asarray(actions).reshape(-1))):
            n, rew[k], done[k] = IO.step(MAZE, self.states[s], int(a))
            self.states[s] = n
            fr = IO.frame(MAZE, BG, n.x, n.y, n.heading, GEOM)
            self.obs[int(s)] = torch.from_numpy(IO.push(self.obs[int(s)].numpy(), fr))
        return rew, done

    def get_ram(self, slots):
        return np.array([[float(self.states[s].x), float(self.states[s].y)] for s in np.asarray(slots, np.int64)])


@pytest.mark.parametrize("ptype,group", [("LargeModelPolicy", 1), ("GAAtariPolicy", 1), ("ESAtariPolicy", 2)])
def test_runner_matches_host_twin(ctx, noise, ptype, group):
    from es_distributed import es as ES
    from es_distributed import policies
    ES.set_default_noise(noise)
    n_slots = 8
    dev_env, twin = ImageMazeEnv(n_slots), HostImageMaze(n_slots)
    pol = getattr(policies, ptype)(dev_env.observation_space, dev_env.action_space, seed=4, ctx=ctx)
    P = pol.num_params
    ref = None
    if pol.needs_ref_batch:
        rb_dev = ES.get_ref_batch(dev_env, batch_size=16, rs=np.random.RandomState(3))
        rb_host = ES.get_ref_batch(twin, batch_size=16, rs=np.random.RandomState(3))
        assert all(a.tobytes() == b.tobytes() for a, b in zip(rb_dev, rb_host))
        pol.set_ref_batch(rb_dev)
        ref = pol.ref_batch
    rs = np.random.RandomState(9)
    if group == 1:                                 # GA offspring of two parents; 11 units over 8 slots: ragged refills
        theta = torch.stack([pol.device_theta, pol.device_theta * 0.5])
        units = [Unit(int(rs.randint(0, NOISE_COUNT - P)), (f32(0.01),), theta_idx=i % 2) for i in range(11)]
    else:                                          # +- pairs; 7 pairs over 4 pair slots
        theta = pol.device_theta
        units = [Unit(int(rs.randint(0, NOISE_COUNT - P)), (f32(0.02), f32(-0.02))) for _ in range(7)]
    out = []
    for env in (dev_env, twin):
        r = RolloutRunner(ctx, pol.net, env, n_slots, group=group, pipeline=2, ref_batch=ref)
        out.append(r.run(theta, units, None, collect_bc="final"))
    a, b = out
    np.testing.assert_array_equal(a.returns, b.returns)
    np.testing.assert_array_equal(a.lengths, b.lengths)
    assert (a.lengths == 400).all() and (a.returns < 0).all()
    fa = np.array([bc for u in a.bcs for bc in u])
    fb = np.array([bc for u in b.bcs for bc in u])
    assert fa.shape == (len(units) * group, 2) and fa.tobytes() == fb.tobytes()
    print(f"{ptype}: final distances {np.round(-a.returns.ravel(), 1).tolist()}")
    with pytest.raises(NotImplementedError, match="no RAM trace"):
        RolloutRunner(ctx, pol.net, dev_env, n_slots, group=group, pipeline=2, ref_batch=ref).run(
            theta, units[:1], 5, collect_bc="trace")


# ---- drivers ------------------------------------------------------------------------------------------------------------
def _exp(name, **over):
    with open(os.path.join(CONFIGS, name)) as f:
        exp = json.load(f)
    exp["config"].update(snapshot_freq=0, **over)
    return exp


def test_drivers_run_on_image_maze(noise, tmp_path):
    from es_distributed import es as ES
    from es_distributed import ga as GA
    from es_distributed import nses as NS
    from es_distributed import rs as RS
    ES.set_default_noise(noise)
    glog = []
    exp = _exp("image_hardmaze_ga.json")
    exp.update(population_size=12, selection_threshold=4, validation_threshold=3, num_validation_episodes=2)
    GA.run_master(None, str(tmp_path / "ga"), exp, max_iterations=2, n_slots=8, noise=noise, seed=5,
                  on_iteration=lambda it, st, ex: glog.append((st, ex)))
    assert len(glog) == 2
    for st, ex in glog:
        assert len(ex["returns"]) == 12 and (ex["returns"] < 0).all()
        assert ex["val_returns"].shape == (3, 2) and (ex["val_returns"][:, 0] == ex["val_returns"][:, 1]).all()
        assert "TruncatedPopulationEliteValidationRewMean" in st
    for algo in ("ns", "nsr"):
        nlog = []
        exp = _exp("image_hardmaze_nses.json", episodes_per_batch=8)
        exp.update(algo_type=algo)
        exp["novelty_search"].update(population_size=2, k=3)
        NS.run_master(None, str(tmp_path / algo), exp, max_iterations=2, n_slots=8, noise=noise, seed=2,
                      on_iteration=lambda it, st, ex: nlog.append(ex))
        assert len(nlog) == 2 and all(np.asarray(b).shape == (2,) for b in nlog[0]["bcs"])
        assert np.isfinite(nlog[-1]["novelty_n2"]).all() and len(nlog[-1]["archive"]) == 4
    elog = []
    exp = _exp("image_hardmaze_nses.json", episodes_per_batch=8, return_proc_mode="centered_rank")
    ES.run_master(None, None, exp, max_iterations=2, n_slots=8, noise=noise, seed=3,
                  on_iteration=lambda it, st, ex: elog.append(ex))
    assert len(elog) == 2 and elog[0]["returns_n2"].shape == (4, 2) and (elog[0]["lengths_n2"] == 400).all()
    rlog = []
    RS.run_master(None, str(tmp_path / "rs"), _exp("image_hardmaze_ga.json", episodes_per_batch=8), max_iterations=1,
                  n_slots=8, noise=noise, seed=3, on_iteration=lambda it, st, ex: rlog.append(ex))
    assert len(rlog) == 1 and rlog[0]["returns_n2"].shape == (8, 1) and (rlog[0]["returns_n2"] < 0).all()
    assert isinstance(make_env("ImageHardMaze-v0", 8), ImageMazeEnv)
