"""Host tests of the image hard maze: the referee's background of the hard maze against hand-checked pixels, its heading
marker and frame stack, the registration, the spaces, the factory's errors, the behaviour-characterisation choice of
NS-ES for every environment, and the shipped configurations.  No GPU."""
import inspect
import json
import math
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import image_maze_oracle as IO                     # noqa: E402
import maze_oracle as M                            # noqa: E402
from dne import _ffi as F                          # noqa: E402
from dne import envs as E                          # noqa: E402
from dne import nets, raw_env                      # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIGS = os.path.join(os.path.dirname(HERE), "deep-neuroevolution_b200", "configurations")
f32 = np.float32
MAZE = M.load_maze()


@pytest.fixture(scope="module")
def bg():
    return IO.background(MAZE)


def test_geometry_of_the_hard_maze():
    # walls span x 3..195 and y 5..202: the larger extent, 197 units, maps onto 84 pixels
    x0, y0, upp, half = IO.geometry(MAZE.walls)
    assert (x0, y0) == (3.0, 5.0) and upp == f32(197.0) / f32(84.0) and half == upp / 2


def test_background_hand_checked_pixels(bg):
    """Pixel (row i, column j) has its centre at (3 + (j + 0.5) * 2.3452, 5 + (i + 0.5) * 2.3452); a wall pixel is one
    whose centre lies within half a pixel (1.1726 units) of a wall."""
    assert bg.shape == (84, 84) and bg.dtype == np.uint8 and set(np.unique(bg)) == {0, 255}
    # the left wall (4, 49) -> (7, 202) passes x = 5.0 at y = 100; row 40's centre is y = 99.98: column 0 (x = 4.17) is
    # 0.83 from it, column 1 (x = 6.52) 1.52
    assert bg[40, 0] == 255 and bg[40, 1] == 0
    # the bottom wall (7, 202) -> (195, 198) at column 41 (x = 100.33) lies at y = 200.01: row 83 (y = 200.83) is 0.82
    # from it, row 82 (y = 198.48) 1.53
    assert bg[83, 41] == 255 and bg[82, 41] == 0
    # the top wall (186, 8) -> (39, 5) at column 60 (x = 144.9) lies at y = 7.16: row 0 (y = 6.17) is 0.99 from it,
    # row 1 (y = 8.52) 1.36
    assert bg[0, 60] == 255 and bg[1, 60] == 0
    # the open corridor around (120, 100) and the start (36, 184) are clear
    assert bg[40, 49] == 0 and bg[75, 14] == 0
    # the shorter x extent (192 units, 81.9 pixels) leaves the last two columns (centres x >= 196.5) without walls
    assert not bg[:, 82:].any() and bg[:, 81].any()
    # about one pixel per 2.3 units of the walls' 1100 units of length
    assert 450 < int((bg == 255).sum()) < 900


def test_heading_marker_and_disc(bg):
    for h in np.arange(0.0, 360.0, 7.5).astype(np.float32).tolist() + [90.0, 180.0, 270.0, 360.0]:
        hx, hy = IO.heading_dir(h)
        assert abs(float(hx) - math.cos(math.radians(h))) < 2e-3 and abs(float(hy) - math.sin(math.radians(h))) < 2e-3
    x, y = f32(120.0), f32(100.0)                  # in the open: the disc is all navigator
    # the disc covers rows 37..43 and columns 46..52 around pixel (40, 49.4); the front pixel of each heading
    for h, front in ((0.0, (40, 52)), (90.0, (43, 49)), (180.0, (40, 47)), (270.0, (37, 49))):
        fr = IO.frame(MAZE, bg, x, y, h)
        assert fr[front] == 64, h
        assert int((fr == 64).sum()) + int((fr == 128).sum()) in range(30, 50)
        assert abs(int((fr == 64).sum()) - int((fr == 128).sum())) <= 8
        diff = fr != bg
        assert (fr[diff] != 255).all() and (bg[~diff] == fr[~diff]).all()


def test_stack_push_and_fill():
    a, b = np.full((84, 84), 1, np.uint8), np.full((84, 84), 2, np.uint8)
    st = IO.fill(a)
    assert st.shape == (84, 84, 4) and (st == 1).all()
    st = IO.push(st, b)
    assert (st[:, :, :3] == 1).all() and (st[:, :, 3] == 2).all()


def test_referee_step_maps_the_action_table():
    s = M.reset_state(MAZE)
    for a, (turn, speed) in enumerate(IO.DEFAULT_ACTIONS):
        n, r, done = IO.step(MAZE, s, a)
        want, _ = M.step(MAZE, s, turn, speed)
        assert n == want and r == 0 and not done
    assert len(IO.DEFAULT_ACTIONS) == 9 and sorted(set(IO.DEFAULT_ACTIONS.ravel().tolist())) == [-0.5, 0.0, 0.5]


# ---- registration, spaces, factory -----------------------------------------------------------------------------------
def test_registration_and_spaces():
    env = E.make_env("ImageHardMaze-v0", 4)
    assert isinstance(env, E.ImageMazeEnv)
    assert env.observation_space.shape == (84, 84, 4) and env.observation_space.low.dtype == np.uint8
    assert int(env.observation_space.high.max()) == 255 and env.action_space.n == 9 and env.max_episode_steps == 400
    np.testing.assert_array_equal(env.action_table, IO.DEFAULT_ACTIONS)
    assert env.bc_kind == "final" and env.bc_dim == 2
    assert isinstance(E.make_env("maze", 4), E.MazeEnv)                   # the maze prefix is untouched
    assert not isinstance(E.make_env("maze", 4), E.ImageMazeEnv)
    env.reset(np.array([1, 3]))
    np.testing.assert_array_equal(env.get_ram([1, 3]), [[36.0, 184.0]] * 2)
    assert env.random_actions(100, np.random.RandomState(0)).max() < 9
    custom = E.make_env("ImageHardMaze-v0", 2, actions=[[0.5, 0.5], [-0.5, 0.5]], maze_file=M.FIXTURE)
    assert custom.action_space.n == 2 and custom.maze_file == M.FIXTURE


def test_factory_errors(tmp_path):
    with pytest.raises(ValueError, match="fixed 400-step"):
        E.make_env("ImageHardMaze-v0", 4, episode_len=100)
    for bad in ([[0.5]], np.zeros((33, 2)), np.zeros((0, 2))):
        with pytest.raises(ValueError, match="actions"):
            E.ImageMazeEnv(2, actions=bad)
    empty = tmp_path / "empty.txt"
    empty.write_text("0\n400\n0\n1 2\n0\n3 4\n5 6\n")
    with pytest.raises(ValueError, match="at least one wall"):
        E.ImageMazeEnv(2, maze_file=str(empty))
    with pytest.raises(KeyError):
        E.make_env("ImageHardMaze", 2)


def test_bc_mode_default_unchanged_for_existing_environments():
    from es_distributed.nses import choose_bc_mode
    atari, vector = nets.make_net("Model", num_actions=4), nets.make_net("MujocoPolicy", ob_dim=11, ac_dim=2)
    classes = [c for mod in (E, raw_env) for _, c in inspect.getmembers(mod, inspect.isclass)
               if issubclass(c, E.BatchEnv) and c is not E.ImageMazeEnv]
    assert len(classes) >= 10
    for c in classes:
        assert getattr(c, "bc_kind", None) is None, c
        assert choose_bc_mode(c, atari) == "trace" and choose_bc_mode(c, vector) == "final"
    assert choose_bc_mode(E.ImageMazeEnv, atari) == "final"


def test_configurations():
    with open(os.path.join(CONFIGS, "image_hardmaze_ga.json")) as f:
        ga = json.load(f)
    assert ga["env_id"] == "ImageHardMaze-v0" and ga["policy"]["type"] == "LargeModelPolicy"
    assert {"selection_threshold", "validation_threshold", "num_validation_episodes"} <= set(ga)   # Deep GA
    with open(os.path.join(CONFIGS, "image_hardmaze_nses.json")) as f:
        ns = json.load(f)
    assert ns["env_id"] == "ImageHardMaze-v0" and ns["policy"]["type"] == "ESAtariPolicy" and ns["algo_type"] == "ns"
    assert ns["config"]["return_proc_mode"] == "centered_sign_rank"
    for exp in (ga, ns):
        assert exp["config"]["episode_cutoff_mode"] == "env_default"
    assert F.IMAGE_MAZE_MAX_ACTIONS == 32
