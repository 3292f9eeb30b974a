"""Host tests of the hard maze: the scalar referee (tests/maze_oracle.py) against the reference's own code
(tests/golden/ref_maze.npz, written by oracle/maze_ref.cpp around the reference's maze.h), bit for bit; the maze-file
parser, the registration, the spaces and the configurations.  No GPU."""
import json
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import maze_oracle as M                            # noqa: E402
from dne import envs as E                          # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CONFIGS = os.path.join(os.path.dirname(HERE), "deep-neuroevolution_b200", "configurations")
f32 = np.float32


@pytest.fixture(scope="module")
def golden():
    with np.load(os.path.join(HERE, "golden", "ref_maze.npz")) as z:
        return {k: z[k] for k in z.files}


def _row(maze, s, r):
    ob = M.observation(maze, s.x, s.y, s.heading)
    return np.array([s.x, s.y, s.heading, s.speed, s.ang_vel, float(s.collide), s.t, r] + list(ob), np.float32)


def _state(r):
    return M.State(*[f32(v) for v in r[:5]], bool(r[5] != 0), int(r[6]))


def test_reset_observation(golden):
    maze = M.load_maze()
    s = M.reset_state(maze)
    assert M.observation(maze, s.x, s.y, s.heading).tobytes() == golden["reset_obs"].tobytes()


@pytest.mark.parametrize("which", ["step", "sticky"])
def test_single_steps_bit_for_bit(golden, which):
    maze = M.load_maze()
    if which == "sticky":
        maze = maze._replace(disable=True)
    inp, out = golden[f"{which}_in"], golden[f"{which}_out"]
    assert len(inp) >= (4000 if which == "step" else 500)
    bad = [i for i, (r, o) in enumerate(zip(inp, out))
           if _row(maze, *M.step(maze, _state(r), r[7], r[8])).tobytes() != o.tobytes()]
    assert not bad, f"{len(bad)} steps differ, first {bad[:5]}"
    if which == "step":                         # the fixture reaches the events it is meant to cover
        assert np.isnan(out).any() and (out[:, 7] < 0).any()
        assert (np.abs(out[:, 3]) == 3).any() and (np.abs(out[:, 4]) == 3).any()
        moved = (out[:, 0] != inp[:, 0]) | (out[:, 1] != inp[:, 1])
        assert (~moved & (inp[:, 3] != 0) & (inp[:, 5] == 0)).sum() > 100        # wall contacts that stopped a move
    else:
        assert (out[:, 5] == 1).sum() > 100


def test_open_loop_episodes_bit_for_bit(golden):
    maze = M.load_maze()
    acts, out = golden["ep_actions"], golden["ep_out"]
    assert acts.shape[0] >= 24 and acts.shape[1] == 400
    for e in range(len(acts)):
        s = M.reset_state(maze)
        for t in range(400):
            s, r = M.step(maze, s, acts[e, t, 0], acts[e, t, 1])
            row = _row(maze, s, r)
            assert row.tobytes() == out[e, t].tobytes(), (e, t, row, out[e, t])
    assert (out[:, :399, 7] == 0).all() and (out[:, 399, 7] < 0).all()


def test_parser_and_registration():
    walls, start, goal, sticky = E.parse_maze(E.DEFAULT_MAZE_FILE)
    assert walls.shape == (13, 4) and walls.dtype == np.float32
    assert start == (36.0, 184.0) and goal == (31.0, 20.0) and not sticky
    ref = M.load_maze()
    assert np.array_equal(walls, ref.walls)
    env = E.make_env("maze", 4)
    assert isinstance(env, E.MazeEnv) and env.max_episode_steps == 400
    assert env.observation_space.shape == (11,) and env.action_space.shape == (2,)
    assert (env.action_space.low == -0.5).all() and (env.action_space.high == 0.5).all()
    assert env.state_dim == 7 and env.bc_dim == 2
    assert env.device_episodes and env.kernel_policy_io and not env.host_step
    s = env.initial_states(3)
    assert s.shape == (3, 7) and (s[:, :2] == [36.0, 184.0]).all() and (s[:, 2:] == 0).all()
    assert env.desc.n_walls == 13 and env.desc.collisions_stick == 0 and tuple(env.desc.goal) == (31.0, 20.0)
    assert [env.desc.walls[12][k] for k in range(4)] == [56.0, 55.0, 133.0, 30.0]
    with pytest.raises(ValueError):
        E.make_env("maze", 4, episode_len=100)
    with pytest.raises(NotImplementedError):
        env.reset(np.arange(2))


def test_parser_rejects_malformed(tmp_path):
    bad = tmp_path / "bad.txt"
    bad.write_text("0\n400\n3\n1 2\n0\n3 4\n5 6\n0 0 1 1\n")
    with pytest.raises(ValueError, match="3 walls announced"):
        E.parse_maze(str(bad))
    many = tmp_path / "many.txt"
    many.write_text("1\n400\n65\n1 2\n0\n3 4\n5 6\n" + "0 0 1 1\n" * 65)
    with pytest.raises(ValueError, match="at most 64"):
        E.parse_maze(str(many))
    sticky = tmp_path / "sticky.txt"
    sticky.write_text("1" + open(E.DEFAULT_MAZE_FILE).read()[1:])
    env = E.make_env("maze", 2, maze_file=str(sticky))
    assert env.collisions_stick and env.desc.collisions_stick == 1


def test_configurations():
    for name, algo, proc in (("hardmaze_nses.json", "ns", "centered_sign_rank"), ("hardmaze_es.json", None, "centered_rank")):
        with open(os.path.join(CONFIGS, name)) as f:
            exp = json.load(f)
        assert exp["env_id"] == "maze" and exp.get("algo_type") == algo
        assert exp["config"]["return_proc_mode"] == proc      # NS ranks the novelty, which the driver passes as sign-returns
        assert exp["policy"]["type"] == "MujocoPolicy" and exp["policy"]["args"]["ac_bins"] == "continuous:"
        assert exp["config"]["episode_cutoff_mode"] == "env_default"


def test_make_runner_refuses_a_host_action_map_on_a_kernel_only_env():
    from dne.rollout import make_runner
    env = E.MazeEnv(2)
    with pytest.raises(NotImplementedError, match="continuous"):
        make_runner(None, None, env, action_fn=lambda a: a)
