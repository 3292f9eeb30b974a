"""GPU tests of the discrete-action episode kernel (dne_discrete_episodes) on Acrobot-v1 and MountainCar-v0, and of the
drivers running on it.

Referee: tests/discrete_oracle.py (oracle.forward + gymnasium's equations in numpy float64).  Exact agreement is not
defined for every step: the oracle's float32 matmul sums in a different order than the kernel, and CUDA's double sin / cos
are not correctly rounded.  An episode is MARGINAL when it has a logit gap below 1e-4 at some decision, or a visited
quantity within 1e-9 of a termination, wrap or clip threshold; only marginal episodes may be excluded from a comparison,
and the tests print how many were.  Acrobot is chaotic over 500 steps, so its whole episodes are checked transition by
transition instead of end to end."""
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

from oracle import oracle as O                    # noqa: E402
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cartpole_oracle as CP                       # noqa: E402
import discrete_oracle as D                        # noqa: E402
from dne import _ffi as F                          # noqa: E402
from dne import nets                               # noqa: E402
from dne.engine import make_context                # noqa: E402
from dne.envs import AcrobotEnv, MountainCarEnv    # noqa: E402
from dne.noise import SharedNoiseTable             # noqa: E402
from dne.rollout import EpisodeKernelRunner, Unit  # noqa: E402

NOISE_COUNT = 2_000_000
GAP, MARGIN = 1e-4, 1e-9
PI = math.pi
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations")
# |kernel - referee| after one step, per state component.  CUDA's double sin / cos are within 2 ulp, glibc's within 1;
# one RK4 step multiplies such a difference by at most a few hundred, so 1e-12 holds with room while a referee with the
# "nips" dynamics or a wrong torque misses it by orders of magnitude.  MountainCar's step is three roundings deep.
STEP_ATOL = {"acrobot": 1e-12, "mountaincar": 1e-15}


class Task:
    def __init__(self, name, env_id, cls, ob_dim, state_dim, limit):
        self.name, self.env_id, self.cls = name, env_id, cls
        self.ob_dim, self.state_dim, self.limit = ob_dim, state_dim, limit


TASKS = {"acrobot": Task("acrobot", F.EPISODE_ACROBOT, AcrobotEnv, 6, 4, 500),
         "mountaincar": Task("mountaincar", F.EPISODE_MOUNTAINCAR, MountainCarEnv, 2, 2, 200)}


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def noise(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device="cuda:0")


@pytest.fixture(scope="module")
def ctx(noise):
    return make_context(0, noise)


def _launch(ctx, task, net, theta, idx, scale, rows, init, max_steps, final=True):
    """dne_discrete_episodes on numpy inputs -> (rc, returns, lengths, final states) as numpy."""
    dev = torch.device("cuda", 0)
    n = len(idx)
    th = torch.from_numpy(np.ascontiguousarray(theta, dtype=np.float32)).to(dev)

    def buf(a, dt, width=1):               # n == 0 still hands the library valid (non-null) one-row buffers
        a = np.asarray(a, dt).reshape(n, width)
        return torch.from_numpy(np.ascontiguousarray(a if n else np.zeros((1, width), dt))).to(dev)
    sd = task.state_dim
    d_idx, d_sc = buf(idx, np.int64), buf(scale, np.float32)
    d_row = None if rows is None else buf(rows, np.int32)
    d_init = buf(init, np.float64, sd)
    ret = torch.full((max(n, 1),), -7.0, dtype=torch.float32, device=dev)
    ln = torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev)
    fin = torch.full((max(n, 1), sd), -7.0, dtype=torch.float64, device=dev) if final else None
    rc = F.lib().dne_discrete_episodes(ctx.handle, task.env_id, C.byref(net.desc), F.ptr(th), F.ptr(d_idx), F.ptr(d_sc),
                                       F.ptr(d_row), n, F.ptr(d_init), int(max_steps), F.ptr(ret), F.ptr(ln), F.ptr(fin),
                                       F.stream_ptr())
    torch.cuda.synchronize()
    return rc, ret.cpu().numpy()[:n], ln.cpu().numpy()[:n], (fin.cpu().numpy()[:n] if final else None)


def _nets(task, name="SimpleClassifier"):
    return (nets.make_net(name, num_actions=3, ob_dim=task.ob_dim),
            CP.make_classifier(name, num_actions=3, ob_dim=task.ob_dim))


def _member(theta_rows, host_noise, idx, s, row):
    P = theta_rows.shape[1]
    return (theta_rows[row] + np.float32(s) * host_noise[idx:idx + P]).astype(np.float32)      # fl(theta + fl(s * n))


def _mixed_population(rs, P, n=512, n_rows=4):
    """± pairs on random noise indices (row 0), scale-0 members, GA-style members on rows of a [n_rows, P] matrix."""
    n_pair, n_zero = n // 4, n // 8
    n_ga = n - 2 * n_pair - n_zero
    pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n_pair)
    idx = np.concatenate([np.repeat(pidx, 2), rs.randint(0, NOISE_COUNT - P + 1, size=n_zero),
                          rs.randint(0, NOISE_COUNT - P + 1, size=n_ga)]).astype(np.int64)
    scale = np.concatenate([np.tile([0.05, -0.05], n_pair), np.zeros(n_zero),
                            rs.choice([0.02, 0.1, -0.3], size=n_ga)]).astype(np.float32)
    rows = np.concatenate([np.zeros(2 * n_pair + n_zero), rs.randint(0, n_rows, size=n_ga)]).astype(np.int32)
    return idx, scale, rows


def _theta_rows(rs, P, n_rows, sd=0.5):
    return np.stack([(rs.randn(P) * sd).astype(np.float32) for _ in range(n_rows)])


def _obs(task, states):
    return D.acrobot_obs(states) if task.name == "acrobot" else np.asarray(states, np.float64).astype(np.float32)


def _policy_logits(onet, members, task, states):
    """Oracle logits [n, T, 3] of member m at its states [n, T, state_dim]."""
    return np.stack([O.forward(onet, members[m], _obs(task, states[m]))[0] for m in range(len(members))])


def _gap(logits):
    top = np.sort(logits.astype(np.float64), axis=-1)
    return top[..., -1] - top[..., -2]


def _referee_step(task, states, actions, **wrong):
    if task.name == "acrobot":
        ns, rew, done, raw = D.acrobot_step(states, actions, **wrong)
        return ns, rew, done, D.acrobot_margin(ns, raw)
    out = [D.mountaincar_step(s, (int(a) + wrong.get("torque_offset", 0)) % 3) for s, a in zip(states, actions)]
    return (np.stack([o[0] for o in out]), np.array([o[1] for o in out]), np.array([o[2] for o in out]),
            np.array([o[3] for o in out]))


def _state_err(task, got, want):
    """Per-member max |got - want| over the components, the angles compared modulo 2 pi."""
    d = np.abs(np.asarray(got) - np.asarray(want))
    if task.name == "acrobot":
        d[..., :2] = np.minimum(d[..., :2], np.abs(d[..., :2] - 2 * PI))
    return d.max(axis=-1)


def _random_states(task, rs, n):
    if task.name == "acrobot":
        return np.stack([rs.uniform(-PI, PI, n), rs.uniform(-PI, PI, n), rs.uniform(-4 * PI, 4 * PI, n),
                         rs.uniform(-9 * PI, 9 * PI, n)], axis=1)
    return np.stack([rs.uniform(-1.2, 0.6, n), rs.uniform(-0.07, 0.07, n)], axis=1)


def _special_states(task):
    """The states the step's branches hinge on."""
    if task.name == "acrobot":
        line = 2 * PI / 3                                      # -cos(t1) - cos(t2 + t1) = 1 at t1 = 2pi/3, t2 = 0
        return np.array([[PI, 0, 0, 0], [-PI, 0, 0, 0], [0, PI, 0, 0], [0, -PI, 0, 0], [PI, -PI, 1, -1],
                         [0, 0, 4 * PI, 0], [0, 0, -4 * PI, 0], [0, 0, 0, 9 * PI], [0, 0, 0, -9 * PI],
                         [0, 0, 4 * PI, 9 * PI], [0, 0, -4 * PI, -9 * PI], [PI - 1e-3, 0, 4 * PI, 0],
                         [line, 0, 0, 0], [line + 1e-3, 0, 0, 0], [line - 1e-3, 0, 0, 0], [0, 0, 0, 0]])
    return np.array([[-1.2, 0.0], [-1.2, -0.07], [-1.2, 0.07], [-1.19, -0.05], [-PI / 3, 0.069], [-PI / 3, 0.07],
                     [0.0, -0.069], [0.0, -0.07], [0.5, 0.0], [0.49, 0.01], [0.55, -0.01], [0.59, 0.06], [0.6, 0.07],
                     [-0.5, 0.0]])


# ---- 1. chained launches -----------------------------------------------------------------------------------------------
def _chain(ctx, task, net, theta, idx, scale, rows, init, T):
    """T chained one-step launches, each from the previous final states, for the members still running.  Returns
    (lengths, returns (float64 sums of the one-step returns), final states, the trajectory [n, T + 1, sd] padded with
    the final state, the per-step rewards [n, T])."""
    n, sd = len(idx), task.state_dim
    traj = np.repeat(np.asarray(init, np.float64)[:, None, :], T + 1, axis=1)
    rew = np.zeros((n, T))
    length = np.zeros(n, np.int64)
    ret = np.zeros(n)
    alive = np.ones(n, bool)
    state = np.asarray(init, np.float64).copy()
    rows = np.zeros(n, np.int32) if rows is None else rows
    for t in range(T):
        act = np.nonzero(alive)[0]
        if len(act) == 0:
            break
        rc, r, ln, fin = _launch(ctx, task, net, theta, idx[act], scale[act], rows[act], state[act], 1)
        assert rc == 0 and (ln == 1).all()
        state[act] = fin
        traj[act, t + 1:] = fin[:, None, :]
        rew[act, t] = r
        ret[act] += r.astype(np.float64)
        length[act] += 1
        if task.name == "acrobot":
            done = r == 0.0                                     # reward 0 only on the terminating step
        else:
            done = (fin[:, 0] >= 0.5) & (fin[:, 1] >= 0.0)      # the termination test on the exact state
        alive[act[done]] = False
    return length, ret, state, traj, rew


@pytest.mark.parametrize("task_name", ["acrobot", "mountaincar"])
def test_one_launch_equals_chained_one_step_launches(ctx, task_name):
    task = TASKS[task_name]
    net, onet = _nets(task)
    rs = np.random.RandomState(3 + len(task_name))
    theta = _theta_rows(rs, net.num_params, 4)
    idx, scale, rows = _mixed_population(rs, net.num_params)
    init = task.cls(4, seed=5).initial_states(len(idx))
    rc, ret, ln, fin = _launch(ctx, task, net, theta, idx, scale, rows, init, task.limit)
    assert rc == 0 and (ln >= 1).all() and (ln <= task.limit).all()
    c_len, c_ret, c_fin, _, _ = _chain(ctx, task, net, theta, idx, scale, rows, init, task.limit)
    np.testing.assert_array_equal(ln, c_len)
    assert fin.tobytes() == c_fin.tobytes()
    np.testing.assert_array_equal(ret, c_ret.astype(np.float32))
    if task.name == "mountaincar":
        np.testing.assert_array_equal(ret, -ln.astype(np.float32))
    else:
        term = ln < task.limit                                  # reward 0 on the terminating step
        np.testing.assert_array_equal(ret, np.where(term, -(ln - 1), -ln).astype(np.float32))
    print(f"{task.name}: mean length {ln.mean():.1f}, {int((ln < task.limit).sum())} of {len(ln)} terminated")


# ---- 2. one step against the referee -----------------------------------------------------------------------------------
@pytest.mark.parametrize("task_name", ["acrobot", "mountaincar"])
def test_one_step_within_bound_of_referee(ctx, host_noise, task_name):
    task = TASKS[task_name]
    net, onet = _nets(task)
    rs = np.random.RandomState(17 + len(task_name))
    theta = _theta_rows(rs, net.num_params, 4)
    idx, scale, rows = _mixed_population(rs, net.num_params)
    n = len(idx)
    special = _special_states(task)
    init = _random_states(task, rs, n)
    init[:len(special) * 4] = np.tile(special, (4, 1))            # every special state under several members
    rc, ret, ln, fin = _launch(ctx, task, net, theta, idx, scale, rows, init, 1)
    assert rc == 0 and (ln == 1).all()
    members = np.stack([_member(theta, host_noise, int(idx[m]), scale[m], int(rows[m])) for m in range(n)])
    logits = _policy_logits(onet, members, task, init[:, None, :])[:, 0]
    actions = np.argmax(logits, axis=1)
    want, rew, done, margin = _referee_step(task, init, actions)
    err = _state_err(task, fin, want)
    atol = STEP_ATOL[task.name]
    marginal = (_gap(logits) < GAP) | (margin < MARGIN)
    bad = np.nonzero((err > atol) & ~marginal)[0]
    assert len(bad) == 0, f"members {bad[:8].tolist()}: |kernel - referee| {err[bad[:8]]} > {atol}"
    np.testing.assert_array_equal(ret[~marginal], rew[~marginal].astype(np.float32))
    print(f"{task.name}: max error {err[~marginal].max():.2e} (bound {atol}), {int(marginal.sum())} of {n} marginal")
    # sharpness: wrong referees miss the bound on most members
    wrongs = {"torque index off by one": dict(torque_offset=1)}
    if task.name == "acrobot":
        wrongs["nips dynamics"] = dict(book=False)
    for what, kw in wrongs.items():
        w = _referee_step(task, init, actions, **kw)[0]
        rejected = (_state_err(task, fin, w) > atol)[~marginal].mean()
        print(f"{task.name}: a referee with {what} is rejected on {rejected:.1%} of the members")
        assert rejected > 0.5, what


# ---- 3. whole Acrobot episodes, transition by transition ---------------------------------------------------------------
def test_acrobot_episodes_step_by_step(ctx, host_noise):
    task = TASKS["acrobot"]
    net, onet = _nets(task)
    rs = np.random.RandomState(31)
    theta = _theta_rows(rs, net.num_params, 4)
    idx, scale, rows = _mixed_population(rs, net.num_params)
    n = len(idx)
    init = AcrobotEnv(4, seed=8).initial_states(n)
    length, _, _, traj, rew = _chain(ctx, task, net, theta, idx, scale, rows, init, task.limit)
    members = np.stack([_member(theta, host_noise, int(idx[m]), scale[m], int(rows[m])) for m in range(n)])
    atol = STEP_ATOL["acrobot"]
    checked = skipped_actions = 0
    for m in range(n):
        T = int(length[m])
        s = traj[m, :T]
        logits = O.forward(onet, members[m], D.acrobot_obs(s))[0]
        # the kernel's action: the one whose referee step lands within the bound of the kernel's next state
        errs = np.stack([_state_err(task, traj[m, 1:T + 1], _referee_step(task, s, np.full(T, a))[0]) for a in range(3)])
        hit = errs <= atol
        assert hit.any(axis=0).all(), f"member {m}: steps {np.nonzero(~hit.any(axis=0))[0][:8].tolist()} match no action"
        kernel_action = np.argmax(hit, axis=0)
        gap = _gap(logits)
        sure = gap >= GAP
        bad = np.nonzero(sure & (kernel_action != np.argmax(logits, axis=1)))[0]
        assert len(bad) == 0, f"member {m}: steps {bad[:8].tolist()} act against the oracle forward"
        # the reward: 0 exactly on a terminating step, unless the state is on the line
        ns, r, _, mg = _referee_step(task, s, kernel_action)
        on_line = mg < MARGIN
        np.testing.assert_array_equal(rew[m, :T][~on_line], r[~on_line])
        checked += T
        skipped_actions += int((~sure).sum())
    print(f"acrobot: {checked} transitions checked, {skipped_actions} actions not compared (logit gap < {GAP}); "
          f"mean length {length.mean():.1f}")


# ---- 4. MountainCar against the oracle ---------------------------------------------------------------------------------
def _check_episodes(got_len, got_fin, eps, what, atol_state=1e-12):
    marginal = np.array([e.min_logit_gap < GAP or e.min_threshold_margin < MARGIN for e in eps])
    want = np.array([e.length for e in eps])
    fin = np.stack([e.final_state for e in eps])
    differ = (got_len != want) | (np.abs(got_fin - fin).max(axis=1) > atol_state)
    bad = np.nonzero(differ & ~marginal)[0]
    assert len(bad) == 0, f"{what}: episodes {bad[:8].tolist()} differ without being marginal: " \
                          f"got lengths {got_len[bad[:8]]}, oracle {want[bad[:8]]}"
    excluded = int(differ.sum())
    print(f"{what}: {excluded} of {len(eps)} episodes excluded (differ, all marginal); {int(marginal.sum())} flagged marginal")
    assert excluded <= 0.01 * len(eps)


@pytest.mark.parametrize("max_steps", [1, 2, 10, 200])
def test_mountaincar_episodes_match_oracle(ctx, host_noise, max_steps):
    task = TASKS["mountaincar"]
    net, onet = _nets(task)
    rs = np.random.RandomState(40 + max_steps)
    theta = _theta_rows(rs, net.num_params, 4, sd=3.0)           # large weights: the velocity input matters
    idx, scale, rows = _mixed_population(rs, net.num_params, n=256)
    init = MountainCarEnv(4, seed=max_steps).initial_states(len(idx))
    if max_steps <= 10:                                          # also start next to the goal and the wall
        init[::4] = _random_states(task, rs, len(init[::4]))
    rc, ret, ln, fin = _launch(ctx, task, net, theta, idx, scale, rows, init, max_steps)
    assert rc == 0
    np.testing.assert_array_equal(ret, -ln.astype(np.float32))
    eps = [D.episode("mountaincar", onet, _member(theta, host_noise, int(idx[m]), scale[m], int(rows[m])), init[m],
                     max_steps) for m in range(len(idx))]
    print(f"max_steps={max_steps}: {int((ln < max_steps).sum())} reached the goal")
    _check_episodes(ln, fin, eps, f"mountaincar max_steps={max_steps}")


# ---- 5. argmax -------------------------------------------------------------------------------------------------------
def test_three_action_argmax_rule(ctx):
    """A linear net with zero weights: the logits are its biases.  The action is read back from MountainCar's velocity
    (each action changes it by a distinct 0.001)."""
    task = TASKS["mountaincar"]
    net = nets.make_net("LinearClassifier", num_actions=3, ob_dim=2)
    inf, nan = np.inf, np.nan
    cases = [([1, 3, 3], 1), ([3, 3, 3], 0), ([1, 2, 3], 2), ([nan, 5, 9], 0), ([1, nan, nan], 1), ([9, 1, nan], 2),
             ([inf, 1, 2], 0), ([1, inf, inf], 1), ([inf, 1, nan], 2), ([-inf, -inf, -inf], 0), ([-inf, -inf, -5], 2),
             ([-inf, 0, nan], 2), ([0.0, -0.0, 0.0], 0)]
    P = net.num_params
    theta = np.zeros((len(cases), P), np.float32)
    lb = net.layers[0]
    for i, (b, _) in enumerate(cases):
        theta[i, lb.off_b:lb.off_b + 3] = np.array(b, np.float32)
    n = len(cases)
    init = np.tile([[-0.5, 0.0]], (n, 1))
    rc, _, ln, fin = _launch(ctx, task, net, theta, np.zeros(n, np.int64), np.zeros(n, np.float32),
                             np.arange(n, dtype=np.int32), init, 1)
    assert rc == 0
    got = [int(np.argmin([abs(D.mountaincar_step(init[i], a)[0][1] - fin[i, 1]) for a in range(3)])) for i in range(n)]
    assert got == [a for _, a in cases]


# ---- 6. argument and net contract --------------------------------------------------------------------------------------
def _custom_net(widths, act=F.ACT_RELU):
    layers = [nets._dense(widths[i], widths[i + 1], act=act) for i in range(len(widths) - 2)]
    layers.append(nets._dense(widths[-2], widths[-1], act=F.ACT_NONE))
    return nets._finish(nets.NetSpec("custom", layers, F.OB_VECTOR, widths[0]))


@pytest.mark.parametrize("task_name", ["acrobot", "mountaincar"])
def test_contract(ctx, host_noise, task_name):
    task = TASKS[task_name]
    net, onet = _nets(task)
    rs = np.random.RandomState(8)
    theta = _theta_rows(rs, net.num_params, 4)
    idx, scale, rows = _mixed_population(rs, net.num_params, n=64)
    init = task.cls(4, seed=1).initial_states(64)
    a = _launch(ctx, task, net, theta, idx, scale, rows, init, task.limit)
    b = _launch(ctx, task, net, theta, idx, scale, rows, init, task.limit)
    assert a[0] == b[0] == 0
    for x, y in zip(a[1:], b[1:]):
        assert x.tobytes() == y.tobytes()                      # bit-identical reruns
    dev = torch.device("cuda", 0)
    th = torch.from_numpy(theta[0]).to(dev)
    d_idx = torch.zeros(4, dtype=torch.int64, device=dev)
    d_sc = torch.zeros(4, dtype=torch.float32, device=dev)
    d_init = torch.zeros(4, task.state_dim, dtype=torch.float64, device=dev)
    d_ret = torch.full((4,), -7.0, dtype=torch.float32, device=dev)
    d_len = torch.full((4,), -1, dtype=torch.int32, device=dev)
    L = F.lib()

    def call(n_, max_steps, net_=net, env=task.env_id):
        return L.dne_discrete_episodes(ctx.handle, env, C.byref(net_.desc), F.ptr(th), F.ptr(d_idx), F.ptr(d_sc), None,
                                       n_, F.ptr(d_init), max_steps, F.ptr(d_ret), F.ptr(d_len), None, F.stream_ptr())
    assert call(0, 10) == 0                                     # n_members == 0: a no-op
    torch.cuda.synchronize()
    assert (d_ret == -7.0).all() and (d_len == -1).all()
    assert call(4, 0) == -1                                     # DNE_ERR_ARG
    assert call(4, task.limit + 1) == -1
    assert call(-1, 10) == -1
    assert call(4, 10, env=7) == -1
    assert call(4, task.limit) == 0
    # unsupported nets
    other = 2 if task.ob_dim == 6 else 6
    unsup = {"ob_dim": nets.make_net("SimpleClassifier", num_actions=3, ob_dim=other),
             "n_out": nets.make_net("SimpleClassifier", num_actions=2, ob_dim=task.ob_dim),
             "width 33": _custom_net([task.ob_dim, 33, 3]),
             "tanh hidden": _custom_net([task.ob_dim, 16, 3], act=F.ACT_TANH),
             "conv net": nets.make_net("Model", num_actions=3)}
    for what, bad in unsup.items():
        assert call(4, 10, bad) == -4, what                     # DNE_ERR_UNSUP
        assert L.dne_last_error().decode().startswith("dne_discrete_episodes"), what
    # the widest net (4 layers of width 32) runs and agrees with the oracle for a few steps
    w32 = _custom_net([task.ob_dim, 32, 32, 32, 3])
    o32 = CP.dense_net([task.ob_dim, 32, 32, 32, 3])
    assert o32.num_params == w32.num_params
    t32 = (rs.randn(1, w32.num_params) * 0.3).astype(np.float32)
    i32 = rs.randint(0, NOISE_COUNT - w32.num_params + 1, size=64).astype(np.int64)
    s32 = np.full(64, 0.05, np.float32)
    rc, _, ln, fin = _launch(ctx, task, w32, t32, i32, s32, None, init, 3)
    assert rc == 0
    members = np.stack([_member(t32, host_noise, int(i32[m]), s32[m], 0) for m in range(64)])
    st = init.copy()
    sure = np.ones(64, bool)
    for _ in range(3):
        lg = _policy_logits(o32, members, task, st[:, None, :])[:, 0]
        st, _, _, mg = _referee_step(task, st, np.argmax(lg, axis=1))
        sure &= (_gap(lg) >= GAP) & (mg >= MARGIN)
    assert sure.mean() > 0.9
    assert (_state_err(task, fin, st)[sure] <= 10 * STEP_ATOL[task.name]).all()


# ---- 7. runner ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task_name", ["acrobot", "mountaincar"])
def test_runner_matches_direct_launch(ctx, task_name):
    task = TASKS[task_name]
    net, _ = _nets(task)
    rs = np.random.RandomState(12)
    theta = torch.from_numpy((rs.randn(3, net.num_params) * 0.5).astype(np.float32)).cuda()
    units = [Unit(int(rs.randint(0, NOISE_COUNT - 400)), (0.02, -0.02), theta_idx=i % 3) for i in range(20)]
    r = EpisodeKernelRunner(ctx, net, task.cls(4, seed=33), n_slots=4, group=2)
    res = r.run(theta, units, 5000, collect_bc="final")
    init = task.cls(4, seed=33).initial_states(40)
    idx = np.repeat([u.noise_idx for u in units], 2)
    scale = np.tile([0.02, -0.02], 20).astype(np.float32)
    rows = np.repeat([u.theta_idx for u in units], 2)
    rc, ret, ln, fin = _launch(ctx, task, net, theta.cpu().numpy(), idx, scale, rows, init, task.limit)
    assert rc == 0
    np.testing.assert_array_equal(res.lengths.ravel(), ln)
    np.testing.assert_array_equal(res.returns.ravel(), ret)
    np.testing.assert_array_equal(res.signreturns.ravel(), ret)
    np.testing.assert_array_equal(np.stack([b for u in res.bcs for b in u]), fin)
    assert fin.shape == (40, task.state_dim) and res.steps == int(ln.sum()) and res.ticks == 1


# ---- 8. drivers --------------------------------------------------------------------------------------------------------
def _exp(fname, **over):
    with open(os.path.join(CONFIGS, fname)) as f:
        exp = json.load(f)
    exp["config"].update(snapshot_freq=0, **over)
    return exp


@pytest.mark.parametrize("task_name", ["acrobot", "mountaincar"])
def test_es_run_master_matches_oracle(noise, host_noise, tmp_path, task_name):
    from es_distributed import es as ES
    from es_distributed import policies
    task = TASKS[task_name]
    seed, env_seed = 11, 6
    exp = _exp("acrobot_es.json", episodes_per_batch=64, eval_prob=0.05)
    exp["env_id"] = {"acrobot": "Acrobot-v1", "mountaincar": "MountainCar-v0"}[task_name]
    cfg = exp["config"]
    log = []

    def on_it(it, stats, extra):
        log.append((dict(stats), {k: (v.clone() if hasattr(v, "clone") else np.array(v)) for k, v in extra.items()
                                  if k in ("noise_inds_n", "returns_n2", "lengths_n2", "g", "theta")}))
    ES.set_default_noise(noise)
    env = task.cls(8, seed=env_seed)
    theta_final = ES.run_master(None, str(tmp_path), exp, max_iterations=2, n_slots=8, env=env, noise=noise, seed=seed,
                                on_iteration=on_it)
    assert len(log) == 2
    onet = CP.make_classifier("SimpleClassifier", num_actions=3, ob_dim=task.ob_dim)
    P = onet.num_params
    theta = policies.SimpleClassifierPolicy(env.observation_space, env.action_space, seed=seed).get_trainable_flat()
    adam = O.Adam(theta, exp["optimizer"]["args"]["stepsize"])
    rs, env_ref = np.random.RandomState(seed), task.cls(8, seed=env_seed)
    for stats, ex in log:
        n_pairs = 32
        n_eval = int(rs.binomial(n_pairs, cfg["eval_prob"]))
        idx = np.array([O.sample_index(rs, NOISE_COUNT, P) for _ in range(n_pairs)], dtype=np.int64)
        np.testing.assert_array_equal(ex["noise_inds_n"], idx)
        init = env_ref.initial_states((n_pairs + -(-n_eval // 2)) * 2)
        ret = ex["returns_n2"]
        if task.name == "mountaincar":                # whole episodes against the oracle (Acrobot's are chaotic: test 3)
            np.testing.assert_array_equal(ret, -ex["lengths_n2"].astype(np.float32))
            eps = [D.episode("mountaincar", onet, O.perturb(adam.theta, host_noise, int(idx[u]), cfg["noise_stdev"],
                                                            1 - 2 * g), init[2 * u + g], task.limit)
                   for u in range(n_pairs) for g in range(2)]
            _check_episodes(ex["lengths_n2"].ravel(), np.stack([e.final_state for e in eps]), eps, "ES generation",
                            atol_state=np.inf)
        g, ratio, new_theta = O.es_generation_update(adam.theta, adam, host_noise, idx, ret, cfg["l2coeff"])
        assert np.abs(ex["g"].cpu().numpy() - g).max() <= 1e-5 * max(np.abs(g).max(), 1e-30)
        np.testing.assert_allclose(ex["theta"].cpu().numpy(), new_theta, rtol=0, atol=2e-7)
        assert stats["UpdateRatio"] == pytest.approx(float(ratio), rel=1e-4)
        assert stats["EvalEpCount"] == n_eval
    np.testing.assert_allclose(theta_final, adam.theta, rtol=0, atol=2e-7)


@pytest.mark.parametrize("task_name", ["acrobot", "mountaincar"])
@pytest.mark.parametrize("ga_mode", ["cpu", "gpu"])
def test_ga_run_master_completes(noise, tmp_path, task_name, ga_mode):
    from es_distributed import ga as GA
    task = TASKS[task_name]
    exp = _exp("acrobot_es.json", episodes_per_batch=24)
    exp.update(population_size=4, num_elites=1, ga_mode=ga_mode)
    log = []
    GA.set_default_noise(noise)
    pop, score = GA.run_master(None, str(tmp_path), exp, max_iterations=2, n_slots=8, env=task.cls(8, seed=2),
                               noise=noise, seed=5, on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 2 and len(pop) == 4
    for ex in log:
        assert len(ex["genomes"]) == 24 and (ex["returns"] <= 0).all() and (ex["returns"] >= -task.limit).all()


@pytest.mark.parametrize("task_name", ["acrobot", "mountaincar"])
def test_nsr_es_rs_and_rollout_complete(noise, tmp_path, task_name):
    from es_distributed import es as ES
    from es_distributed import nses as NS
    from es_distributed import policies
    from es_distributed import rs as RS
    task = TASKS[task_name]
    exp = _exp("acrobot_es.json", episodes_per_batch=16, return_proc_mode="centered_sign_rank")
    exp.update(algo_type="nsr", novelty_search={"k": 3, "population_size": 2, "num_rollouts": 1,
                                                "selection_method": "novelty_prob"})
    NS.set_default_noise(noise)
    log = []
    NS.run_master(None, str(tmp_path / "ns"), exp, max_iterations=1, n_slots=8, env=task.cls(8, seed=3), noise=noise,
                  seed=2, on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 1 and log[0]["returns_n2"].shape == (8, 2)
    assert all(np.asarray(b).shape == (task.state_dim,) and np.asarray(b).dtype == np.float64 for b in log[0]["bcs"])
    assert np.isfinite(log[0]["novelty_n2"]).all()
    rlog = []
    RS.set_default_noise(noise)
    RS.run_master(None, str(tmp_path / "rs"), _exp("acrobot_es.json", episodes_per_batch=16), max_iterations=1,
                  n_slots=8, env=task.cls(8, seed=4), noise=noise, seed=3, on_iteration=lambda it, st, ex: rlog.append(ex))
    assert len(rlog) == 1 and rlog[0]["returns_n2"].shape == (16, 1) and rlog[0]["best_score"] <= 0
    ES.set_default_noise(noise)
    env = task.cls(2, seed=0)
    pol = policies.SimpleClassifierPolicy(env.observation_space, env.action_space, seed=1)
    rews, t, bc = pol.rollout(env, timestep_limit=50)
    assert rews.shape == (1,) and 1 <= t <= 50 and -t <= rews[0] <= 0 and bc.shape == (task.state_dim,)
    a = pol.act(np.zeros((3, task.ob_dim), np.float32))
    assert a.shape == (3,) and set(a.tolist()) <= {0, 1, 2}


# ---- 9. learning -------------------------------------------------------------------------------------------------------
class _Reached(Exception):
    pass


# generations within which the shipped configurations (seed 0) must learn: about twice what an H100 run measured
ACROBOT_MAX_GENERATIONS = 6              # reached after 3 on an H100
MOUNTAINCAR_MAX_GENERATIONS = 16         # reached after 8 on an H100


def _noiseless(ctx, task, theta):
    net = nets.make_net("SimpleClassifier", num_actions=3, ob_dim=task.ob_dim)
    ev = EpisodeKernelRunner(ctx, net, task.cls(2, seed=12345), group=2)
    return ev.run(theta, [Unit(0, (0.0, 0.0)) for _ in range(50)], None)


def test_es_learns_acrobot(noise):
    """acrobot_es.json reaches a mean noiseless return >= -100 over 100 episodes (gym's reward threshold)."""
    from es_distributed import es as ES
    task = TASKS["acrobot"]
    ES.set_default_noise(noise)
    ctx = ES.default_context()
    history = []

    def on_it(it, stats, extra):
        history.append(float(_noiseless(ctx, task, extra["theta"]).returns.mean()))
        if history[-1] >= -100:
            raise _Reached(it)
    with pytest.raises(_Reached) as e:
        ES.run_master(None, None, _exp("acrobot_es.json"), max_iterations=ACROBOT_MAX_GENERATIONS,
                      env=AcrobotEnv(8, seed=0), noise=noise, seed=0, on_iteration=on_it)
    print(f"ES reached mean noiseless return {history[-1]:.1f} after {e.value.args[0]} generations; "
          f"history {[round(h, 1) for h in history]}")


def test_ga_learns_mountaincar(noise):
    """mountaincar_ga.json's elite reaches the goal in >= 90 of 100 noiseless episodes."""
    from es_distributed import ga as GA
    task = TASKS["mountaincar"]
    GA.set_default_noise(noise)
    ctx = GA.default_context()
    history = []

    def on_it(it, stats, extra):
        res = _noiseless(ctx, task, extra["elite_theta"])
        history.append((int((res.lengths < task.limit).sum()), float(res.returns.mean())))
        if history[-1][0] >= 90:
            raise _Reached(it)
    with pytest.raises(_Reached) as e:
        GA.run_master(None, None, _exp("mountaincar_ga.json"), max_iterations=MOUNTAINCAR_MAX_GENERATIONS,
                      env=MountainCarEnv(8, seed=0), noise=noise, seed=0, n_slots=256, on_iteration=on_it)
    goals, mean = history[-1]
    print(f"GA's elite reached the goal in {goals} of 100 noiseless episodes after {e.value.args[0]} generations, mean "
          f"return {mean:.1f} ({'reaches' if mean >= -110 else 'does not reach'} -110); history {history}")
