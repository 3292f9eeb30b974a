"""GPU tests of MujocoPolicy's discretised heads ('uniform:N', 'custom:v0,..,vk') inside the Pendulum-v1 and hard-maze
episode kernels (dne_pendulum_binned_episodes, dne_maze_binned_episodes; DESIGN.md 3.9), their runner and the drivers.

Referees:
* the kernels themselves: one launch of T steps equals T chained one-step launches bit for bit; the single-CTA kernel
  equals the cluster kernel at every cluster size; reruns are bit-identical;
* the rules (first NaN, else first maximum; noise after the bin; the table's values) on constructed weights, each
  read back through one step of the task's oracle from a state whose observation and step the kernel computes exactly;
* the scores against the float64 forward referee of tests/test_gpu_dense_paths.py: wherever the referee's top bin beats
  every other by more than both bounds, the kernel's one step equals the oracle stepped with that bin's value;
* Pendulum episodes against the per-tick RolloutRunner with the policy's host action_fn.
"""
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
import maze_oracle as M                            # noqa: E402
import pendulum_oracle as PO                       # noqa: E402
from test_gpu_dense_paths import member, referee   # noqa: E402  (the float64 forward referee)
from dne import _ffi as F                          # noqa: E402
from dne import nets                               # noqa: E402
from dne.engine import make_context                # noqa: E402
from dne.envs import Box, MazeEnv, PendulumEnv     # noqa: E402
from dne.noise import SharedNoiseTable             # noqa: E402
from dne.rollout import EpisodeKernelRunner, RolloutRunner, Unit, make_runner   # noqa: E402

NOISE_COUNT = 2_000_000
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations")
f32 = np.float32
MAZE = M.load_maze()
# the per-tick comparison's tolerances: test_gpu_pendulum.py's at 200 steps
STATE_TOL_200, RETURN_RTOL_200 = 1e-3, 2e-5
# task -> (ob_dim, action dimensions, state_dim, episode length, entry)
TASKS = {"pendulum": (3, 1, 2, 200, "dne_pendulum_binned_episodes"), "maze": (11, 2, 7, 400, "dne_maze_binned_episodes")}


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def noise(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device="cuda:0")


@pytest.fixture(scope="module")
def ctx(noise):
    return make_context(0, noise)


def _net(task, nb, hidden=(64, 64), act=F.ACT_TANH, n_out=None):
    ob, adim = TASKS[task][:2]
    dims = [ob] + list(hidden)
    layers = [nets._dense(dims[i], dims[i + 1], act=act) for i in range(len(hidden))]
    layers.append(nets._dense(dims[-1], adim * nb if n_out is None else n_out, act=F.ACT_NONE))
    return nets._finish(nets.NetSpec(task, layers, F.OB_VECTOR, ob))


def _uniform(task, nb):
    """'uniform:nb' over the task's action bounds, as MujocoPolicy builds it."""
    lo, hi = (np.array([-2.0], f32), np.array([2.0], f32)) if task == "pendulum" else (np.full(2, -0.5, f32),
                                                                                        np.full(2, 0.5, f32))
    return (f32(1.0 / (nb - 1.0)) * np.arange(nb, dtype=f32)[None, :] * (hi - lo)[:, None] + lo[:, None]).astype(f32)


def _cuda(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(DEV)


def _launch(ctx, task, net, bins, theta, idx, scale, rows, init, T, ob_mean=None, ob_std=None, ac_noise=None,
            stats=True, cluster=0, n_bins=None):
    """dne_<task>_binned_episodes on numpy inputs -> dict of numpy outputs (and 'rc')."""
    ob, adim, sd = TASKS[task][:3]
    n = len(idx)
    k = max(n, 1)
    d = dict(ret=torch.full((k,), -1.0, dtype=torch.float32, device=DEV),
             sret=torch.full((k,), -1.0, dtype=torch.float32, device=DEV),
             len=torch.full((k,), -1, dtype=torch.int32, device=DEV),
             fin=torch.full((k, sd), -7.0, dtype=torch.float64, device=DEV))
    if stats:
        d["s"] = torch.full((k, ob), -7.0, dtype=torch.float64, device=DEV)
        d["q"] = torch.full((k, ob), -7.0, dtype=torch.float64, device=DEV)
    args = [_cuda(theta, np.float32), _cuda(idx, np.int64), _cuda(scale, np.float32),
            None if rows is None else _cuda(rows, np.int32), _cuda(init, np.float64),
            None if ob_mean is None else _cuda(ob_mean, np.float32), None if ob_std is None else _cuda(ob_std, np.float32),
            None if ac_noise is None else _cuda(ac_noise, np.float32)]
    tab = None if bins is None else np.ascontiguousarray(bins, dtype=f32)
    head = (C.byref(MazeEnv(1).desc),) if task == "maze" else ()
    rc = getattr(F.lib(), TASKS[task][4])(
        ctx.handle, *head, C.byref(net.desc), F.ptr(args[0]), F.ptr(args[1]), F.ptr(args[2]), F.ptr(args[3]), n,
        F.ptr(args[4]), int(T), F.ptr(args[5]), F.ptr(args[6]), F.ptr(args[7]), F.ptr(d["ret"]), F.ptr(d["sret"]),
        F.ptr(d["len"]), F.ptr(d["fin"]), F.ptr(d.get("s")), F.ptr(d.get("q")),
        None if tab is None else tab.ctypes.data_as(C.c_void_p), int(tab.shape[1] if n_bins is None else n_bins),
        int(cluster), F.stream_ptr())
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


def _inits(task, rs, n):
    if task == "pendulum":
        return np.stack([rs.uniform(-np.pi, np.pi, n), rs.uniform(-1, 1, n)], axis=1)
    return MazeEnv(1).initial_states(n)


# ---- bit identity ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["pendulum", "maze"])
@pytest.mark.parametrize("stats,noisy", [(True, True), (False, False)])
def test_one_launch_equals_chained_one_step_launches(ctx, task, stats, noisy):
    nb = 10 if task == "maze" else 5
    net, bins = _net(task, nb), _uniform(task, nb)
    ob, adim, _, T, _ = TASKS[task]
    P = net.num_params
    rs = np.random.RandomState(3 + 2 * stats + noisy)
    theta = (rs.randn(4, P) * 0.3).astype(f32)
    idx, scale, rows = _mixed(rs, P)
    n = len(idx)
    init = _inits(task, rs, n)
    mean, std = (rs.randn(ob).astype(f32) * 0.1, rs.uniform(0.5, 1.0, ob).astype(f32)) if stats else (None, None)
    acn = (rs.randn(n, T, adim) * 0.05).astype(f32) if noisy else None
    if noisy:
        acn[scale == 0] = 0.0
    full = _launch(ctx, task, net, bins, theta, idx, scale, rows, init, T, mean, std, acn, stats)
    assert full["rc"] == 0 and (full["len"] == T).all()
    st = init.copy()
    ret, sret = np.zeros(n), np.zeros(n)
    s, q = np.zeros((n, ob)), np.zeros((n, ob))
    for t in range(T):
        one = _launch(ctx, task, net, bins, theta, idx, scale, rows, st, 1, mean, std,
                      None if acn is None else acn[:, t:t + 1], stats)
        assert one["rc"] == 0
        st = one["fin"]
        ret += one["ret"].astype(np.float64)
        sret += one["sret"].astype(np.float64)
        if stats:
            s += one["s"]
            q += one["q"]
    assert full["fin"].tobytes() == st.tobytes()
    assert full["ret"].tobytes() == ret.astype(f32).tobytes()
    assert full["sret"].tobytes() == sret.astype(f32).tobytes()
    if stats:
        assert full["s"].tobytes() == s.tobytes() and full["q"].tobytes() == q.tobytes()
    again = _launch(ctx, task, net, bins, theta, idx, scale, rows, init, T, mean, std, acn, stats)
    for key in [k for k in full if k != "rc"]:
        assert again[key].tobytes() == full[key].tobytes()      # bit-identical reruns
    assert len(np.unique(full["fin"][:, 0])) > 10                # the members went their own ways


@pytest.mark.parametrize("task,hidden,nb", [("pendulum", (64, 64), 5), ("pendulum", (200, 200), 32),
                                            ("maze", (64, 64), 10), ("maze", (96, 40), 32)])
def test_single_cta_equals_cluster_at_every_size(ctx, task, hidden, nb):
    net, bins = _net(task, nb, hidden), _uniform(task, nb)
    ob, adim, _, T, _ = TASKS[task]
    P = net.num_params
    rs = np.random.RandomState(40 + nb)
    theta = (rs.randn(4, P) * 0.2).astype(f32)
    idx, scale, rows = _mixed(rs, P, n=96)
    n = len(idx)
    init = _inits(task, rs, n)
    mean, std = rs.randn(ob).astype(f32) * 0.1, rs.uniform(0.5, 1.0, ob).astype(f32)
    acn = (rs.randn(n, T, adim) * 0.05).astype(f32)
    one = _launch(ctx, task, net, bins, theta, idx, scale, rows, init, T, mean, std, acn)
    assert one["rc"] == 0
    for c in (2, 4, 8):
        cl = _launch(ctx, task, net, bins, theta, idx, scale, rows, init, T, mean, std, acn, cluster=c)
        assert cl["rc"] == 0, F.lib().dne_last_error().decode()
        for key in ("ret", "sret", "len", "fin", "s", "q"):
            assert cl[key].tobytes() == one[key].tobytes(), (c, key)


def test_wide_net_runs_on_a_cluster(ctx):
    """Maze [256, 256] with 'uniform:10': the binned entry picks a cluster itself; chained one-step launches agree."""
    net, bins = _net("maze", 10, (256, 256)), _uniform("maze", 10)
    assert F.lib().dne_maze_net_supported(C.byref(_net("maze", 1, (256, 256), n_out=2).desc)) != 0
    assert F.lib().dne_maze_binned_net_supported(C.byref(net.desc), 10) == 0
    rs = np.random.RandomState(8)
    theta = (rs.randn(1, net.num_params) * 0.1).astype(f32)
    idx, scale, _ = _mixed(rs, net.num_params, n=16, n_rows=1)
    init = _inits("maze", rs, 16)
    full = _launch(ctx, "maze", net, bins, theta, idx, scale, None, init, 20)
    assert full["rc"] == 0, F.lib().dne_last_error().decode()
    st = init.copy()
    for _ in range(20):
        st = _launch(ctx, "maze", net, bins, theta, idx, scale, None, st, 1)["fin"]
    assert full["fin"].tobytes() == st.tobytes()


# ---- the rules, on constructed weights -----------------------------------------------------------------------------------
def _head_only(task, nb):
    """A net whose only layer is the head: scores = observation . W + b."""
    return _net(task, nb, hidden=())


def _one_step(ctx, task, net, bins, w, acn=None, init=None):
    """One step of one member with weights w (scale 0) from `init` (default: Pendulum at rest, th = 0; the maze's reset)."""
    init = (np.zeros((1, 2)) if task == "pendulum" else MazeEnv(1).initial_states(1)) if init is None else init
    out = _launch(ctx, task, net, bins, w[None, :], np.zeros(1, np.int64), np.zeros(1, f32), None, init, 1,
                  ac_noise=acn, stats=False)
    assert out["rc"] == 0, F.lib().dne_last_error().decode()
    return out["fin"][0]


def _oracle_next(task, a, init=None):
    """The oracle's next state from the same state under the float32 action a [adim]."""
    if task == "pendulum":
        th, thdot = (0.0, 0.0) if init is None else init
        nth, nthdot, _ = PO.pendulum_step(th, thdot, f32(a[0]))
        return np.array([nth, nthdot])
    s, _ = M.step(MAZE, M.reset_state(MAZE), f32(a[0]), f32(a[1]))
    return np.array([s.x, s.y, s.heading, s.speed, s.ang_vel, s.t, float(s.collide)], dtype=np.float64)


def _small_bins(task):
    """Bins whose values the task's one step tells apart: for the maze from rest the rate limit (6 |a| <= 0.2) keeps
    |a| < 1/30 distinct, and the ends (+-0.5) clip to +-0.2."""
    if task == "pendulum":
        return _uniform("pendulum", 5)
    v = np.array([-0.5, -0.015, -0.01, -0.005, 0.0, 0.005, 0.01, 0.015, 0.5], f32)
    return np.stack([v, v[::-1].copy()])


@pytest.mark.parametrize("task", ["pendulum", "maze"])
def test_ties_pick_the_first_bin(ctx, task):
    bins = _small_bins(task)
    nb = bins.shape[1]
    net = _head_only(task, nb)
    w = np.zeros(net.num_params, f32)
    L = net.layers[-1]
    w[L.off_b:L.off_b + L.cout] = 0.25                        # every score 0.25
    got = _one_step(ctx, task, net, bins, w)
    np.testing.assert_array_equal(got, _oracle_next(task, bins[:, 0]))
    assert not np.array_equal(got, _oracle_next(task, bins[:, -1]))      # "last maximum" would differ


@pytest.mark.parametrize("task", ["pendulum", "maze"])
def test_nan_score_wins(ctx, task):
    bins = _small_bins(task)
    adim, nb = bins.shape
    net = _head_only(task, nb)
    L = net.layers[-1]
    w = np.zeros(net.num_params, f32)
    b = np.zeros(L.cout, f32)
    pick = [3, 1][:adim]
    for d in range(adim):
        b[d * nb + nb - 1] = 10.0                             # the largest number: the last bin
        w[L.off_w + 0 * L.cout + d * nb + pick[d]] = np.nan   # a NaN weight makes bin pick[d]'s score NaN
    w[L.off_b:L.off_b + L.cout] = b
    got = _one_step(ctx, task, net, bins, w)
    want = bins[np.arange(adim), pick]
    np.testing.assert_array_equal(got, _oracle_next(task, want))
    assert not np.array_equal(got, _oracle_next(task, bins[:, -1]))      # "maximum ignoring NaN" would differ


@pytest.mark.parametrize("task", ["pendulum", "maze"])
def test_noise_is_added_after_the_bin(ctx, task):
    bins = _small_bins(task)
    adim, nb = bins.shape
    net = _head_only(task, nb)
    L = net.layers[-1]
    w = np.zeros(net.num_params, f32)
    mid = nb // 2
    for d in range(adim):                                     # bin mid wins by 0.1 over bin 0
        w[L.off_b + d * nb + mid] = 1.0
        w[L.off_b + d * nb + 0] = 0.9
    nz = f32(0.2) if task == "pendulum" else f32(0.004)
    acn = np.full((1, 1, adim), nz, f32)
    got = _one_step(ctx, task, net, bins, w, acn)
    want = (bins[:, mid] + nz).astype(f32)
    np.testing.assert_array_equal(got, _oracle_next(task, want))
    # noise on the scores of bin 0 would pick bin 0; noise dropped would act with the bin value alone
    assert not np.array_equal(got, _oracle_next(task, bins[:, 0] + nz))
    assert not np.array_equal(got, _oracle_next(task, bins[:, mid]))


def test_custom_bins_with_asymmetric_bounds(ctx):
    from es_distributed import policies
    env = PendulumEnv(2)
    pol = policies.MujocoPolicy(env.observation_space, Box(np.array([-1.5], f32), np.array([0.5], f32)),
                                ac_bins="custom:-1,-0.5,0,1", ac_noise_std=0.0, nonlin_type="tanh", hidden_dims=[8],
                                connection_type="ff", seed=0)
    bins = pol._bin_values
    np.testing.assert_array_equal(bins, np.array([[-1.5, -1.0, -0.5, 0.5]], f32))
    net = _head_only("pendulum", 4)
    L = net.layers[-1]
    for b in range(4):
        w = np.zeros(net.num_params, f32)
        w[L.off_b + b] = 1.0
        np.testing.assert_array_equal(_one_step(ctx, "pendulum", net, bins, w), _oracle_next("pendulum", bins[:, b]))


# ---- against the referees ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["pendulum", "maze"])
def test_scores_against_float64_referee(ctx, host_noise, task):
    """One step from states whose observation the kernel computes exactly (Pendulum: th = 0, any thdot; the maze: its
    reset), where the step tells every bin apart.  Members whose referee top bin does not beat every other by more than
    both float32 bounds are excluded as near-ties."""
    bins = _small_bins(task)
    adim, nb = bins.shape
    net = _net(task, nb)
    P = net.num_params
    rs = np.random.RandomState(21)
    theta = (rs.randn(1, P) * 0.3).astype(f32)
    n = 768
    idx = rs.randint(0, NOISE_COUNT - P, n).astype(np.int64)
    scale = rs.choice([0.05, -0.1, 0.3, -0.5, 1.0], n).astype(f32)
    if task == "pendulum":
        init = np.stack([np.zeros(n), rs.uniform(-7, 7, n)], axis=1)
    else:
        init = MazeEnv(1).initial_states(n)
    got = _launch(ctx, task, net, bins, theta, idx, scale, None, init, 1, stats=False)
    assert got["rc"] == 0
    checked = excluded = 0
    chosen = set()
    for m in range(n):
        if task == "pendulum":
            x0 = np.array([1.0, 0.0, init[m, 1]], f32)        # cos 0, sin 0 exactly
        else:
            x0 = M.observation(MAZE, MAZE.start[0], MAZE.start[1], f32(0))
        w, wm = member(theta, 0, host_noise, int(idx[m]), scale[m], P)
        ref, bound = referee(net, w, wm, x0)
        ref, bound = ref.reshape(adim, nb), bound.reshape(adim, nb)
        top = np.argmax(ref, axis=1)
        clear = all(ref[d, top[d]] - bound[d, top[d]] > np.delete(ref[d] + bound[d], top[d]).max() for d in range(adim))
        if not clear:
            excluded += 1
            continue
        checked += 1
        chosen.add(tuple(top))
        want = _oracle_next(task, bins[np.arange(adim), top], None if task == "maze" else tuple(init[m]))
        np.testing.assert_array_equal(got["fin"][m], want, err_msg=f"member {m}")
    print(f"{task} binned scores: {checked} steps checked, {excluded} excluded as near-ties, {len(chosen)} bin choices")
    assert checked >= 0.9 * n and len(chosen) >= 4


def test_pendulum_kernel_against_per_tick_runner(ctx):
    """EpisodeKernelRunner(action_bins) and RolloutRunner + the policy's action_fn on the same noiseless members."""
    from es_distributed import policies
    env = PendulumEnv(2)
    pol = policies.MujocoPolicy(env.observation_space, env.action_space, ac_bins="uniform:5", ac_noise_std=0.0,
                                nonlin_type="tanh", hidden_dims=[64, 64], connection_type="ff", seed=0)
    net = pol.net
    rs = np.random.RandomState(5)
    theta = torch.from_numpy((rs.randn(net.num_params) * 0.3).astype(f32)).to(DEV)
    units = [Unit(int(rs.randint(0, NOISE_COUNT - net.num_params)), (0.05, -0.05)) for _ in range(31)] + \
            [Unit(0, (0.0, 0.0), noiseless=True)]
    mean, std = torch.tensor([0.1, 0.0, 0.2], device=DEV), torch.tensor([0.8, 0.8, 2.0], device=DEV)
    n = 2 * len(units)
    kr = EpisodeKernelRunner(ctx, net, PendulumEnv(n, seed=9), group=2, action_bins=pol._bin_values)
    pr = make_runner(ctx, net, PendulumEnv(n, seed=9), n_slots=n, group=2, pipeline=2, **pol.runner_head_kw())
    assert isinstance(pr, RolloutRunner) and pr.action_fn is not None
    k = kr.run(theta, units, None, ob_mean=mean, ob_std=std, collect_bc="final")
    p = pr.run(theta, units, None, ob_mean=mean, ob_std=std, collect_bc="final")
    np.testing.assert_array_equal(k.lengths, p.lengths)
    fk, fp = np.array([b for u in k.bcs for b in u]), np.array([b for u in p.bcs for b in u])
    d_state = float(np.abs(fk - fp).max())
    d_ret = float((np.abs(k.returns - p.returns) / np.maximum(np.abs(p.returns), 1.0)).max())
    print(f"binned per-tick referee: max |state| difference {d_state:.3g}, relative return {d_ret:.3g}")
    assert d_state <= STATE_TOL_200 and d_ret <= RETURN_RTOL_200
    np.testing.assert_array_equal(k.signreturns, p.signreturns)


# ---- the contract --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["pendulum", "maze"])
def test_contract(ctx, task):
    L = F.lib()
    probe = getattr(L, f"dne_{task}_binned_net_supported")
    adim = TASKS[task][1]
    net = _net(task, 10)
    assert probe(C.byref(net.desc), 10) == 0
    assert probe(C.byref(_net(task, 2).desc), 2) == 0 and probe(C.byref(_net(task, 32).desc), 32) == 0
    for nb, n_out, what in ((1, adim, "2..32 bins"), (33, adim * 33, "2..32 bins"), (10, adim * 10 + 1, "n_out"),
                            (10, adim * 9, "n_out")):
        bad = _net(task, nb, n_out=n_out)
        assert probe(C.byref(bad.desc), nb) == -4
        assert what in L.dne_last_error().decode()
        rng = np.random.RandomState(0)
        out = _launch(ctx, task, bad, np.zeros((adim, max(nb, 1)), f32), rng.randn(1, bad.num_params).astype(f32),
                      np.zeros(2, np.int64), np.zeros(2, f32), None, _inits(task, rng, 2), 3)
        assert out["rc"] == -4 and what in L.dne_last_error().decode()
    rng = np.random.RandomState(1)
    w, init = rng.randn(1, net.num_params).astype(f32), _inits(task, rng, 2)
    null = _launch(ctx, task, net, None, w, np.zeros(2, np.int64), np.zeros(2, f32), None, init, 3, n_bins=10)
    assert null["rc"] == -1 and "bin_values_host" in L.dne_last_error().decode()
    bad_c = _launch(ctx, task, net, _uniform(task, 10), w, np.zeros(2, np.int64), np.zeros(2, f32), None, init, 3,
                    cluster=3)
    assert bad_c["rc"] == -1
    # the continuous entries and probes still refuse a binned net
    assert getattr(L, f"dne_{task}_net_supported")(C.byref(net.desc)) == -4
    assert getattr(L, f"dne_{task}_cluster_net_supported")(C.byref(net.desc)) == -4


# ---- runner and drivers --------------------------------------------------------------------------------------------------
def test_make_runner_choices(ctx):
    from es_distributed import policies
    maze = MazeEnv(4)
    pol = policies.MujocoPolicy(maze.observation_space, maze.action_space, ac_bins="uniform:10", ac_noise_std=0.01,
                                nonlin_type="tanh", hidden_dims=[64, 64], connection_type="ff", seed=0)
    r = make_runner(ctx, pol.net, maze, n_slots=4, group=2, **pol.runner_head_kw())
    assert isinstance(r, EpisodeKernelRunner) and r.action_bins.shape == (2, 10)
    with pytest.raises(ValueError):
        make_runner(ctx, pol.net, maze, n_slots=4, group=2, action_bins=pol._bin_values)     # without its action_fn
    pend = PendulumEnv(4)
    pp = policies.MujocoPolicy(pend.observation_space, pend.action_space, ac_bins="uniform:5", ac_noise_std=0.01,
                               nonlin_type="tanh", hidden_dims=[64, 64], connection_type="ff", seed=0)
    assert pend.episode_net_supported(pp.net, pp._bin_values) and not pend.episode_net_supported(pp.net)
    assert isinstance(make_runner(ctx, pp.net, pend, n_slots=4, group=2, **pp.runner_head_kw()), RolloutRunner)
    # the runner draws [n_noisy, limit, adim] action noise: the same numbers as a direct launch with that noise
    theta = torch.from_numpy(np.asarray(pol.get_trainable_flat(), f32)).to(DEV)
    units = [Unit(1000 + 7 * i, (0.05, -0.05)) for i in range(6)]
    res = r.run(theta, units, None, ob_mean=pol.ob_mean, ob_std=pol.ob_std, collect_bc="final", ac_noise_std=0.01,
                random_stream=np.random.RandomState(4))
    n = 12
    acn = (np.random.RandomState(4).randn(n, 400, 2).astype(f32) * f32(0.01))
    d = _launch(ctx, "maze", pol.net, pol._bin_values, theta.cpu().numpy()[None], np.repeat([u.noise_idx for u in units], 2),
                np.tile([0.05, -0.05], 6).astype(f32), None, maze.initial_states(n), 400, pol.ob_mean.cpu().numpy(),
                pol.ob_std.cpu().numpy(), acn, stats=False)
    np.testing.assert_array_equal(res.returns.ravel(), d["ret"])
    np.testing.assert_array_equal(np.stack([b for u in res.bcs for b in u]), d["fin"][:, :2])


def _exp(name, ac_bins, **over):
    with open(os.path.join(CONFIGS, name)) as f:
        exp = json.load(f)
    exp["config"].update(snapshot_freq=0, **over)
    exp["policy"]["args"]["ac_bins"] = ac_bins
    return exp


@pytest.mark.parametrize("ac_bins", ["uniform:10", "custom:-1,-0.1,0,0.1,1"])
def test_drivers_complete_on_maze(noise, tmp_path, ac_bins):
    from es_distributed import es as ES
    from es_distributed import ga as GA
    from es_distributed import nses as NS
    from es_distributed import policies
    from es_distributed import rs as RS
    exp = _exp("hardmaze_es.json", ac_bins, episodes_per_batch=16)
    exp["maze_file"] = M.FIXTURE
    log = []
    ES.set_default_noise(noise)
    ES.run_master(None, None, exp, max_iterations=1, n_slots=8, noise=noise, seed=3,
                  on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 1 and (log[0]["lengths_n2"] == 400).all() and (log[0]["returns_n2"] < 0).all()
    for algo in ("ns", "nsr"):
        nlog = []
        exp = _exp("hardmaze_nses.json", ac_bins, episodes_per_batch=16)
        exp.update(algo_type=algo)
        exp["novelty_search"].update(population_size=2)
        NS.set_default_noise(noise)
        NS.run_master(None, str(tmp_path / algo), exp, max_iterations=2, n_slots=8, noise=noise, seed=2,
                      on_iteration=lambda it, st, ex: nlog.append(ex))
        assert len(nlog) == 2 and np.isfinite(nlog[-1]["novelty_n2"]).all()
    glog = []
    exp = _exp("hardmaze_es.json", ac_bins, episodes_per_batch=12)
    exp.update(population_size=4, num_elites=1)
    GA.set_default_noise(noise)
    GA.run_master(None, str(tmp_path / "ga"), exp, max_iterations=2, n_slots=8, noise=noise, seed=5,
                  on_iteration=lambda it, st, ex: glog.append(ex))
    assert len(glog) == 2 and all((ex["returns"] < 0).all() for ex in glog)
    rlog = []
    RS.set_default_noise(noise)
    RS.run_master(None, str(tmp_path / "rs"), _exp("hardmaze_es.json", ac_bins, episodes_per_batch=16),
                  max_iterations=1, n_slots=8, noise=noise, seed=3, on_iteration=lambda it, st, ex: rlog.append(ex))
    assert len(rlog) == 1 and rlog[0]["returns_n2"].shape == (16, 1)
    env = MazeEnv(2)
    pol = policies.MujocoPolicy(env.observation_space, env.action_space, seed=1,
                                **_exp("hardmaze_es.json", ac_bins)["policy"]["args"])
    rews, t, bc = pol.rollout(env, timestep_limit=400, random_stream=np.random.RandomState(0))
    assert rews.shape == (1,) and rews[0] < 0 and t == 400 and bc.shape == (2,)


class _RecordingPendulum(PendulumEnv):
    """PendulumEnv that keeps every action its host step was given."""

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.seen = []

    def step(self, slots, actions):
        self.seen.append(np.array(actions, dtype=f32).reshape(-1))
        return super().step(slots, actions)


def test_pendulum_drivers_act_with_bin_values(noise, tmp_path):
    from es_distributed import ga as GA
    from es_distributed import policies
    from es_distributed import rs as RS
    values = set(_uniform("pendulum", 5).ravel().tolist())
    exp = _exp("pendulum_es.json", "uniform:5", episodes_per_batch=8)
    exp["policy"]["args"]["ac_noise_std"] = 0.0
    exp.update(population_size=4, num_elites=1)
    env = _RecordingPendulum(8)
    GA.set_default_noise(noise)
    GA.run_master(None, str(tmp_path / "ga"), exp, max_iterations=1, n_slots=8, env=env, noise=noise, seed=5)
    env2 = _RecordingPendulum(8)
    RS.set_default_noise(noise)
    RS.run_master(None, str(tmp_path / "rs"), exp, max_iterations=1, n_slots=8, env=env2, noise=noise, seed=3)
    env3 = _RecordingPendulum(2)
    pol = policies.MujocoPolicy(env3.observation_space, env3.action_space, seed=1, **exp["policy"]["args"])
    rews, t, _ = pol.rollout(env3, timestep_limit=200)
    assert t == 200 and np.isfinite(rews).all()
    for e in (env, env2, env3):
        acts = np.concatenate(e.seen)
        assert len(acts) > 0 and set(np.unique(acts).tolist()) <= values
