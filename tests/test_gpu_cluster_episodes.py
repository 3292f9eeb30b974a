"""GPU tests of the thread-block-cluster episode kernel (dne_pendulum_cluster_episodes, dne_maze_cluster_episodes): one
member per cluster of 2, 4 or 8 CTAs, for nets too wide for one CTA (MujocoPolicy's hidden [256, 256]).

Referees:
* the single-CTA kernel (dne_pendulum_episodes / dne_maze_episodes) on every net both take: the split changes no
  operation, so returns, sign-returns, lengths, final states and observation sums must be bit-identical at every
  cluster size;
* for the wide nets, which only the cluster kernel takes: one launch of T steps equals T chained one-step launches bit
  for bit, reruns are bit-identical, and every cluster size that fits gives the automatic size's bits;
* for [256, 256]: Pendulum episodes against the per-tick RolloutRunner stepping the host PendulumEnv (test_gpu_pendulum's
  200-step tolerances), and the maze head against the float64 forward referee of test_gpu_dense_paths, read back through
  the first step's angular velocity and speed (as test_gpu_maze.py::test_head_against_float64_referee does).
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
from test_gpu_dense_paths import U, member, normalise, referee   # noqa: E402  (the float64 forward referee)
from test_gpu_maze import _inits as maze_inits, _mixed as maze_mixed   # noqa: E402
from test_gpu_pendulum import RETURN_RTOL_200, STATE_TOL_200, _init as pendulum_inits   # noqa: E402
from test_gpu_pendulum import _mixed as pendulum_mixed   # noqa: E402
from dne import _ffi as F                          # noqa: E402
from dne import nets                               # noqa: E402
from dne.engine import make_context                # noqa: E402
from dne.envs import MazeEnv, PendulumEnv, make_env   # noqa: E402
from dne.noise import SharedNoiseTable             # noqa: E402
from dne.rollout import EpisodeKernelRunner, RolloutRunner, Unit, make_runner   # noqa: E402

NOISE_COUNT = 2_000_000
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIGS = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations")
ULP = lambda v: float(np.spacing(np.float32(abs(v))))      # noqa: E731
# the 'policy' block of the reference's humanoid.json / humanoid_nses.json / humanoid_nsres.json
HUMANOID_POLICY_ARGS = {"ac_bins": "continuous:", "ac_noise_std": 0.01, "connection_type": "ff",
                        "hidden_dims": [256, 256], "nonlin_type": "tanh"}
TASKS = {"pendulum": dict(ob=3, out=1, state=2, T=200), "maze": dict(ob=11, out=2, state=7, T=400)}


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def noise(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device="cuda:0")


@pytest.fixture(scope="module")
def ctx(noise):
    return make_context(0, noise)


def _net(task, hidden, act=F.ACT_TANH, n_out=None, ob_dim=None):
    ob_dim = TASKS[task]["ob"] if ob_dim is None else ob_dim
    n_out = TASKS[task]["out"] if n_out is None else n_out
    dims = [ob_dim] + list(hidden)
    layers = [nets._dense(dims[i], dims[i + 1], act=act) for i in range(len(hidden))]
    layers.append(nets._dense(dims[-1], n_out, act=F.ACT_NONE))
    return nets._finish(nets.NetSpec(task, layers, F.OB_VECTOR, ob_dim))


def _cuda(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(DEV)


def _launch(ctx, task, net, theta, idx, scale, rows, init, T, ob_mean=None, ob_std=None, ac_noise=None, stats=True,
            cluster=None, pad=0, n=None):
    """dne_<task>_episodes (cluster None) or dne_<task>_cluster_episodes(cluster) for the first n (default all) members
    on numpy inputs -> dict of numpy outputs, 'rc' and, with pad > 0, 'tail': the `pad` output rows past n, which must
    keep their sentinels."""
    n = len(idx) if n is None else n
    k = n + pad if n + pad > 0 else 1
    sd, ob = TASKS[task]["state"], TASKS[task]["ob"]
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
    a = [C.byref(net.desc), F.ptr(args[0]), F.ptr(args[1]), F.ptr(args[2]), F.ptr(args[3]), n, F.ptr(args[4]), int(T),
         F.ptr(args[5]), F.ptr(args[6]), F.ptr(args[7]), F.ptr(d["ret"]), F.ptr(d["sret"]), F.ptr(d["len"]),
         F.ptr(d["fin"]), F.ptr(d.get("s")), F.ptr(d.get("q"))]
    if task == "maze":
        a.insert(0, C.byref(MazeEnv(1).desc))
    L = F.lib()
    if cluster is None:
        rc = getattr(L, f"dne_{task}_episodes")(ctx.handle, *a, F.stream_ptr())
    else:
        rc = getattr(L, f"dne_{task}_cluster_episodes")(ctx.handle, *a, int(cluster), F.stream_ptr())
    torch.cuda.synchronize()
    out = {key: v.cpu().numpy()[:n] for key, v in d.items()}
    if pad:
        out["tail"] = {key: v.cpu().numpy()[n:] for key, v in d.items()}
    out["rc"] = rc
    return out


def _population(task, net, rs, n=512):
    """Mixed members (± pairs, unpaired scales, GA rows through theta_idx, noiseless), their theta rows and initial states
    (maze: half from random open positions)."""
    P = net.num_params
    theta = (rs.randn(4, P) * (0.3 if task == "pendulum" else 0.1)).astype(np.float32)
    if task == "pendulum":
        idx, scale, rows = pendulum_mixed(rs, P, n=n)
        init = pendulum_inits(rs, n)
    else:
        idx, scale, rows = maze_mixed(rs, P, n=n)
        init = maze_inits(rs, n)
    return theta, idx, scale, rows, init


def _inputs(task, rs, n, T, stats, noisy, scale):
    ob = TASKS[task]["ob"]
    mean, std = ((rs.randn(ob) * 0.1).astype(np.float32), rs.uniform(0.3, 1.0, ob).astype(np.float32)) if stats else \
        (None, None)
    acn = None
    if noisy:
        acn = (rs.randn(n, T, TASKS[task]["out"]) * 0.2).astype(np.float32)
        acn[scale == 0] = 0.0
    return mean, std, acn


def _same(a, b, keys):
    for key in keys:
        assert a[key].tobytes() == b[key].tobytes(), key


def _keys(stats):
    return ("ret", "sret", "len", "fin") + (("s", "q") if stats else ())


def _sizes(task, net):
    """The cluster sizes whose slices fit a CTA for `net` (the automatic choice among them)."""
    out = []
    for c in (2, 4, 8):
        g = (C.c_int * 4)()
        if getattr(F.lib(), f"dne_{task}_cluster_geometry")(C.byref(net.desc), c, g) == 0:
            out.append(c)
    return out


# ---- bit identity against the single-CTA kernel ------------------------------------------------------------------------
@pytest.mark.parametrize("task,hidden", [("pendulum", (64, 64)), ("pendulum", (200, 200)), ("pendulum", (512,)),
                                         ("pendulum", (400, 50)), ("maze", (64, 64)), ("maze", (1024,))])
def test_bit_identical_to_single_cta_kernel(ctx, task, hidden):
    net = _net(task, hidden)
    L = F.lib()
    assert getattr(L, f"dne_{task}_net_supported")(C.byref(net.desc)) == 0
    assert getattr(L, f"dne_{task}_cluster_net_supported")(C.byref(net.desc)) == 0
    T = TASKS[task]["T"]
    rs = np.random.RandomState(sum(hidden) + len(task))
    theta, idx, scale, rows, init = _population(task, net, rs)
    n = len(idx)
    for stats, noisy in ((True, True), (False, False)):
        mean, std, acn = _inputs(task, rs, n, T, stats, noisy, scale)
        ref = _launch(ctx, task, net, theta, idx, scale, rows, init, T, mean, std, acn, stats=stats)
        assert ref["rc"] == 0 and (ref["len"] == T).all()
        for c in (0, 2, 4, 8):
            got = _launch(ctx, task, net, theta, idx, scale, rows, init, T, mean, std, acn, stats=stats, cluster=c)
            assert got["rc"] == 0, (c, L.dne_last_error().decode())
            _same(got, ref, _keys(stats))
        if task == "maze":
            moved = np.hypot(ref["fin"][:, 0] - init[:, 0], ref["fin"][:, 1] - init[:, 1])
            assert (moved > 20).sum() > n // 4         # the episodes go somewhere: the comparison is not vacuous
        else:
            assert np.unique(ref["ret"]).size > n // 2


# ---- nets only the cluster kernel takes ---------------------------------------------------------------------------------
WIDE = [("maze", (256, 256)), ("pendulum", (256, 256)), ("maze", (512, 512))]


@pytest.mark.parametrize("task,hidden", WIDE)
def test_wide_one_launch_equals_chained_launches_and_every_size(ctx, task, hidden):
    net = _net(task, hidden)
    L = F.lib()
    assert getattr(L, f"dne_{task}_net_supported")(C.byref(net.desc)) == -4
    assert getattr(L, f"dne_{task}_cluster_net_supported")(C.byref(net.desc)) == 0
    T = TASKS[task]["T"]
    rs = np.random.RandomState(7 + hidden[0])
    theta, idx, scale, rows, init = _population(task, net, rs, n=256)
    n = len(idx)
    mean, std, acn = _inputs(task, rs, n, T, True, True, scale)
    full = _launch(ctx, task, net, theta, idx, scale, rows, init, T, mean, std, acn, cluster=0)
    assert full["rc"] == 0, L.dne_last_error().decode()
    assert (full["len"] == T).all() and np.isfinite(full["ret"]).all()
    st = init.copy()
    ret, sret = np.zeros(n), np.zeros(n)
    s, q = np.zeros((n, TASKS[task]["ob"])), np.zeros((n, TASKS[task]["ob"]))
    for t in range(T):
        one = _launch(ctx, task, net, theta, idx, scale, rows, st, 1, mean, std, acn[:, t:t + 1], cluster=0)
        assert one["rc"] == 0
        st = one["fin"]
        ret += one["ret"].astype(np.float64)
        sret += one["sret"].astype(np.float64)
        s += one["s"]
        q += one["q"]
    assert full["fin"].tobytes() == st.tobytes()
    assert full["ret"].tobytes() == ret.astype(np.float32).tobytes()
    assert full["sret"].tobytes() == sret.astype(np.float32).tobytes()
    assert full["s"].tobytes() == s.tobytes() and full["q"].tobytes() == q.tobytes()
    again = _launch(ctx, task, net, theta, idx, scale, rows, init, T, mean, std, acn, cluster=0)
    _same(again, full, _keys(True))                                    # bit-identical reruns
    sizes = _sizes(task, net)
    assert sizes and (hidden != (512, 512) or sizes == [8])
    auto = F.cluster_geometry(task, net.desc)
    print(f"{task} {hidden}: sizes that fit {sizes}, automatic {auto}")
    assert auto["cluster"] in sizes and auto["resident_members"] > 0
    for c in sizes:
        got = _launch(ctx, task, net, theta, idx, scale, rows, init, T, mean, std, acn, cluster=c)
        assert got["rc"] == 0
        _same(got, full, _keys(True))
    for c in {2, 4, 8} - set(sizes):                                   # a forced size too small for the net
        assert _launch(ctx, task, net, theta, idx[:4], scale[:4], rows[:4], init[:4], T, cluster=c)["rc"] == -4


# ---- independent referees for [256, 256] --------------------------------------------------------------------------------
def test_pendulum_256_against_per_tick_engine(ctx):
    """RolloutRunner + host PendulumEnv (dne_perturb_forward_mlp per tick) plays the same members from the same states as
    an EpisodeKernelRunner built directly, which runs [256, 256] on the cluster kernel."""
    net = _net("pendulum", (256, 256))
    rs = np.random.RandomState(5)
    theta = torch.from_numpy((rs.randn(net.num_params) * 0.1).astype(np.float32)).to(DEV)
    units = [Unit(int(rs.randint(0, NOISE_COUNT - net.num_params)), (0.02, -0.02)) for _ in range(63)] + \
            [Unit(0, (0.0, 0.0), noiseless=True)]
    mean, std = torch.tensor([0.1, 0.0, 0.2], device=DEV), torch.tensor([0.8, 0.8, 2.0], device=DEV)
    n = 2 * len(units)
    out = {}
    for name, runner in (("kernel", EpisodeKernelRunner(ctx, net, PendulumEnv(n, seed=9), group=2)),
                         ("per-tick", RolloutRunner(ctx, net, PendulumEnv(n, seed=9), n, group=2, pipeline=2))):
        out[name] = runner.run(theta, units, None, ob_mean=mean, ob_std=std, collect_bc="final")
    k, p = out["kernel"], out["per-tick"]
    np.testing.assert_array_equal(k.lengths, p.lengths)
    assert (k.lengths == 200).all()
    fk, fp = np.array([b for u in k.bcs for b in u]), np.array([b for u in p.bcs for b in u])
    d_state = float(np.abs(fk - fp).max())
    d_ret = float((np.abs(k.returns - p.returns) / np.maximum(np.abs(p.returns), 1.0)).max())
    print(f"[256, 256] per-tick referee: max |state| difference {d_state:.3g}, relative return {d_ret:.3g}")
    assert d_state <= STATE_TOL_200 and d_ret <= RETURN_RTOL_200
    np.testing.assert_array_equal(k.signreturns, p.signreturns)
    assert np.unique(k.returns).size > n // 2


def test_maze_256_head_against_float64_referee(ctx, host_noise):
    net = _net("maze", (256, 256))
    P = net.num_params
    rs = np.random.RandomState(23)
    theta = (rs.randn(2, P) * 0.01).astype(np.float32)
    idx, scale, rows = maze_mixed(rs, P, n=128, n_rows=2)
    scale *= np.float32(0.1)
    n = len(idx)
    init = maze_inits(rs, n)
    init[:, 2:5] = 0.0                                             # heading 0, at rest
    mean, std = (rs.randn(11) * 0.1).astype(np.float32), rs.uniform(0.3, 1.0, 11).astype(np.float32)
    got = _launch(ctx, "maze", net, theta, idx, scale, rows, init, 1, mean, std, cluster=0)
    assert got["rc"] == 0
    bad = checked = 0
    maze = M.load_maze()
    for m in range(n):
        o = M.observation(maze, init[m, 0], init[m, 1], 0.0)
        np.testing.assert_array_equal(got["s"][m], o.astype(np.float64))       # the exact observation at heading 0
        w, wm = member(theta, int(rows[m]), host_noise, int(idx[m]), scale[m], P)
        y, e = referee(net, w, wm, normalise(o[None, :], mean, std)[0])
        # new ang_vel = fl(fl(fl(a + 0.5) - 0.5) * 6) while |6a| < 0.2: a is recovered within 2^-25 + 6 ulps of the result
        for j, col in ((0, 4), (1, 3)):
            v = float(got["fin"][m, col])
            if abs(v) >= 0.2:
                continue
            checked += 1
            bnd = e[j] + 2.0 ** -25 + 6 * ULP(v) / 6 + 2 * U * abs(y[j])
            bad += int(abs(v / 6.0 - y[j]) > bnd)
    assert bad == 0 and checked > n // 2


# ---- contract -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("task", ["pendulum", "maze"])
def test_contract(ctx, task):
    L = F.lib()
    net = _net(task, (256, 256))
    probe = getattr(L, f"dne_{task}_cluster_net_supported")
    entry = f"dne_{task}_cluster_episodes"
    assert probe(C.byref(net.desc)) == 0
    assert getattr(L, f"dne_{task}_net_supported")(C.byref(net.desc)) == -4    # the single-CTA probe is unchanged
    ob, out = TASKS[task]["ob"], TASKS[task]["out"]
    unsup = {"too wide at 8": _net(task, (2048, 2048)), "ob_dim": _net(task, (64, 64), ob_dim=ob + 1),
             "n_out": _net(task, (64, 64), n_out=out + 1), "conv": nets.make_net("Model", num_actions=2),
             "hidden act": _net(task, (256, 256), act=F.ACT_NONE),
             "bn": nets._finish(nets.NetSpec("bn", [nets._dense(ob, 8, act=F.ACT_TANH, bn=F.BN_TF),
                                                    nets._dense(8, out, act=F.ACT_NONE)], F.OB_VECTOR, ob)),
             "tanh head": nets._finish(nets.NetSpec("th", [nets._dense(ob, 8, act=F.ACT_TANH),
                                                           nets._dense(8, out, act=F.ACT_TANH)], F.OB_VECTOR, ob))}
    P = net.num_params
    rs = np.random.RandomState(3)
    theta = np.zeros((1, P), np.float32)
    init = np.zeros((4, TASKS[task]["state"]))
    idx, scale = np.zeros(4, np.int64), np.zeros(4, np.float32)
    for what, bad in unsup.items():
        assert probe(C.byref(bad.desc)) == -4, what
        assert L.dne_last_error().decode().startswith(f"dne_{task}_cluster_net_supported"), what
        r = _launch(ctx, task, bad, np.zeros((1, max(bad.num_params, 1)), np.float32), idx, scale, None, init, 10,
                    cluster=0)
        assert r["rc"] == -4, what
        assert L.dne_last_error().decode().startswith(entry), what
    for c in (1, 3, 16, -1):
        assert _launch(ctx, task, net, theta, idx, scale, None, init, 10, cluster=c)["rc"] == -1, c
        assert "cluster" in L.dne_last_error().decode()
    g = (C.c_int * 4)()
    assert getattr(L, f"dne_{task}_cluster_geometry")(C.byref(net.desc), 3, g) == -1
    for T in (0, TASKS[task]["T"] + 1):
        assert _launch(ctx, task, net, theta, idx, scale, None, init, T, cluster=0)["rc"] == -1, T
    # n = 0 launches nothing; the rows past n keep their sentinels
    L.dne_launch_count(1)
    r0 = _launch(ctx, task, net, theta, idx, scale, None, init, 10, cluster=0, pad=3, n=0)
    assert r0["rc"] == 0 and L.dne_launch_count(0) == 0
    assert (r0["tail"]["ret"] == -1).all() and (r0["tail"]["len"] == -1).all() and (r0["tail"]["fin"] == -7).all()
    if task == "maze":
        init = MazeEnv(1).initial_states(4)
    r = _launch(ctx, task, net, (rs.randn(1, P) * 0.1).astype(np.float32), idx, scale, None, init, 10, cluster=0, pad=5)
    assert r["rc"] == 0 and (r["len"] == 10).all()
    for key, v in r["tail"].items():
        assert (v == (-1 if key in ("ret", "sret", "len") else -7)).all(), key
    geo = F.cluster_geometry(task, net.desc)
    print(f"{task} [256, 256] automatic geometry: {geo}")
    assert geo["threads"] % 32 == 0 and 32 <= geo["threads"] <= 256 and geo["smem_bytes"] <= 227 * 1024


# ---- runner and drivers -------------------------------------------------------------------------------------------------
def test_maze_runner_on_256_matches_direct_cluster_launch(ctx):
    net = _net("maze", (256, 256))
    P = net.num_params
    rs = np.random.RandomState(12)
    theta = torch.from_numpy((rs.randn(3, P) * 0.1).astype(np.float32)).to(DEV)
    units = [Unit(int(rs.randint(0, NOISE_COUNT - P)), (0.05, -0.05), theta_idx=i % 3) for i in range(40)] + \
            [Unit(0, (0.0, 0.0), theta_idx=1, noiseless=True) for _ in range(3)]
    mean = torch.from_numpy(rs.randn(11).astype(np.float32) * 0.1)
    std = torch.from_numpy(rs.uniform(0.5, 1, 11).astype(np.float32))
    env = make_env("maze", 4)
    r = make_runner(ctx, net, env, n_slots=4, group=2)
    assert isinstance(r, EpisodeKernelRunner)
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
    d = _launch(ctx, "maze", net, theta.cpu().numpy(), idx, scale, rows, init, 400, mean.numpy(), std.numpy(), acn,
                cluster=0)
    assert d["rc"] == 0
    np.testing.assert_array_equal(res.returns.ravel(), d["ret"])
    np.testing.assert_array_equal(res.signreturns.ravel(), d["sret"])
    np.testing.assert_array_equal(res.lengths.ravel(), d["len"])
    bcs = np.stack([b for u in res.bcs for b in u])
    np.testing.assert_array_equal(bcs, d["fin"][:, :2])
    s = sum(d["s"][m] for m in np.nonzero(save)[0])
    np.testing.assert_array_equal(res.ob_sum, s)
    assert res.ob_count == 400 * int(save.sum()) and save.sum() > 0


def _exp(name, **over):
    with open(os.path.join(CONFIGS, name)) as f:
        exp = json.load(f)
    exp["config"].update(snapshot_freq=0, **over)
    exp["policy"]["args"] = dict(HUMANOID_POLICY_ARGS)
    return exp


def test_drivers_complete_on_maze_with_humanoid_policy(noise, tmp_path):
    from es_distributed import es as ES
    from es_distributed import ga as GA
    from es_distributed import nses as NS
    from es_distributed import policies
    from es_distributed import rs as RS
    ES.set_default_noise(noise)
    log = []
    ES.run_master(None, None, _exp("hardmaze_es.json", episodes_per_batch=16), max_iterations=2, n_slots=8,
                  noise=noise, seed=3, on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 2 and all(ex["returns_n2"].shape == (8, 2) and (ex["lengths_n2"] == 400).all() for ex in log)
    assert all((ex["returns_n2"] < 0).all() for ex in log)
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
    RS.run_master(None, str(tmp_path / "rs"), _exp("hardmaze_es.json", episodes_per_batch=16), max_iterations=2,
                  n_slots=8, noise=noise, seed=3, on_iteration=lambda it, st, ex: rlog.append(ex))
    assert len(rlog) == 2 and rlog[0]["returns_n2"].shape == (16, 1)
    env = MazeEnv(2)
    pol = policies.MujocoPolicy(env.observation_space, env.action_space, seed=1, **HUMANOID_POLICY_ARGS)
    assert pol.net.num_params == 69378
    rews, t, bc = pol.rollout(env, timestep_limit=400, random_stream=np.random.RandomState(0))
    assert rews.shape == (1,) and rews[0] < 0 and t == 400 and bc.shape == (2,)
