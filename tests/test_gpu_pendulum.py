"""GPU tests of the fused Pendulum-v1 episode kernel (dne_pendulum_episodes), its runner and the drivers running on it.

Referees:
* the kernel itself: one launch of T steps must equal T chained one-step launches bit for bit (final states, returns and
  sign-returns summed on the host in float64, per-member observation sums);
* one step against a float64 referee of the forward (tests/test_gpu_dense_paths.py: per-output bound from a magnitude
  forward) followed by the float64 step of tests/pendulum_oracle.py, with the head's bound carried through the step's
  Lipschitz constants (d thdot / d u = 0.15, d reward / d u = 0.002 u);
* episodes of 2..200 steps against tests/pendulum_oracle.py (oracle.forward in float32), and the engine's per-tick
  RolloutRunner stepping the host PendulumEnv: these sum in other orders and use other sin / cos / tanh, so they agree
  within a tolerance that grows with the horizon (HORIZON_TOL, measured maxima in DESIGN.md 4).
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
import pendulum_oracle as PO                       # noqa: E402
from test_gpu_dense_paths import U, member, normalise, referee   # noqa: E402  (the float64 forward referee)
from dne import _ffi as F                          # noqa: E402
from dne import nets                               # noqa: E402
from dne.engine import make_context                # noqa: E402
from dne.envs import PendulumEnv                   # noqa: E402
from dne.noise import SharedNoiseTable             # noqa: E402
from dne.rollout import EpisodeKernelRunner, RolloutRunner, Unit, make_runner   # noqa: E402

NOISE_COUNT = 2_000_000
DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations", "pendulum_es.json")
# |state| and relative |return| differences allowed against the float32 oracle and the per-tick engine, by horizon: both
# start from float32 forwards that differ from the kernel's in the last bits (other summation orders, numpy's tanh / sin /
# cos), and the pendulum integrates those differences.  Measured on an H100 (DESIGN.md 4): 2.6e-7 at 2 steps, 4.0e-7 at
# 10, 1.7e-5 at 50, 4.2e-5 (states) and 5.4e-7 (returns) at 200; the tolerances leave a factor of 20 or more.  An
# off-by-one noise slice moves a state by ~1e-2 in one step.
HORIZON_TOL = {2: 1e-5, 10: 1e-5, 50: 1e-3}
STATE_TOL_200, RETURN_RTOL_200 = 1e-3, 2e-5
# generations within which pendulum_es.json (seed 0) must reach a mean noiseless return >= -300 over 100 episodes
LEARN_MAX_GENERATIONS = 120          # reached after 61 on an H100 (about twice that)
LEARN_TARGET = -300.0


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def noise(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device="cuda:0")


@pytest.fixture(scope="module")
def ctx(noise):
    return make_context(0, noise)


def _net(hidden=(64, 64), act=F.ACT_TANH, n_out=1, ob_dim=3):
    dims = [ob_dim] + list(hidden)
    layers = [nets._dense(dims[i], dims[i + 1], act=act) for i in range(len(hidden))]
    layers.append(nets._dense(dims[-1], n_out, act=F.ACT_NONE))
    return nets._finish(nets.NetSpec("pendulum", layers, F.OB_VECTOR, ob_dim))


def _cuda(a, dt):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(DEV)


def _launch(ctx, net, theta, idx, scale, rows, init, T, ob_mean=None, ob_std=None, ac_noise=None, stats=True):
    """dne_pendulum_episodes on numpy inputs -> dict of numpy outputs (and 'rc')."""
    n = len(idx)
    k = max(n, 1)
    d = dict(ret=torch.full((k,), -1.0, dtype=torch.float32, device=DEV),
             sret=torch.full((k,), -1.0, dtype=torch.float32, device=DEV),
             len=torch.full((k,), -1, dtype=torch.int32, device=DEV),
             fin=torch.full((k, 2), -7.0, dtype=torch.float64, device=DEV))
    if stats:
        d["s"] = torch.full((k, 3), -7.0, dtype=torch.float64, device=DEV)
        d["q"] = torch.full((k, 3), -7.0, dtype=torch.float64, device=DEV)
    args = [_cuda(theta, np.float32), _cuda(idx, np.int64), _cuda(scale, np.float32),
            None if rows is None else _cuda(rows, np.int32), _cuda(init, np.float64),
            None if ob_mean is None else _cuda(ob_mean, np.float32), None if ob_std is None else _cuda(ob_std, np.float32),
            None if ac_noise is None else _cuda(ac_noise, np.float32)]
    rc = F.lib().dne_pendulum_episodes(
        ctx.handle, C.byref(net.desc), F.ptr(args[0]), F.ptr(args[1]), F.ptr(args[2]), F.ptr(args[3]), n, F.ptr(args[4]),
        int(T), F.ptr(args[5]), F.ptr(args[6]), F.ptr(args[7]), F.ptr(d["ret"]), F.ptr(d["sret"]), F.ptr(d["len"]),
        F.ptr(d["fin"]), F.ptr(d.get("s")), F.ptr(d.get("q")), F.stream_ptr())
    torch.cuda.synchronize()
    out = {key: v.cpu().numpy()[:n] for key, v in d.items()}
    out["rc"] = rc
    return out


def _theta_rows(rs, P, n_rows, s=0.3):
    return (rs.randn(n_rows, P) * s).astype(np.float32)


def _mixed(rs, P, n=512, n_rows=4):
    """± pairs on row 0, unpaired scales, GA members on rows of a [n_rows, P] matrix, noiseless (scale 0) members."""
    n_pair, n_un, n_zero = n // 4, n // 8, n // 8
    n_ga = n - 2 * n_pair - n_un - n_zero
    hi = NOISE_COUNT - P + 1
    idx = np.concatenate([np.repeat(rs.randint(0, hi, n_pair), 2), rs.randint(0, hi, n_un), rs.randint(0, hi, n_zero),
                          rs.randint(0, hi, n_ga)]).astype(np.int64)
    scale = np.concatenate([np.tile([0.05, -0.05], n_pair), rs.choice([0.02, 0.1, -0.3], n_un), np.zeros(n_zero),
                            rs.choice([0.02, -0.05], n_ga)]).astype(np.float32)
    rows = np.concatenate([np.zeros(2 * n_pair + n_un + n_zero), rs.randint(0, n_rows, n_ga)]).astype(np.int32)
    return idx, scale, rows


def _init(rs, n):
    return np.stack([rs.uniform(-np.pi, np.pi, n), rs.uniform(-1, 1, n)], axis=1)


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("stats,noisy,hidden", [(True, True, (64, 64)), (False, False, (64, 64)), (True, False, (64, 64)),
                                               (True, True, (400, 50))])
def test_one_launch_equals_chained_one_step_launches(ctx, stats, noisy, hidden):
    net = _net(hidden)
    P, T = net.num_params, 200
    rs = np.random.RandomState(1 + 2 * stats + noisy)
    theta = _theta_rows(rs, P, 4)
    idx, scale, rows = _mixed(rs, P)
    n = len(idx)
    init = _init(rs, n)
    init[::5, 1] = rs.choice([-8.0, 8.0], len(init[::5]))
    mean, std = (np.array([0.1, -0.2, 0.5], np.float32), np.array([0.7, 0.8, 2.5], np.float32)) if stats else (None, None)
    acn = (rs.randn(n, T, 1) * 0.3).astype(np.float32) if noisy else None
    if noisy:
        acn[scale == 0] = 0.0                                     # noiseless members, as the runner builds them
    full = _launch(ctx, net, theta, idx, scale, rows, init, T, mean, std, acn)
    assert full["rc"] == 0 and (full["len"] == T).all()
    st = init.copy()
    ret, sret = np.zeros(n), np.zeros(n)
    s, q = np.zeros((n, 3)), np.zeros((n, 3))
    for t in range(T):
        one = _launch(ctx, net, theta, idx, scale, rows, st, 1, mean, std, None if acn is None else acn[:, t:t + 1])
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
    again = _launch(ctx, net, theta, idx, scale, rows, init, T, mean, std, acn)
    for key in ("ret", "sret", "fin", "s", "q"):
        assert again[key].tobytes() == full[key].tobytes()      # bit-identical reruns


def _robust_obs(th):
    """cos / sin of th are not within 16 float64 ulps of a float32 rounding boundary (CUDA's and libm's double sin / cos
    may differ by an ulp; away from a boundary both round to the same float32 observation)."""
    for v in (math.cos(th), math.sin(th)):
        f = np.float32(v)
        for nb in (np.nextafter(f, np.float32(-np.inf)), np.nextafter(f, np.float32(np.inf))):
            if abs(v - (float(f) + float(nb)) / 2) <= 16 * np.spacing(abs(v)):
                return False
    return True


def _one_step_referee(net, theta, host_noise, idx, s, row, state, mean, std, acn, shift=0):
    """(th, thdot, reward) of one step in float64 and their bounds."""
    P = net.num_params
    i = idx + shift if idx + shift + P <= NOISE_COUNT else idx - shift
    w, wm = member(theta, row, host_noise, i, s, P)
    o = PO.observation(*state)
    x0 = normalise(o[None, :], mean, std)[0]
    y, e = referee(net, w, wm, x0)
    a = y[0] + float(acn)
    da = e[0] + 2 * U * abs(a) + 1e-30
    u = min(max(a, -2.0), 2.0)
    th, thdot = state
    an = PO.angle_normalize(th)
    r = -(an * an + 0.1 * thdot * thdot + 0.001 * u * u)
    nthdot = min(max(thdot + (15.0 * math.sin(th) + 3.0 * u) * 0.05, -8.0), 8.0)
    nth = th + nthdot * 0.05
    d_thdot = 0.15 * da + 1e-13 * (1 + abs(thdot))
    d_th = 0.05 * d_thdot + 1e-13 * (1 + abs(th))
    d_r = 0.001 * (4 * da + da * da) + 8 * U * abs(r) + 1e-12 * (1 + abs(r))
    return np.array([nth, nthdot, r]), np.array([d_th, d_thdot, d_r]), o


@pytest.mark.parametrize("hidden", [(64, 64), (128, 128), (512,), (400, 50)])
def test_one_step_against_float64_referee(ctx, host_noise, hidden):
    net = _net(hidden)
    P = net.num_params
    rs = np.random.RandomState(17)
    theta = _theta_rows(rs, P, 3, s=0.1)
    idx, scale, rows = _mixed(rs, P, n=256, n_rows=3)
    n = len(idx)
    init = _init(rs, n)
    init[0:32, 0] = rs.uniform(-60, 60, 32)                          # large |th|
    init[32:64, 1] = rs.choice([-8.0, 8.0, 7.99, -7.99], 32)         # speeds at the clip
    for m in range(n):
        while not _robust_obs(init[m, 0]):
            init[m, 0] = np.nextafter(init[m, 0] + 1e-9, np.inf)
    acn = (rs.randn(n, 1, 1) * 0.5).astype(np.float32)
    acn[64:96] = rs.choice([-6.0, 6.0], (32, 1, 1))                  # saturated torque both ways
    mean, std = np.array([0.3, -0.1, 1.5], np.float32), np.array([0.6, 0.9, 3.0], np.float32)
    got = _launch(ctx, net, theta, idx, scale, rows, init, 1, mean, std, acn)
    assert got["rc"] == 0
    out = np.stack([got["fin"][:, 0], got["fin"][:, 1], got["ret"].astype(np.float64)], axis=1)
    bad, worst, shifted_bad = 0, 0.0, 0
    for m in range(n):
        ref, bnd, o = _one_step_referee(net, theta, host_noise, int(idx[m]), scale[m], int(rows[m]), init[m], mean, std,
                                        acn[m, 0, 0])
        err = np.abs(out[m] - ref)
        bad += int((err > bnd).sum())
        worst = max(worst, float((err / bnd).max()))
        np.testing.assert_array_equal(got["s"][m], o.astype(np.float64))
        np.testing.assert_array_equal(got["q"][m], np.square(o.astype(np.float64)))
        assert got["sret"][m] == np.sign(got["ret"][m])
        if scale[m] != 0:
            ref1, _, _ = _one_step_referee(net, theta, host_noise, int(idx[m]), scale[m], int(rows[m]), init[m], mean, std,
                                           acn[m, 0, 0], shift=1)
            shifted_bad += int((np.abs(out[m] - ref1) > bnd).any())
    print(f"one step: worst error / bound {worst:.3g}; off-by-one referee rejected on {shifted_bad} members")
    assert bad == 0, f"{bad} outputs outside the bound (worst error / bound {worst:.3g})"
    assert shifted_bad > n // 4, "the bound does not reject a referee with the noise index off by one"


def _oracle_episodes(net_o, theta, host_noise, idx, scale, rows, init, T, mean, std, acn=None):
    eps = []
    for m in range(len(idx)):
        w = (theta[rows[m]] + np.float32(scale[m]) * host_noise[idx[m]:idx[m] + theta.shape[1]]).astype(np.float32)
        eps.append(PO.pendulum_episode(net_o, w, init[m], T, mean, std, None if acn is None else acn[m, :, 0]))
    return eps


@pytest.mark.parametrize("T", [2, 10, 50, 200])
def test_horizons_against_oracle(ctx, host_noise, T):
    net, net_o = _net(), PO.policy_net((64, 64))
    assert net.num_params == net_o.num_params
    rs = np.random.RandomState(40 + T)
    theta = _theta_rows(rs, net.num_params, 2)
    n = 128 if T < 200 else 64
    idx, scale, rows = _mixed(rs, net.num_params, n=n, n_rows=2)
    init = _init(rs, n)
    mean, std = np.array([0.0, 0.1, -0.3], np.float32), np.array([0.7, 0.7, 2.0], np.float32)
    acn = (rs.randn(n, T, 1) * 0.01).astype(np.float32)
    got = _launch(ctx, net, theta, idx, scale, rows, init, T, mean, std, acn)
    assert got["rc"] == 0
    eps = _oracle_episodes(net_o, theta, host_noise, idx, scale, rows, init, T, mean, std, acn)
    fin = np.array([[e.th, e.thdot] for e in eps])
    ret = np.array([e.ret for e in eps], np.float64)
    d_state = float(np.abs(got["fin"] - fin).max())
    d_ret = float((np.abs(got["ret"] - ret) / np.maximum(np.abs(ret), 1.0)).max())
    print(f"T={T}: max |state - oracle| {d_state:.3g}, max relative return difference {d_ret:.3g}")
    if T in HORIZON_TOL:
        assert d_state <= HORIZON_TOL[T]
        assert d_ret <= HORIZON_TOL[T]
    else:
        assert d_state <= STATE_TOL_200 and d_ret <= RETURN_RTOL_200
    np.testing.assert_allclose(got["s"], np.stack([e.ob_sum for e in eps]), rtol=0, atol=50 * HORIZON_TOL.get(T, 1e-2) * T)


def test_per_tick_engine_referee(ctx):
    """RolloutRunner + host PendulumEnv (dne_perturb_forward_mlp per tick) plays the same members from the same states."""
    net = _net()
    rs = np.random.RandomState(5)
    theta = torch.from_numpy(_theta_rows(rs, net.num_params, 1)[0]).to(DEV)
    units = [Unit(int(rs.randint(0, NOISE_COUNT - net.num_params)), (0.05, -0.05)) for _ in range(63)] + \
            [Unit(0, (0.0, 0.0), noiseless=True)]
    mean, std = torch.tensor([0.1, 0.0, 0.2], device=DEV), torch.tensor([0.8, 0.8, 2.0], device=DEV)
    n = 2 * len(units)
    out = {}
    for name, runner in (("kernel", EpisodeKernelRunner(ctx, net, PendulumEnv(n, seed=9), group=2)),
                         ("per-tick", RolloutRunner(ctx, net, PendulumEnv(n, seed=9), n, group=2, pipeline=2))):
        out[name] = runner.run(theta, units, None, ob_mean=mean, ob_std=std, collect_bc="final")
    k, p = out["kernel"], out["per-tick"]
    np.testing.assert_array_equal(k.lengths, p.lengths)
    fk, fp = np.array([b for u in k.bcs for b in u]), np.array([b for u in p.bcs for b in u])
    d_state = float(np.abs(fk - fp).max())
    d_ret = float((np.abs(k.returns - p.returns) / np.maximum(np.abs(p.returns), 1.0)).max())
    print(f"per-tick referee: max |state| difference {d_state:.3g}, relative return {d_ret:.3g}")
    assert d_state <= STATE_TOL_200 and d_ret <= RETURN_RTOL_200
    np.testing.assert_array_equal(k.signreturns, p.signreturns)


def test_contract(ctx):
    net = _net()
    L = F.lib()
    assert L.dne_pendulum_net_supported(C.byref(_net((64, 64)).desc)) == 0
    assert L.dne_pendulum_net_supported(C.byref(_net((200, 200)).desc)) == 0
    for wide in ((257,), (512,), (1024,), (400, 50)):       # wider than a group's 256 threads: each loops over outputs
        assert L.dne_pendulum_net_supported(C.byref(_net(wide).desc)) == 0, wide
    assert L.dne_pendulum_net_supported(C.byref(_net((256, 256)).desc)) == -4
    assert L.dne_last_error().decode().startswith("dne_pendulum_net_supported")
    assert "shared memory" in L.dne_last_error().decode()
    unsup = {"ob_dim": _net(ob_dim=4), "n_out": _net(n_out=2), "conv": nets.make_net("Model", num_actions=2),
             "hidden act": _net(act=F.ACT_NONE), "wide": _net((256, 256)),
             "bn": nets._finish(nets.NetSpec("bn", [nets._dense(3, 8, act=F.ACT_TANH, bn=F.BN_TF),
                                                    nets._dense(8, 1, act=F.ACT_NONE)], F.OB_VECTOR, 3)),
             "tanh head": nets._finish(nets.NetSpec("th", [nets._dense(3, 8, act=F.ACT_TANH),
                                                           nets._dense(8, 1, act=F.ACT_TANH)], F.OB_VECTOR, 3))}
    th = torch.zeros(net.num_params, device=DEV)
    d_idx = torch.zeros(4, dtype=torch.int64, device=DEV)
    d_sc = torch.zeros(4, device=DEV)
    d_init = torch.zeros(4, 2, dtype=torch.float64, device=DEV)
    d_ret, d_sret = torch.full((4,), -1.0, device=DEV), torch.full((4,), -1.0, device=DEV)
    d_len = torch.full((4,), -1, dtype=torch.int32, device=DEV)
    m = torch.zeros(3, device=DEV)

    def call(n_, T, net_=net, ret=d_ret, sret=d_sret, mean=None, std=None, s=None, q=None):
        return L.dne_pendulum_episodes(ctx.handle, C.byref(net_.desc), F.ptr(th), F.ptr(d_idx), F.ptr(d_sc), None, n_,
                                       F.ptr(d_init), T, F.ptr(mean), F.ptr(std), None, F.ptr(ret), F.ptr(sret),
                                       F.ptr(d_len), None, F.ptr(s), F.ptr(q), F.stream_ptr())
    for what, bad in unsup.items():
        assert call(4, 10, bad) == -4, what
        assert L.dne_last_error().decode().startswith("dne_pendulum_episodes"), what
        assert L.dne_pendulum_net_supported(C.byref(bad.desc)) == -4, what
    assert call(0, 10, unsup["wide"]) == -4                 # the net is checked before the n == 0 early return
    assert call(0, 10) == 0
    torch.cuda.synchronize()
    assert (d_ret == -1.0).all() and (d_len == -1).all()
    for T in (0, 201, -1):
        assert call(4, T) == -1, T
    assert call(4, 10, ret=None) == -1 and call(4, 10, sret=None) == -1 and call(-1, 10) == -1
    assert call(4, 10, mean=m) == -1 and call(4, 10, std=m) == -1
    s = torch.zeros(4, 3, dtype=torch.float64, device=DEV)
    assert call(4, 10, s=s) == -1 and call(4, 10, q=s) == -1
    assert call(4, 200, mean=m, std=m + 1, s=s, q=s.clone()) == 0
    torch.cuda.synchronize()
    assert (d_len == 200).all()


def test_runner_matches_direct_launch(ctx, host_noise):
    net = _net()
    P = net.num_params
    rs = np.random.RandomState(12)
    theta = torch.from_numpy(_theta_rows(rs, P, 3)).to(DEV)
    units = [Unit(int(rs.randint(0, NOISE_COUNT - P)), (0.02, -0.02), theta_idx=i % 3) for i in range(40)] + \
            [Unit(0, (0.0, 0.0), theta_idx=1, noiseless=True) for _ in range(3)]
    mean, std = torch.tensor([0.1, -0.1, 0.3], device=DEV), torch.tensor([0.7, 0.7, 2.0], device=DEV)
    r = make_runner(ctx, net, PendulumEnv(4, seed=33), n_slots=4, group=2)
    assert isinstance(r, EpisodeKernelRunner)
    res = r.run(theta, units, 150, ob_mean=mean, ob_std=std, collect_bc="final", ac_noise_std=0.01,
                random_stream=np.random.RandomState(77), save_obs_prob=0.3)
    n = 2 * len(units)
    init = PendulumEnv(4, seed=33).initial_states(n)
    idx = np.repeat([u.noise_idx for u in units], 2)
    scale = np.array([s for u in units for s in u.scales], np.float32)
    rows = np.repeat([u.theta_idx for u in units], 2)
    noisy = scale != 0
    stream = np.random.RandomState(77)
    save = np.zeros(n, bool)
    for m in np.nonzero(noisy)[0]:
        save[m] = stream.rand() < 0.3
    acn = np.zeros((n, 150, 1), np.float32)
    acn[noisy] = stream.randn(int(noisy.sum()), 150, 1).astype(np.float32) * np.float32(0.01)
    d = _launch(ctx, net, theta.cpu().numpy(), idx, scale, rows, init, 150, mean.cpu().numpy(), std.cpu().numpy(), acn)
    np.testing.assert_array_equal(res.returns.ravel(), d["ret"])
    np.testing.assert_array_equal(res.signreturns.ravel(), d["sret"])
    np.testing.assert_array_equal(res.lengths.ravel(), d["len"])
    np.testing.assert_array_equal(np.stack([b for u in res.bcs for b in u]), d["fin"])
    assert 0 < save.sum() < noisy.sum() and res.ob_count == 150 * int(save.sum())
    s, q = np.zeros(3), np.zeros(3)
    for m in np.nonzero(save)[0]:
        s += d["s"][m]
        q += d["q"][m]
    assert res.ob_sum.tobytes() == s.tobytes() and res.ob_sumsq.tobytes() == q.tobytes()
    assert res.steps == 150 * n and res.ticks == 1


def _exp(**over):
    with open(CONFIG) as f:
        exp = json.load(f)
    exp["config"].update(snapshot_freq=0, **over)
    return exp


@pytest.mark.parametrize("hidden,bins,kernel", [((64, 64), "continuous:", True), ((512,), "continuous:", True),
                                                ((256, 256), "continuous:", False),
                                                ((64, 64), "uniform:5", False)])
def test_make_runner_choice_and_es_generation(ctx, noise, hidden, bins, kernel):
    from es_distributed import es as ES
    from es_distributed import policies
    env = PendulumEnv(8, seed=0)
    pol = policies.MujocoPolicy(env.observation_space, env.action_space, ac_bins=bins, ac_noise_std=0.01,
                                nonlin_type="tanh", hidden_dims=list(hidden), connection_type="ff", seed=1)
    fn = pol.action_fn if pol._bin_values is not None else None
    r = make_runner(ctx, pol.net, env, n_slots=8, group=2, pipeline=2, action_fn=fn)
    assert isinstance(r, EpisodeKernelRunner) == kernel and r.action_fn is fn
    exp = _exp(episodes_per_batch=16)
    exp["policy"]["args"].update(hidden_dims=list(hidden), ac_bins=bins)
    ES.set_default_noise(noise)
    log = []
    ES.run_master(None, None, exp, max_iterations=1, n_slots=8, env=PendulumEnv(8, seed=2), noise=noise, seed=3,
                  on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 1 and log[0]["returns_n2"].shape == (8, 2) and (log[0]["lengths_n2"] == 200).all()
    assert np.isfinite(log[0]["returns_n2"]).all() and (log[0]["returns_n2"] < 0).all()


def test_es_run_master_on_pendulum_matches_oracle(noise, host_noise):
    from es_distributed import es as ES
    from es_distributed import policies
    seed = 11
    exp = _exp(episodes_per_batch=64, eval_prob=0.05, calc_obstat_prob=0.2)
    log = []

    def on_it(it, stats, extra):
        log.append((dict(stats), {k: (v.clone() if hasattr(v, "clone") else np.array(v)) for k, v in extra.items()
                                  if k in ("noise_inds_n", "returns_n2", "g", "theta")},
                    extra["ob_stat"].mean.copy(), float(extra["ob_stat"].count)))
    ES.set_default_noise(noise)
    env = PendulumEnv(8, seed=6)
    theta_final = ES.run_master(None, None, exp, max_iterations=2, n_slots=8, env=env, noise=noise, seed=seed,
                                on_iteration=on_it)
    P = PO.policy_net((64, 64)).num_params
    theta = policies.MujocoPolicy(env.observation_space, env.action_space, seed=seed,
                                  **exp["policy"]["args"]).get_trainable_flat()
    adam = O.Adam(theta, exp["optimizer"]["args"]["stepsize"])
    rs = np.random.RandomState(seed)
    for stats, ex, mean, count in log:
        n_pairs = 32
        n_eval = int(rs.binomial(n_pairs, 0.05))
        idx = np.array([O.sample_index(rs, NOISE_COUNT, P) for _ in range(n_pairs)], dtype=np.int64)
        np.testing.assert_array_equal(ex["noise_inds_n"], idx)
        ret = ex["returns_n2"]
        g, ratio, new_theta = O.es_generation_update(adam.theta, adam, host_noise, idx, ret, exp["config"]["l2coeff"])
        assert np.abs(ex["g"].cpu().numpy() - g).max() <= 1e-5 * max(np.abs(g).max(), 1e-30)
        np.testing.assert_allclose(ex["theta"].cpu().numpy(), new_theta, rtol=0, atol=2e-7)
        assert stats["UpdateRatio"] == pytest.approx(float(ratio), rel=1e-4)
        assert stats["EvalEpCount"] == n_eval and stats["ObCount"] > 0 and stats["ObCount"] % 200 == 0
        assert count > 1 and np.abs(mean).max() > 0                 # the RunningStat moved
    np.testing.assert_allclose(theta_final, adam.theta, rtol=0, atol=2e-7)


@pytest.mark.parametrize("ga_mode", ["cpu", "gpu"])
def test_ga_run_master_on_pendulum(noise, tmp_path, ga_mode):
    from es_distributed import ga as GA
    exp = _exp(episodes_per_batch=24)
    exp.update(population_size=4, num_elites=1, ga_mode=ga_mode)
    log = []
    GA.set_default_noise(noise)
    pop, score = GA.run_master(None, str(tmp_path), exp, max_iterations=2, n_slots=8, env=PendulumEnv(8, seed=2),
                               noise=noise, seed=5, on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 2 and len(pop) == 4
    assert all(len(ex["genomes"]) == 24 and (ex["returns"] < 0).all() for ex in log)


def test_nsr_es_rs_and_rollout_on_pendulum(noise, tmp_path):
    from es_distributed import es as ES
    from es_distributed import nses as NS
    from es_distributed import policies
    from es_distributed import rs as RS
    exp = _exp(episodes_per_batch=16, return_proc_mode="centered_sign_rank")
    exp.update(algo_type="nsr", novelty_search={"k": 3, "population_size": 2, "num_rollouts": 1,
                                                "selection_method": "novelty_prob"})
    NS.set_default_noise(noise)
    log = []
    NS.run_master(None, str(tmp_path / "ns"), exp, max_iterations=1, n_slots=8, env=PendulumEnv(8, seed=3), noise=noise,
                  seed=2, on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 1 and log[0]["returns_n2"].shape == (8, 2)
    assert all(np.asarray(b).shape == (2,) and np.asarray(b).dtype == np.float64 for b in log[0]["bcs"])
    assert np.isfinite(log[0]["novelty_n2"]).all()
    rlog = []
    RS.set_default_noise(noise)
    RS.run_master(None, str(tmp_path / "rs"), _exp(episodes_per_batch=16), max_iterations=1, n_slots=8,
                  env=PendulumEnv(8, seed=4), noise=noise, seed=3, on_iteration=lambda it, st, ex: rlog.append(ex))
    assert len(rlog) == 1 and rlog[0]["returns_n2"].shape == (16, 1)
    ES.set_default_noise(noise)
    env = PendulumEnv(2, seed=0)
    pol = policies.MujocoPolicy(env.observation_space, env.action_space, seed=1, **_exp()["policy"]["args"])
    rews, t, bc = pol.rollout(env, timestep_limit=100, random_stream=np.random.RandomState(0))
    assert rews.shape == (1,) and rews[0] < 0 and t == 100 and bc.shape == (2,)


# ------------------------------------------------------------------------------------------------------------------------
class _Reached(Exception):
    pass


def test_es_learns_pendulum(noise):
    """pendulum_es.json at seed 0 reaches a mean noiseless return >= -300 over 100 episodes (the initial policy scores about
    -1200, a swing-up about -150)."""
    from es_distributed import es as ES
    exp = _exp()
    ES.set_default_noise(noise)
    ctx = ES.default_context()
    net = _net(tuple(exp["policy"]["args"]["hidden_dims"]))
    evaluator = EpisodeKernelRunner(ctx, net, PendulumEnv(2, seed=12345), group=2)
    history = []

    def on_it(it, stats, extra):
        st = extra["ob_stat"]
        res = evaluator.run(extra["theta"], [Unit(0, (0.0, 0.0), noiseless=True) for _ in range(50)], None,
                            ob_mean=torch.from_numpy(st.mean.astype(np.float32)),
                            ob_std=torch.from_numpy(st.std.astype(np.float32)))
        history.append(float(res.returns.mean()))
        if history[-1] >= LEARN_TARGET:
            raise _Reached(it)
    with pytest.raises(_Reached) as e:
        ES.run_master(None, None, exp, max_iterations=LEARN_MAX_GENERATIONS, env=PendulumEnv(8, seed=0), noise=noise,
                      seed=0, on_iteration=on_it)
    print(f"ES reached mean noiseless return {history[-1]:.1f} after {e.value.args[0]} generations; "
          f"history {[round(h) for h in history[::5]]}")
