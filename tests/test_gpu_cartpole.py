"""GPU tests of the fused CartPole-v1 episode kernel (dne_cartpole_episodes) and the drivers running on it.

Referees: the CPU oracle (tests/cartpole_oracle.py: oracle.forward + gym's equations in numpy float64) and, independently,
the engine's per-tick MLP forward (SlotForward / dne_perturb_forward_mlp) stepping the same episodes on the host.

Exact agreement is not defined for every episode: the oracle's float32 matmul sums in a different order than the kernel,
and CUDA's double sin / cos are not correctly rounded.  An episode is excluded from a comparison only if the oracle flags
it MARGINAL -- a logit gap below 1e-4 at some decision, or a visited state within 1e-9 of a termination threshold -- and the
tests print how many were excluded and require at most 1 %."""
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

from oracle import oracle as O                    # noqa: E402
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import cartpole_oracle as CP                       # noqa: E402
from dne import _ffi as F                          # noqa: E402
from dne import nets                               # noqa: E402
from dne.engine import SlotForward, make_context   # noqa: E402
from dne.envs import CartPoleEnv                   # noqa: E402
from dne.noise import SharedNoiseTable             # noqa: E402
from dne.rollout import EpisodeKernelRunner, Unit  # noqa: E402

NOISE_COUNT = 2_000_000
GAP, MARGIN = 1e-4, 1e-9
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONFIG = os.path.join(ROOT, "deep-neuroevolution_b200", "configurations", "cartpole_es.json")
# generations within which cartpole_es.json (episodes_per_batch 1000, seed 0) must reach a mean noiseless return >= 475
LEARN_MAX_GENERATIONS = 90           # reached after 43 on an H100 (twice that, rounded up)


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def noise(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device="cuda:0")


@pytest.fixture(scope="module")
def ctx(noise):
    return make_context(0, noise)


def _launch(ctx, net, theta, idx, scale, rows, init, max_steps, final=True):
    """dne_cartpole_episodes on numpy inputs -> (returns, lengths, final states) as numpy, plus the raw return code."""
    dev = torch.device("cuda", 0)
    n = len(idx)
    th = torch.from_numpy(np.ascontiguousarray(theta, dtype=np.float32)).to(dev)

    def buf(a, dt, width=1):               # n == 0 still hands the library valid (non-null) one-row buffers
        a = np.asarray(a, dt).reshape(n, width)
        return torch.from_numpy(np.ascontiguousarray(a if n else np.zeros((1, width), dt))).to(dev)
    d_idx, d_sc = buf(idx, np.int64), buf(scale, np.float32)
    d_row = None if rows is None else buf(rows, np.int32)
    d_init = buf(init, np.float64, 4)
    ret = torch.full((max(n, 1),), -1.0, dtype=torch.float32, device=dev)
    ln = torch.full((max(n, 1),), -1, dtype=torch.int32, device=dev)
    fin = torch.full((max(n, 1), 4), -7.0, dtype=torch.float64, device=dev) if final else None
    rc = F.lib().dne_cartpole_episodes(ctx.handle, C.byref(net.desc), F.ptr(th), F.ptr(d_idx), F.ptr(d_sc), F.ptr(d_row),
                                       n, F.ptr(d_init), int(max_steps), F.ptr(ret), F.ptr(ln), F.ptr(fin),
                                       F.stream_ptr())
    torch.cuda.synchronize()
    return rc, ret.cpu().numpy()[:n], ln.cpu().numpy()[:n], (fin.cpu().numpy()[:n] if final else None)


def _member(theta_rows, host_noise, idx, s, row):
    P = theta_rows.shape[1]
    return (theta_rows[row] + np.float32(s) * host_noise[idx:idx + P]).astype(np.float32)      # fl(theta + fl(s * n))


def _oracle(onet, theta_rows, host_noise, idx, scale, rows, init, max_steps):
    rows = np.zeros(len(idx), np.int64) if rows is None else rows
    return [CP.cartpole_episode(onet, _member(theta_rows, host_noise, int(idx[m]), scale[m], int(rows[m])), init[m], max_steps)
            for m in range(len(idx))]


def _marginal(ep):
    return ep.min_logit_gap < GAP or ep.min_threshold_margin < MARGIN


def _check_lengths(got_len, eps, what, got_fin=None, atol_state=None, excusable=None):
    """Every episode whose length (or final state, within atol_state) differs from the oracle's must be marginal
    (or ``excusable``); those are the excluded ones, and there may be at most 1 %."""
    marginal = np.array([_marginal(e) for e in eps])
    if excusable is not None:
        marginal |= excusable
    want = np.array([e.length for e in eps])
    differ = got_len != want
    if got_fin is not None:
        fin = np.stack([e.final_state for e in eps])
        differ |= np.abs(got_fin - fin).max(axis=1) > atol_state
    bad = np.nonzero(differ & ~marginal)[0]
    assert len(bad) == 0, f"{what}: episodes {bad[:8].tolist()} differ without being marginal: " \
                          f"got lengths {got_len[bad[:8]]}, oracle {want[bad[:8]]}"
    excluded = int(differ.sum())
    print(f"{what}: {excluded} of {len(eps)} episodes excluded (differ, all marginal); {int(marginal.sum())} flagged marginal")
    assert excluded <= 0.01 * len(eps)
    return ~differ


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


def _theta_rows(rs, onet, n_rows):
    return np.stack([(rs.randn(onet.num_params) * 0.5).astype(np.float32) for _ in range(n_rows)])


# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["SimpleClassifier", "LinearClassifier"])
@pytest.mark.parametrize("max_steps", [1, 2, 7, 50])
def test_short_horizons_match_oracle(ctx, host_noise, name, max_steps):
    net, onet = nets.make_net(name, num_actions=2, ob_dim=4), CP.make_classifier(name)
    rs = np.random.RandomState(100 + max_steps)
    theta = _theta_rows(rs, onet, 4)
    idx, scale, rows = _mixed_population(rs, net.num_params)
    init = rs.uniform(-0.05, 0.05, size=(len(idx), 4))
    if max_steps == 50:                                 # also start some members far from rest: early terminations
        init[::3] *= 30
    rc, ret, ln, fin = _launch(ctx, net, theta, idx, scale, rows, init, max_steps)
    assert rc == 0
    assert (ln >= 1).all() and (ln <= max_steps).all()
    np.testing.assert_array_equal(ret, ln.astype(np.float32))
    eps = _oracle(onet, theta, host_noise, idx, scale, rows, init, max_steps)
    _check_lengths(ln, eps, f"{name} max_steps={max_steps}", fin, 1e-12)


def _es_theta(noise, n_gen=4):
    """theta of SimpleClassifierPolicy after a few ES generations on CartPole (a policy that balances for a while)."""
    from es_distributed import es as ES
    with open(CONFIG) as f:
        exp = json.load(f)
    exp["config"]["episodes_per_batch"] = 200
    exp["config"]["snapshot_freq"] = 0
    ES.set_default_noise(noise)
    return ES.run_master(None, None, exp, max_iterations=n_gen, env=CartPoleEnv(8, seed=1), noise=noise, seed=4)


@pytest.mark.parametrize("which", ["random", "es"])
def test_full_episodes_match_oracle(ctx, noise, host_noise, which):
    from es_distributed import policies
    net, onet = nets.make_net("SimpleClassifier", num_actions=2, ob_dim=4), CP.make_classifier("SimpleClassifier")
    env = CartPoleEnv(8, seed=9)
    if which == "random":
        theta = policies.SimpleClassifierPolicy(env.observation_space, env.action_space, seed=3, ctx=ctx).get_trainable_flat()
        n = 256
    else:
        theta = _es_theta(noise)
        n = 128
    rs = np.random.RandomState(5)
    pidx = rs.randint(0, NOISE_COUNT - net.num_params + 1, size=n // 2)
    idx = np.repeat(pidx, 2).astype(np.int64)
    scale = np.tile([0.02, -0.02], n // 2).astype(np.float32)
    scale[-8:] = 0.0
    init = env.initial_states(n)
    rc, ret, ln, fin = _launch(ctx, net, theta, idx, scale, None, init, 500)
    assert rc == 0
    eps = _oracle(onet, theta[None, :], host_noise, idx, scale, None, init, 500)
    print(f"{which}: mean length {ln.mean():.1f}, max {ln.max()}")
    _check_lengths(ln, eps, f"full episodes ({which})")


def test_per_tick_engine_referee(ctx, noise, host_noise):
    """The per-tick MLP forward (SlotForward, dne_perturb_forward_mlp) + cartpole_oracle.cartpole_step on the host plays the same
    episodes.  Without observation statistics that path feeds the observations unclipped, as the episode kernel does:
    only the marginal episodes may differ."""
    net, onet = nets.make_net("SimpleClassifier", num_actions=2, ob_dim=4), CP.make_classifier("SimpleClassifier")
    P, n, T = net.num_params, 128, 500
    rs = np.random.RandomState(21)
    theta = _es_theta(noise)
    pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n // 2)
    idx = np.repeat(pidx, 2).astype(np.int64)
    scale = np.tile([0.05, -0.05], n // 2).astype(np.float32)
    init = rs.uniform(-0.05, 0.05, size=(n, 4))
    rc, _, ln, _ = _launch(ctx, net, theta, idx, scale, None, init, T, final=False)
    assert rc == 0

    sf = SlotForward(ctx, net, n)
    d_theta = torch.from_numpy(theta).cuda()
    state = init.copy()
    length = np.zeros(n, np.int64)
    active = np.ones(n, bool)
    while active.any():
        obs = state.astype(np.float32)
        sf.set_slots(idx, scale, active=active.astype(np.uint8))
        logits = sf.forward(d_theta, torch.from_numpy(obs).cuda(), paired=False).cpu().numpy()
        for m in np.nonzero(active)[0]:
            state[m], done = CP.cartpole_step(state[m], int(np.argmax(logits[m])))
            length[m] += 1
            if done or length[m] >= T:
                active[m] = False
    eps = _oracle(onet, theta[None, :], host_noise, idx, scale, None, init, T)
    print(f"per-tick referee: mean length {ln.mean():.1f}")
    same = ln == length
    excused = np.array([_marginal(e) for e in eps])
    bad = np.nonzero(~same & ~excused)[0]
    assert len(bad) == 0, f"kernel {ln[bad[:8]]} vs per-tick engine {length[bad[:8]]} at {bad[:8].tolist()}"
    print(f"per-tick referee: {int((~same).sum())} of {n} excluded (all marginal)")
    assert (~same).sum() <= 0.01 * n


def _custom_net(widths, act=F.ACT_RELU, ob_dim=4):
    layers = [nets._dense(widths[i], widths[i + 1], act=act) for i in range(len(widths) - 2)]
    layers.append(nets._dense(widths[-2], widths[-1], act=F.ACT_NONE))
    return nets._finish(nets.NetSpec("custom", layers, F.OB_VECTOR, ob_dim))


def test_contract(ctx, host_noise):
    net = nets.make_net("SimpleClassifier", num_actions=2, ob_dim=4)
    rs = np.random.RandomState(8)
    onet = CP.make_classifier("SimpleClassifier")
    theta = _theta_rows(rs, onet, 4)
    idx, scale, rows = _mixed_population(rs, net.num_params)
    init = rs.uniform(-0.05, 0.05, size=(len(idx), 4))
    a = _launch(ctx, net, theta, idx, scale, rows, init, 500)
    b = _launch(ctx, net, theta, idx, scale, rows, init, 500)
    assert a[0] == b[0] == 0
    for x, y in zip(a[1:], b[1:]):
        assert x.tobytes() == y.tobytes()                      # bit-identical reruns
    # argument errors
    dev = torch.device("cuda", 0)
    th = torch.from_numpy(theta[0]).to(dev)
    d_idx = torch.zeros(4, dtype=torch.int64, device=dev)
    d_sc = torch.zeros(4, dtype=torch.float32, device=dev)
    d_init = torch.zeros(4, 4, dtype=torch.float64, device=dev)
    d_ret = torch.zeros(4, dtype=torch.float32, device=dev)
    d_len = torch.zeros(4, dtype=torch.int32, device=dev)
    L = F.lib()

    def call(n_, max_steps, ret_, len_, net_=net):
        return L.dne_cartpole_episodes(ctx.handle, C.byref(net_.desc), F.ptr(th), F.ptr(d_idx), F.ptr(d_sc), None, n_,
                                       F.ptr(d_init), max_steps, F.ptr(ret_), F.ptr(len_), None, F.stream_ptr())
    d_ret.fill_(-1.0)
    d_len.fill_(-1)
    assert call(0, 10, d_ret, d_len) == 0                       # n_members == 0: a no-op
    torch.cuda.synchronize()
    assert (d_ret == -1.0).all() and (d_len == -1).all()
    assert call(4, 0, d_ret, d_len) == -1                       # DNE_ERR_ARG
    assert call(4, 10, None, d_len) == -1
    assert call(4, 10, d_ret, None) == -1
    assert call(-1, 10, d_ret, d_len) == -1
    # unsupported nets
    unsup = {"width 33": _custom_net([4, 33, 2]), "conv net": nets.make_net("Model", num_actions=2),
             "ob_dim 6": nets.make_net("SimpleClassifier", num_actions=2, ob_dim=6),
             "tanh hidden": _custom_net([4, 16, 2], act=F.ACT_TANH)}
    for what, bad in unsup.items():
        assert call(4, 10, d_ret, d_len, bad) == -4, what          # DNE_ERR_UNSUP
        assert L.dne_last_error().decode().startswith("dne_cartpole_episodes"), what
    # a width-32 net (4 dense layers) is accepted and agrees with the oracle
    w32 = _custom_net([4, 32, 32, 32, 2])
    o32 = CP.dense_net([4, 32, 32, 32, 2])
    assert o32.num_params == w32.num_params
    t32 = (rs.randn(1, w32.num_params) * 0.3).astype(np.float32)
    i32 = rs.randint(0, NOISE_COUNT - w32.num_params + 1, size=64).astype(np.int64)
    s32 = np.full(64, 0.05, np.float32)
    init32 = rs.uniform(-0.05, 0.05, size=(64, 4))
    rc, _, ln, fin = _launch(ctx, w32, t32, i32, s32, None, init32, 50)
    assert rc == 0
    _check_lengths(ln, _oracle(o32, t32, host_noise, i32, s32, None, init32, 50), "width-32 net", fin, 1e-12)


def test_runner_matches_direct_launch(ctx, host_noise):
    """EpisodeKernelRunner: (unit, member) flattening, one initial_states call per run, theta_idx rows, final-state BCs."""
    net = nets.make_net("SimpleClassifier", num_actions=2, ob_dim=4)
    rs = np.random.RandomState(12)
    theta = torch.from_numpy((rs.randn(3, net.num_params) * 0.5).astype(np.float32)).cuda()
    units = [Unit(int(rs.randint(0, NOISE_COUNT - 400)), (0.02, -0.02), theta_idx=i % 3) for i in range(20)]
    env = CartPoleEnv(4, seed=33)
    r = EpisodeKernelRunner(ctx, net, env, n_slots=4, group=2)
    res = r.run(theta, units, 5000, collect_bc="final")
    init = CartPoleEnv(4, seed=33).initial_states(40)
    idx = np.repeat([u.noise_idx for u in units], 2)
    scale = np.tile([0.02, -0.02], 20).astype(np.float32)
    rows = np.repeat([u.theta_idx for u in units], 2)
    rc, ret, ln, fin = _launch(ctx, net, theta.cpu().numpy(), idx, scale, rows, init, 500)
    np.testing.assert_array_equal(res.lengths.ravel(), ln)
    np.testing.assert_array_equal(res.returns.ravel(), ret)
    np.testing.assert_array_equal(res.signreturns.ravel(), ln.astype(np.float32))
    np.testing.assert_array_equal(np.stack([b for u in res.bcs for b in u]), fin)
    assert res.steps == int(ln.sum()) and res.ticks == 1


# ------------------------------------------------------------------------------------------------------------------------
def _cartpole_exp(**over):
    with open(CONFIG) as f:
        exp = json.load(f)
    exp["config"].update(snapshot_freq=0, **over)
    return exp


def test_es_run_master_on_cartpole_matches_oracle(noise, host_noise, tmp_path):
    from es_distributed import es as ES
    from es_distributed import policies
    seed, env_seed = 11, 6
    exp = _cartpole_exp(episodes_per_batch=64, eval_prob=0.05)
    log = []

    def on_it(it, stats, extra):
        log.append((dict(stats), {k: (v.clone() if hasattr(v, "clone") else np.array(v)) for k, v in extra.items()
                                  if k in ("noise_inds_n", "returns_n2", "lengths_n2", "g", "theta")}))
    ES.set_default_noise(noise)
    env = CartPoleEnv(8, seed=env_seed)
    theta_final = ES.run_master(None, str(tmp_path), exp, max_iterations=2, n_slots=8, env=env, noise=noise, seed=seed,
                                on_iteration=on_it)
    assert len(log) == 2
    net = CP.make_classifier("SimpleClassifier")
    P = net.num_params
    theta = policies.SimpleClassifierPolicy(env.observation_space, env.action_space, seed=seed).get_trainable_flat()
    adam = O.Adam(theta, 0.01)
    rs, env_rs = np.random.RandomState(seed), np.random.RandomState(env_seed)
    for stats, ex in log:
        n_pairs = 32
        n_eval = int(rs.binomial(n_pairs, 0.05))
        idx = np.array([O.sample_index(rs, NOISE_COUNT, P) for _ in range(n_pairs)], dtype=np.int64)
        np.testing.assert_array_equal(ex["noise_inds_n"], idx)
        init = env_rs.uniform(-0.05, 0.05, size=((n_pairs + -(-n_eval // 2)) * 2, 4))
        ret = ex["returns_n2"]
        np.testing.assert_array_equal(ret, ex["lengths_n2"].astype(np.float32))     # return == length
        eps = [CP.cartpole_episode(net, O.perturb(adam.theta, host_noise, int(idx[u]), 0.02, 1 - 2 * g), init[2 * u + g], 500)
               for u in range(n_pairs) for g in range(2)]
        _check_lengths(ex["lengths_n2"].ravel(), eps, "ES generation")
        cen = O.compute_centered_ranks(ret)
        g, ratio, new_theta = O.es_generation_update(adam.theta, adam, host_noise, idx, ret, 0.005)
        assert np.abs(ex["g"].cpu().numpy() - g).max() <= 1e-5 * max(np.abs(g).max(), 1e-30)
        np.testing.assert_allclose(ex["theta"].cpu().numpy(), new_theta, rtol=0, atol=2e-7)
        assert stats["UpdateRatio"] == pytest.approx(float(ratio), rel=1e-4)
        assert stats["EvalEpCount"] == n_eval and cen.shape == ret.shape
    np.testing.assert_allclose(theta_final, adam.theta, rtol=0, atol=2e-7)


@pytest.mark.parametrize("ga_mode", ["cpu", "gpu"])
def test_ga_run_master_on_cartpole(noise, host_noise, tmp_path, ga_mode):
    from es_distributed import ga as GA
    exp = _cartpole_exp(episodes_per_batch=24)
    exp.update(population_size=4, num_elites=1, ga_mode=ga_mode)
    log = []
    GA.set_default_noise(noise)
    pop, score = GA.run_master(None, str(tmp_path), exp, max_iterations=2, n_slots=8, env=CartPoleEnv(8, seed=2),
                               noise=noise, seed=5, on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 2 and len(pop) == 4
    prev_pop, prev_score = [], np.array([], dtype=np.float32)
    for ex in log:
        genomes, returns = ex["genomes"], ex["returns"]
        assert len(genomes) == 24 and (returns >= 1).all() and (returns <= 500).all()
        cand = [tuple(p) for p in prev_pop[:1]] + [tuple(g) for g in genomes]
        fit = np.concatenate([prev_score[:1], returns]).astype(np.float32)
        sel = O.ga_truncate(fit, 4)
        assert [tuple(p) for p in ex["population"]] == [cand[i] for i in sel]
        np.testing.assert_array_equal(ex["population_score"], fit[sel])
        prev_pop, prev_score = ex["population"], ex["population_score"]


def test_nsr_es_and_rs_complete_a_generation_on_cartpole(noise, tmp_path):
    from es_distributed import nses as NS
    from es_distributed import rs as RS
    exp = _cartpole_exp(episodes_per_batch=16, return_proc_mode="centered_sign_rank")
    exp.update(algo_type="nsr", novelty_search={"k": 3, "population_size": 2, "num_rollouts": 1,
                                                "selection_method": "novelty_prob"})
    NS.set_default_noise(noise)
    log = []
    NS.run_master(None, str(tmp_path / "ns"), exp, max_iterations=1, n_slots=8, env=CartPoleEnv(8, seed=3), noise=noise,
                  seed=2, on_iteration=lambda it, st, ex: log.append(ex))
    assert len(log) == 1 and log[0]["returns_n2"].shape == (8, 2)
    assert all(np.asarray(b).shape == (4,) and np.asarray(b).dtype == np.float64 for b in log[0]["bcs"])
    assert np.isfinite(log[0]["novelty_n2"]).all()
    rlog = []
    RS.set_default_noise(noise)
    rexp = _cartpole_exp(episodes_per_batch=16)
    RS.run_master(None, str(tmp_path / "rs"), rexp, max_iterations=1, n_slots=8, env=CartPoleEnv(8, seed=4), noise=noise,
                  seed=3, on_iteration=lambda it, st, ex: rlog.append(ex))
    assert len(rlog) == 1 and rlog[0]["returns_n2"].shape == (16, 1) and rlog[0]["best_score"] >= 1


def test_policy_rollout_on_cartpole(noise):
    from es_distributed import es as ES
    from es_distributed import policies
    ES.set_default_noise(noise)
    env = CartPoleEnv(2, seed=0)
    pol = policies.LinearClassifierPolicy(env.observation_space, env.action_space, seed=1)
    rews, t, bc = pol.rollout(env, timestep_limit=100)
    assert rews.shape == (1,) and rews[0] == t and 1 <= t <= 100 and bc.shape == (4,)
    a = pol.act(np.zeros((3, 4), np.float32))
    assert a.shape == (3,) and set(a.tolist()) <= {0, 1}


# ------------------------------------------------------------------------------------------------------------------------
class _Reached(Exception):
    pass


def test_es_learns_cartpole(noise):
    """cartpole_es.json at episodes_per_batch 1000 reaches a mean noiseless return >= 475 over 100 episodes."""
    from es_distributed import es as ES
    exp = _cartpole_exp(episodes_per_batch=1000)
    ES.set_default_noise(noise)
    ctx = ES.default_context()
    net = nets.make_net("SimpleClassifier", num_actions=2, ob_dim=4)
    evaluator = EpisodeKernelRunner(ctx, net, CartPoleEnv(2, seed=12345), group=2)
    history = []

    def on_it(it, stats, extra):
        res = evaluator.run(extra["theta"], [Unit(0, (0.0, 0.0)) for _ in range(50)], 500)
        history.append(float(res.returns.mean()))
        if history[-1] >= 475:
            raise _Reached(it)
    with pytest.raises(_Reached) as e:
        ES.run_master(None, None, exp, max_iterations=LEARN_MAX_GENERATIONS, env=CartPoleEnv(8, seed=0), noise=noise,
                      seed=0, on_iteration=on_it)
    print(f"ES reached mean noiseless return {history[-1]:.1f} after {e.value.args[0]} generations; "
          f"history {[round(h) for h in history]}")
