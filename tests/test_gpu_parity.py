"""GPU parity tests: the CUDA path (through the C ABI of libdne.so) against the CPU oracle and the committed
golden vectors generated from the reference's own numpy code.  Run on an H100: pytest -m gpu.

Tolerances (stated once):
  * integer / index / rank / selection bookkeeping: bit-exact
  * optimizer steps (float32 elementwise): bit-exact vs the float32 oracle; rtol 2e-6 vs the reference's
    float64-promoted output under numpy 2 (tests/golden/make_golden.py docstring)
  * ES gradient: |g - g_ref|_inf <= 1e-5 * |g_ref|_inf  (north_star: 1e-5 relative)
  * forward logits (float32, different summation order than TF/torch): |d|_inf <= 2e-5 * max(1, |logits|_inf)
    (5e-4 through virtual batch norm, 2e-4 for the tanh MLP);
    actions must agree wherever the oracle's top-2 logit gap exceeds that bound.
"""
import ctypes as C
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
if not torch.cuda.is_available():           # collected on the CPU box too: skip there, never fall back
    pytest.skip("needs a CUDA device", allow_module_level=True)

from oracle import oracle as O            # noqa: E402  (checker only)
from dne import _ffi as F                 # noqa: E402
from dne import nets as N                 # noqa: E402
from dne.engine import ESUpdate, SlotForward, make_context   # noqa: E402
from dne.noise import SharedNoiseTable    # noqa: E402

DEV = torch.device("cuda", 0)
NOISE_COUNT = 6_000_000


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def table(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device=DEV)


@pytest.fixture(scope="module")
def ctx(table):
    return make_context(0, table)


def cuda(x, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(x))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(DEV).contiguous()


# ---------------------------------------------------------------------------------------------------
def test_library_loaded_and_noise_bit_exact(table, host_noise, golden):
    assert F.lib().dne_version() >= 100
    got = table.device_tensor[:NOISE_COUNT].cpu().numpy()
    np.testing.assert_array_equal(got, host_noise)
    np.testing.assert_array_equal(got[:64], golden["noise_head"])          # reference es.py:60 prefix
    np.testing.assert_array_equal(table.get(5, 7).cpu().numpy(), host_noise[5:12])
    s1, s2 = np.random.RandomState(7), np.random.RandomState(7)
    big = 250_000_000
    # sample_index bookkeeping (es.py:66-67) is host integer arithmetic and must be bit-exact
    class _Fake(SharedNoiseTable):
        def __init__(self):
            self.count = big
    fake = _Fake()
    got_idx = [fake.sample_index(s1, 4052658) for _ in range(16)]
    np.testing.assert_array_equal(got_idx, golden["sample_index_P4052658"])
    assert got_idx == [O.sample_index(s2, big, 4052658) for _ in range(16)]


@pytest.mark.parametrize("n", [1, 8, 500, 5000])
def test_centered_rank_golden_bit_exact(ctx, golden, n):
    upd = ESUpdate(ctx, np.zeros(4, np.float32), "sgd", stepsize=0.1)
    x = golden[f"rank_in_{n}"]
    cen, ranks = upd.centered_ranks(cuda(x))
    np.testing.assert_array_equal(ranks.cpu().numpy(), golden[f"rank_ranks_{n}"])
    np.testing.assert_array_equal(cen.cpu().numpy(), golden[f"rank_centered_{n}"])


def test_centered_rank_ties_and_edges(ctx):
    upd = ESUpdate(ctx, np.zeros(4, np.float32), "sgd", stepsize=0.1)
    rs = np.random.RandomState(0)
    # Frostbite-like returns: multiples of 10 -> heavy ties; canonical stable order
    x = (rs.binomial(40, 0.05, size=(500, 2)) * 10).astype(np.float32)
    cen, ranks = upd.centered_ranks(cuda(x))
    np.testing.assert_array_equal(ranks.cpu().numpy(), O.compute_ranks(x.ravel()))
    np.testing.assert_array_equal(cen.cpu().numpy(), O.compute_centered_ranks(x))
    # all equal, negatives, -0.0/+0.0, inf, nan-last
    x = np.array([[0.0, -0.0], [np.inf, -np.inf], [np.nan, 3.0], [3.0, -7.5]], dtype=np.float32)
    cen, ranks = upd.centered_ranks(cuda(x))
    np.testing.assert_array_equal(ranks.cpu().numpy(), O.compute_ranks(x.ravel()))
    # large: 20000 values (pop 10000), property: ranks are a permutation and order-consistent
    x = rs.randn(10000, 2).astype(np.float32)
    cen, ranks = upd.centered_ranks(cuda(x))
    r = ranks.cpu().numpy()
    assert np.array_equal(np.sort(r), np.arange(20000))
    np.testing.assert_array_equal(r, O.compute_ranks(x.ravel()))


def test_es_grad_golden_and_referee(ctx, golden, host_noise):
    P, idx, returns = int(golden["grad_P"]), golden["grad_idx"], golden["grad_returns"]
    upd = ESUpdate(ctx, np.zeros(P, np.float32), "adam", stepsize=0.01)
    cen, _ = upd.centered_ranks(cuda(returns))
    g = upd.gradient(cen, cuda(idx), denom=returns.size).cpu().numpy()
    ref = golden["grad_g"]                                   # reference float32 batched_weighted_sum
    scale = np.abs(ref).max()
    assert np.abs(g - ref).max() <= 1e-5 * scale
    g64 = O.es_gradient(O.compute_centered_ranks(returns), host_noise, idx, P, dtype=np.float64)
    assert np.abs(g - g64).max() <= 2e-7 * scale             # kernel accumulates in float64
    # accumulate flag: two half-batches add up to the whole
    h = len(idx) // 2
    upd.gradient(cen[:h].contiguous(), cuda(idx[:h]), denom=returns.size)
    g2 = upd.gradient(cen[h:].contiguous(), cuda(idx[h:]), denom=returns.size, accumulate=True).cpu().numpy()
    assert np.abs(g2 - g64).max() <= 5e-7 * scale


def test_es_grad_large_P_linearity(ctx, host_noise):
    """Full LargeModel width (P = 4,052,658) -- size-independent properties: linearity in the weights and
    agreement with the float64 referee on a sample of coordinates."""
    P = 4052658
    rs = np.random.RandomState(1)
    n = 24
    idx = rs.randint(0, NOISE_COUNT - P + 1, size=n).astype(np.int64)
    a = rs.randn(n, 2).astype(np.float32)
    b = rs.randn(n, 2).astype(np.float32)
    upd = ESUpdate(ctx, np.zeros(P, np.float32), "adam", stepsize=0.01)
    d_idx = cuda(idx)
    ga = upd.gradient(cuda(a), d_idx, denom=2 * n).clone()
    gb = upd.gradient(cuda(b), d_idx, denom=2 * n).clone()
    gab = upd.gradient(cuda(a + b), d_idx, denom=2 * n).clone()
    scale = float(gab.abs().max())
    assert float((ga + gb - gab).abs().max()) <= 1e-5 * scale
    cols = rs.randint(0, P, size=4096)
    cols[:4] = [0, 1, P - 2, P - 1]
    w = (a[:, 0] - a[:, 1]).astype(np.float64)
    ref = np.array([(w * host_noise[idx + c].astype(np.float64)).sum() / (2 * n) for c in cols])
    np.testing.assert_allclose(ga.cpu().numpy()[cols], ref, rtol=0, atol=3e-7 * max(scale, 1e-3))


def test_optimizers_bit_exact_and_golden(ctx, golden):
    theta0, grads = golden["opt_theta0"], golden["opt_grads"]
    for kind, kw, key in (("adam", dict(stepsize=0.01), "adam"), ("sgd", dict(stepsize=0.01, momentum=0.9), "sgd")):
        upd = ESUpdate(ctx, theta0, kind, **kw)
        orc = O.Adam(theta0, 0.01) if kind == "adam" else O.SGD(theta0, 0.01, 0.9)
        for k, gk in enumerate(grads):
            ratio = upd.step(0.005, cuda(gk))
            r_o, t_o = orc.update(O.es_update_direction(gk, orc.theta, 0.005))
            got = upd.theta.cpu().numpy()
            np.testing.assert_array_equal(got, t_o)                               # float32 oracle: bit-exact
            np.testing.assert_allclose(got, golden[f"{key}_theta"][k], rtol=2e-6, atol=1e-7)   # reference (f64-promoted)
            np.testing.assert_allclose(float(ratio.cpu()), golden[f"{key}_ratio"][k], rtol=1e-5)
        if kind == "adam":
            np.testing.assert_array_equal(upd.m.cpu().numpy(), orc.m)
            np.testing.assert_array_equal(upd.v.cpu().numpy(), orc.v)


# ---------------------------------------------------------------------------------------------------
def _theta_for(net_o, rs, scale=0.05):
    theta = (rs.randn(net_o.num_params) * scale).astype(np.float32)
    for v in net_o.variables():
        if v.kind == "gamma":
            theta[v.offset:v.offset + v.size] = 1.0 + 0.1 * rs.randn(v.size).astype(np.float32)
    return theta


def _check_logits_actions(logits, actions, ref_logits, tol=2e-5):
    """Per-row bound (a slot with a large perturbation scale has much larger logits than its neighbours)."""
    bound = tol * np.maximum(1.0, np.abs(ref_logits).max(axis=1))
    err = np.abs(logits - ref_logits).max(axis=1)
    assert (err <= bound).all(), (err, bound)
    srt = np.sort(ref_logits, axis=1)
    decided = (srt[:, -1] - srt[:, -2]) > 2 * bound
    ref_act = np.argmax(ref_logits, axis=1)
    np.testing.assert_array_equal(actions[decided], ref_act[decided])
    return decided.mean()


@pytest.mark.parametrize("name,A", [("LargeModel", 18), ("Model", 18), ("GAAtariPolicy", 6)])
@pytest.mark.parametrize("paired", [True, False])
def test_conv_policy_forward_vs_oracle(ctx, host_noise, name, A, paired):
    net = N.make_net(name, num_actions=A)
    net_o = O.make_net(name, num_actions=A)
    assert net.num_params == net_o.num_params
    rs = np.random.RandomState(zlib.crc32(name.encode()) % 1000)      # deterministic across processes
    P = net.num_params
    theta = _theta_for(net_o, rs)
    n_slots = 6
    sigma = 0.02
    if paired:
        pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots // 2).astype(np.int64)
        pidx[0] = (pidx[0] // 4) * 4 + 1           # cover several alignments of the slice start
        pidx[1] = (pidx[1] // 4) * 4 + 3
        idx = np.repeat(pidx, 2)
        scale = np.tile([sigma, -sigma], n_slots // 2).astype(np.float32)
    else:
        idx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots).astype(np.int64)
        idx[0] = (idx[0] // 4) * 4                 # aligned start
        idx[1] = (idx[1] // 4) * 4 + 2
        idx[2] = 0                                  # first slice of the table
        idx[3] = NOISE_COUNT - P                    # last slice of the table
        scale = np.array([sigma, -sigma, 0.0, 0.3, -0.002, sigma], dtype=np.float32)
    obs = rs.randint(0, 256, size=(n_slots, 84, 84, 4)).astype(np.uint8)
    sf = SlotForward(ctx, net, n_slots)
    sf.set_slots(idx, scale)
    actions = sf.forward(cuda(theta), cuda(obs), paired=paired).cpu().numpy()
    logits = sf.logits.cpu().numpy()
    ref = np.stack([O.forward(net_o, (theta + np.float32(scale[s]) * host_noise[idx[s]:idx[s] + P]).astype(np.float32),
                              obs[s:s + 1])[0][0] for s in range(n_slots)])
    frac = _check_logits_actions(logits, actions, ref)
    assert frac > 0.3, frac          # most rows must have a decided argmax, or the check is vacuous


def test_forward_inactive_slots_untouched(ctx, host_noise):
    net = N.make_net("Model")
    rs = np.random.RandomState(5)
    P = net.num_params
    theta = (rs.randn(P) * 0.05).astype(np.float32)
    n_slots = 4
    idx = np.repeat(rs.randint(0, NOISE_COUNT - P + 1, size=2), 2).astype(np.int64)
    scale = np.tile([0.02, -0.02], 2).astype(np.float32)
    obs = cuda(rs.randint(0, 256, size=(n_slots, 84, 84, 4)).astype(np.uint8))
    sf = SlotForward(ctx, net, n_slots)
    sf.set_slots(idx, scale)
    full = sf.forward(cuda(theta), obs, paired=True).clone()
    full_logits = sf.logits.clone()
    sf.actions.fill_(-7)
    sf.logits.fill_(123.0)
    sf.set_slots(idx, scale, active=np.array([1, 0, 0, 1], dtype=np.uint8))
    part = sf.forward(cuda(theta), obs, paired=True).cpu().numpy()
    assert part[1] == -7 and part[2] == -7
    assert part[0] == int(full[0]) and part[3] == int(full[3])
    np.testing.assert_array_equal(sf.logits[0].cpu().numpy(), full_logits[0].cpu().numpy())
    assert float(sf.logits[1, 0]) == 123.0


def test_mlp_forward_vs_oracle(ctx, host_noise):
    net = N.make_net("MujocoPolicy")
    net_o = O.make_net("MujocoPolicy")
    assert net.num_params == net_o.num_params == 166673
    rs = np.random.RandomState(11)
    P = net.num_params
    theta = (rs.randn(P) * 0.1).astype(np.float32)
    n_slots = 10
    pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots // 2).astype(np.int64)
    idx = np.repeat(pidx, 2)
    scale = np.tile([0.02, -0.02], n_slots // 2).astype(np.float32)
    obs = (rs.randn(n_slots, 376) * 3).astype(np.float32)
    mean = rs.randn(376).astype(np.float32)
    std = (np.abs(rs.randn(376)) + 0.1).astype(np.float32)
    sf = SlotForward(ctx, net, n_slots)
    sf.set_slots(idx, scale)
    out = sf.forward(cuda(theta), cuda(obs), paired=True, ob_mean=cuda(mean), ob_std=cuda(std)).cpu().numpy()
    ref = np.stack([O.forward(net_o, O.perturb(theta, host_noise, int(idx[s]), 0.02, +1 if scale[s] > 0 else -1),
                              obs[s:s + 1], ob_mean=mean, ob_std=std)[0][0] for s in range(n_slots)])
    assert np.abs(out - ref).max() <= 2e-4 * max(1.0, np.abs(ref).max())
    # unpaired path must agree with the paired one to float32 reassociation accuracy
    out2 = sf.forward(cuda(theta), cuda(obs), paired=False, ob_mean=cuda(mean), ob_std=cuda(std)).cpu().numpy()
    assert np.abs(out2 - ref).max() <= 2e-4 * max(1.0, np.abs(ref).max())


def test_es_atari_policy_vbn_vs_oracle(ctx, host_noise):
    """ESAtariPolicy (configurations/frostbite_es.json): virtual batch norm reference pass + act."""
    net = N.make_net("ESAtariPolicy")
    net_o = O.make_net("ESAtariPolicy")
    assert net.num_params == net_o.num_params == 1009058
    rs = np.random.RandomState(21)
    P = net.num_params
    theta = _theta_for(net_o, rs)
    n_slots, n_ref = 4, 16
    pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots // 2).astype(np.int64)
    idx = np.repeat(pidx, 2)
    scale = np.tile([0.005, -0.005], n_slots // 2).astype(np.float32)
    ref_batch = rs.randint(0, 256, size=(n_ref, 84, 84, 4)).astype(np.uint8)
    obs = rs.randint(0, 256, size=(n_slots, 84, 84, 4)).astype(np.uint8)
    sf = SlotForward(ctx, net, n_slots, n_ref=n_ref)
    sf.set_slots(idx, scale)
    sf.vbn_reference_pass(cuda(theta), cuda(ref_batch))
    actions = sf.forward(cuda(theta), cuda(obs), paired=True).cpu().numpy()
    logits = sf.logits.cpu().numpy()
    vbn = sf.vbn.cpu().numpy()
    ref_logits = []
    for s in range(n_slots):
        th = O.perturb(theta, host_noise, int(idx[s]), 0.005, +1 if scale[s] > 0 else -1)
        _, stats = O.forward(net_o, th, ref_batch, is_ref=True)
        off = 0
        for mean, var in stats:
            c = mean.size
            np.testing.assert_allclose(vbn[s, off:off + c], mean, rtol=2e-4, atol=2e-5)
            np.testing.assert_allclose(vbn[s, off + c:off + 2 * c], var, rtol=5e-4, atol=1e-6)
            off += 2 * c
        ref_logits.append(O.forward(net_o, th, obs[s:s + 1], vbn_stats=stats)[0][0])
    _check_logits_actions(logits, actions, np.stack(ref_logits), tol=5e-4)


# ---------------------------------------------------------------------------------------------------
def test_ga_materialize_mutate_truncate(ctx, host_noise):
    L = F.lib()
    st = F.stream_ptr()
    for name in ("GAAtariPolicy", "LargeModel"):
        net = N.make_net(name, num_actions=18)
        net_o = O.make_net(name, num_actions=18)
        P = net.num_params
        rs = np.random.RandomState(3)
        seeds = rs.randint(0, NOISE_COUNT - P + 1, size=5).astype(np.int64)
        powers = np.array([0.0, 0.002, 0.002, 0.005, 0.002], dtype=np.float32)
        std = (C.c_double * len(net.layers))(*net.init_std())
        out = torch.empty(P, dtype=torch.float32, device=DEV)
        d_seeds, d_powers = cuda(seeds), cuda(powers)          # keep references: F.ptr() borrows
        # mode 0: gpu path (models/base.py:140-146)
        F.check(L.dne_ga_materialize(ctx.handle, C.byref(net.desc), F.ptr(d_seeds), F.ptr(d_powers), 5, std, 0,
                                     F.ptr(out), st))
        ref = O.ga_materialize_gpu(net_o, host_noise, (int(seeds[0]),) + tuple((int(s), float(p)) for s, p in zip(seeds[1:], powers[1:])))
        np.testing.assert_array_equal(out.cpu().numpy(), ref)
        # mode 1: cpu path (ga.py:256-264) -- single sigma for every later seed
        d_pw = cuda(np.full(5, 0.005, dtype=np.float32))
        F.check(L.dne_ga_materialize(ctx.handle, C.byref(net.desc), F.ptr(d_seeds), F.ptr(d_pw), 5, std, 1,
                                     F.ptr(out), st))
        ref = O.ga_materialize_cpu(net_o, host_noise, [int(s) for s in seeds], 0.005)
        np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-6, atol=1e-9)
        # single mutation on a cached parent (models/base.py:155-156)
        child = torch.empty_like(out)
        F.check(L.dne_ga_mutate(ctx.handle, F.ptr(out), int(seeds[2]), 0.002, P, F.ptr(child), st))
        np.testing.assert_array_equal(child.cpu().numpy(),
                                      (out.cpu().numpy() + np.float32(0.002) * host_noise[seeds[2]:seeds[2] + P]).astype(np.float32))
    rs = np.random.RandomState(4)
    for pop, T in ((1000, 20), (1000, 1000), (7, 3), (1, 1)):
        fit = (rs.binomial(40, 0.05, size=pop) * 10).astype(np.float32)        # heavy ties
        sel = torch.full((T,), -1, dtype=torch.int32, device=DEV)
        d_fit = cuda(fit)
        F.check(L.dne_ga_truncate(F.ptr(d_fit), pop, T, F.ptr(sel), st))
        np.testing.assert_array_equal(sel.cpu().numpy(), O.ga_truncate(fit, T))


def test_knn_novelty(ctx):
    L = F.lib()
    rs = np.random.RandomState(9)
    t_max, D, q, A, k = 40, 128, 6, 23, 10
    def make(nseq):
        lens = rs.randint(1, t_max + 1, size=nseq).astype(np.int32)
        seqs = [rs.randint(0, 256, size=(t, D)).astype(np.uint8) for t in lens]
        pad = np.stack([np.concatenate([s, np.repeat(s[-1:], t_max - len(s), 0)]) for s in seqs])
        return lens, seqs, pad
    ql, qs, qp = make(q)
    al, as_, ap = make(A)
    nb = C.c_size_t()
    F.check(L.dne_knn_ws_bytes(q, A, C.byref(nb)))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    nov = torch.empty(q, dtype=torch.float32, device=DEV)
    d_qp, d_ql, d_ap, d_al = cuda(qp), cuda(ql), cuda(ap), cuda(al)
    F.check(L.dne_knn_novelty(F.ptr(d_qp), F.ptr(d_ql), q, F.ptr(d_ap), F.ptr(d_al), A, t_max, D, k,
                              F.ptr(nov), F.ptr(ws), ws.numel(), F.stream_ptr()))
    ref = np.array([O.compute_novelty_vs_archive(as_, s, k) for s in qs])
    np.testing.assert_allclose(nov.cpu().numpy(), ref.astype(np.float32), rtol=1e-6)
    # archive smaller than k (nses.py:30 slices [:k])
    d_ap3, d_al3 = cuda(ap[:3]), cuda(al[:3])
    F.check(L.dne_knn_novelty(F.ptr(d_qp), F.ptr(d_ql), q, F.ptr(d_ap3), F.ptr(d_al3), 3, t_max, D, k,
                              F.ptr(nov), F.ptr(ws), ws.numel(), F.stream_ptr()))
    ref = np.array([O.compute_novelty_vs_archive(as_[:3], s, k) for s in qs])
    np.testing.assert_allclose(nov.cpu().numpy(), ref.astype(np.float32), rtol=1e-6)


@pytest.mark.parametrize("mode", [0, 1])
def test_preprocess_atari(mode):
    L = F.lib()
    rs = np.random.RandomState(13)
    n = 5
    prev = rs.randint(0, 256, size=(n, 84, 84)).astype(np.uint8)
    cur = rs.randint(0, 256, size=(n, 84, 84)).astype(np.uint8)
    stack = rs.randint(0, 256, size=(n, 84, 84, 4)).astype(np.uint8)
    reset = np.array([1, 0, 0, 1, 0], dtype=np.uint8)
    d_stack, d_prev, d_cur, d_reset = cuda(stack), cuda(prev), cuda(cur), cuda(reset)
    F.check(L.dne_preprocess_atari(F.ptr(d_prev), F.ptr(d_cur), F.ptr(d_stack), F.ptr(d_reset), n, mode,
                                   F.stream_ptr()))
    ref = O.max_and_stack(prev, cur, stack, reset, mode="cpu" if mode == 0 else "gpu")
    np.testing.assert_array_equal(d_stack.cpu().numpy(), ref)


def test_errors_are_reported_not_fatal(ctx):
    L = F.lib()
    net = N.make_net("Model")
    rc = L.dne_perturb_forward_conv(ctx.handle, C.byref(net.desc), None, None, None, None, None, 4, 1, None, None,
                                    None, None, None, 0, None)
    assert rc == -1 and b"null" in L.dne_last_error()
    with pytest.raises(F.DneError):
        F.ptr(torch.zeros(4))            # CPU tensor: no CPU fallback


# ---- pins against fixtures generated from the reference's own expressions (tests/golden/make_golden_nses_ga.py) ---------
@pytest.fixture(scope="module")
def golden2():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_nses_ga.npz"))


def test_knn_novelty_vs_reference_nses(ctx, golden2):
    """dne_knn_novelty against es_distributed/nses.py:12-32 itself (recorded with a stub tensorflow): ragged BC
    sequences, k below / at / above the archive size, archive smaller than k."""
    L = F.lib()
    qp, ql, ap, al = golden2["nov_q_pad"], golden2["nov_q_len"], golden2["nov_a_pad"], golden2["nov_a_len"]
    q, A, t_max, D = len(ql), len(al), qp.shape[1], qp.shape[2]
    nb = C.c_size_t()
    F.check(L.dne_knn_ws_bytes(q, A, C.byref(nb)))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    nov = torch.empty(q, dtype=torch.float32, device=DEV)
    d_qp, d_ql, d_ap, d_al = cuda(qp), cuda(ql), cuda(ap), cuda(al)
    for k in (1, 10, 19, 40):
        F.check(L.dne_knn_novelty(F.ptr(d_qp), F.ptr(d_ql), q, F.ptr(d_ap), F.ptr(d_al), A, t_max, D, k, F.ptr(nov),
                                  F.ptr(ws), ws.numel(), F.stream_ptr()))
        np.testing.assert_allclose(nov.cpu().numpy(), golden2[f"nov_k{k}"].astype(np.float32), rtol=1e-6)
    F.check(L.dne_knn_novelty(F.ptr(d_qp), F.ptr(d_ql), q, F.ptr(d_ap), F.ptr(d_al), 3, t_max, D, 10, F.ptr(nov),
                              F.ptr(ws), ws.numel(), F.stream_ptr()))
    np.testing.assert_allclose(nov.cpu().numpy(), golden2["nov_k10_arch3"].astype(np.float32), rtol=1e-6)


@pytest.mark.parametrize("pop,T", [(1000, 20), (64, 64), (7, 3)])
def test_ga_truncate_vs_reference_argpartition(golden2, pop, T):
    """dne_ga_truncate against the literal ga.py:145-149 numpy expression: best individual first, same top-T set."""
    fit, ref = golden2[f"ga_fit_{pop}_{T}"], golden2[f"ga_sel_{pop}_{T}"]
    sel = torch.full((T,), -1, dtype=torch.int32, device=DEV)
    d_fit = cuda(fit)
    F.check(F.lib().dne_ga_truncate(F.ptr(d_fit), pop, T, F.ptr(sel), F.stream_ptr()))
    got = sel.cpu().numpy()
    assert got[0] == ref[0] and set(got.tolist()) == set(ref.tolist())
    assert (np.diff(fit[got]) <= 0).all()                      # and in descending order (the canonical rule)


def test_warp_atari_rgb_vs_pillow(golden2):
    """dne_warp_atari_rgb (atari_wrappers.py:105,138-142): bit-exact against the oracle (whose resize is pinned bit-exactly
    to Pillow) on max-of-two-frames inputs, and within the reference's own gray ambiguity (1 ulp -> <= 1 level on < 1 %
    of the pixels) of the recorded numpy + Pillow output."""
    rgb = golden2["warp_rgb"]                                   # [6, 210, 160, 3]
    n = len(rgb)
    pair_same = np.stack([rgb, rgb], axis=1)                    # max(a, a) = a: comparable with the recorded frames
    pair_mix = np.stack([rgb, np.roll(rgb, 1, axis=0)], axis=1)
    for pairs, recorded in ((pair_same, golden2["warp_out"]), (pair_mix, None)):
        d_raw = cuda(pairs)
        out = torch.zeros(n, 84, 84, dtype=torch.uint8, device=DEV)
        F.check(F.lib().dne_warp_atari_rgb(F.ptr(d_raw), F.ptr(out), n, F.stream_ptr()))
        got = out.cpu().numpy()
        want = np.stack([O.warp_frame_cpu(np.maximum(p[0], p[1])) for p in pairs])
        np.testing.assert_array_equal(got, want)
        if recorded is not None:
            diff = np.abs(got.astype(np.int32) - recorded.astype(np.int32))
            assert diff.max() <= 1 and (diff != 0).mean() < 0.01


def test_warp_atari_palette_vs_oracle():
    """dne_warp_atari_palette (tf_atari.py:88-92): LUT gather, max over two frames, align_corners bilinear -- bit-exact
    against the float32 formula restatement; the uint8 output is its round(255*x) quantisation."""
    rs = np.random.RandomState(17)
    pal = O.ntsc_gray_palette()
    n = 5
    raw = (rs.randint(0, 128, size=(n, 2, 210, 160)) * 2).astype(np.uint8)
    d_raw, d_pal = cuda(raw), cuda(pal.astype(np.float32))
    out_f = torch.zeros(n, 84, 84, dtype=torch.float32, device=DEV)
    out_u = torch.zeros(n, 84, 84, dtype=torch.uint8, device=DEV)
    F.check(F.lib().dne_warp_atari_palette(F.ptr(d_raw), F.ptr(d_pal), F.ptr(out_f), F.ptr(out_u), n, F.stream_ptr()))
    want = np.stack([O.warp_frame_gpu(raw[i], pal) for i in range(n)])
    np.testing.assert_array_equal(out_f.cpu().numpy(), want)
    np.testing.assert_array_equal(out_u.cpu().numpy(), np.rint(np.clip(want * np.float32(255.0), 0, 255)).astype(np.uint8))
    # chained with the frame stack: d_prev = NULL (the max was taken on the raw frames)
    stack = torch.zeros(n, 84, 84, 4, dtype=torch.uint8, device=DEV)
    reset = cuda(np.ones(n, dtype=np.uint8))
    F.check(F.lib().dne_preprocess_atari(None, F.ptr(out_u), F.ptr(stack), F.ptr(reset), n, 1, F.stream_ptr()))
    got = stack.cpu().numpy()
    assert (got[..., :3] == 0).all() and np.array_equal(got[..., 3], out_u.cpu().numpy())


@pytest.mark.skipif(int(__import__("os").environ.get("DNE_SKIP_FULL_TABLE", "0")) == 1, reason="full 250M-entry table skipped")
def test_ga_materialize_reference_genome_kat(golden2):
    """The 260-mutation Frostbite genome shipped with the reference (gpu_implementation/neuroevolution/display.py:31) on
    the REAL 250,000,000-entry noise table: dne_ga_materialize (mode 0, models/base.py:140-146,155-156) against the
    recorded theta checksums / sampled coordinates (oracle on the same table, tests/golden/make_golden_nses_ga.py)."""
    table = SharedNoiseTable(device=DEV)                         # es.py:54-60: seed 123, 250M entries (~20 s)
    assert table.count == 250_000_000
    dev = table.device_tensor[:250_000_000:1000].double().sum().item()
    assert dev == pytest.approx(float(golden2["genome_noise_checksum"]), rel=1e-9)
    kctx = make_context(0, table)
    net = N.make_net("LargeModel")
    seeds = np.concatenate([[int(golden2["genome_idx0"])], golden2["genome_idx"]]).astype(np.int64)
    powers = np.concatenate([[0.0], golden2["genome_power"]]).astype(np.float32)
    std = (C.c_double * len(net.layers))(*net.init_std())
    out = torch.empty(net.num_params, dtype=torch.float32, device=DEV)
    d_seeds, d_powers = cuda(seeds), cuda(powers)
    F.check(F.lib().dne_ga_materialize(kctx.handle, C.byref(net.desc), F.ptr(d_seeds), F.ptr(d_powers), len(seeds), std, 0,
                                       F.ptr(out), F.stream_ptr()))
    got = out.cpu().numpy()
    np.testing.assert_array_equal(got[golden2["genome_theta_cols"]], golden2["genome_theta_vals"])
    assert got.astype(np.float64).sum() == pytest.approx(float(golden2["genome_theta_sum"]), rel=1e-12, abs=1e-9)
    assert np.square(got.astype(np.float64)).sum() == pytest.approx(float(golden2["genome_theta_sumsq"]), rel=1e-12)
