"""The union GEMV of the decomposed dense layers (csrc/gemv_bulk.cu) on slot tables whose slices overlap, touch, repeat
or sit at the ends of the table.  Each table runs against the plain-LDG SIMT GEMV (dne_set_option gemv_bulk = 0, one
slice per group) within the forward bound, and on sampled slots against the oracle.  Reruns and CUDA-graph replays must
be bit-identical, and inactive slots untouched."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from oracle import oracle as O            # noqa: E402  (checker only)
from dne import _ffi as F                 # noqa: E402
from dne import nets as N                 # noqa: E402
from dne.engine import SlotForward, make_context   # noqa: E402
from dne.noise import SharedNoiseTable    # noqa: E402

DEV = torch.device("cuda", 0)
NOISE_COUNT = 12_000_000
SIGMA = 0.005


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def ctx(host_noise):
    return make_context(0, SharedNoiseTable(host_noise=host_noise, device=DEV))


def cuda(x):
    return torch.as_tensor(np.ascontiguousarray(x)).to(DEV).contiguous()


def _row_bound(ref, tol):
    return tol * np.maximum(1.0, np.abs(ref).max(axis=1))


def _forward(ctx, net, theta, idx, scale, obs, paired, active=None, theta_idx=None, bulk=1, **kw):
    """Two forwards of one slot table; returns both logits arrays."""
    L = F.lib()
    try:
        F.check(L.dne_set_option(b"gemv_bulk", bulk))
        sf = SlotForward(ctx, net, len(idx))
        sf.set_slots(idx, scale, active=active, theta_idx=theta_idx)
        sf.logits.fill_(123.0)
        outs = []
        for _ in range(2):
            sf.forward(theta, obs, paired=paired, **kw)
            outs.append(sf.logits.clone())
        torch.cuda.synchronize()
    finally:
        F.check(L.dne_set_option(b"gemv_bulk", 1))
    return [o.cpu().numpy() for o in outs]


def _fc_dims(net):
    fc = net.layers[3]
    return fc.cin, fc.cout


def _es_table(rs, P, K, N_):
    """16 antithetic pairs: full overlap (3 pairs on one index), touching and overlapping offsets
    (d = 1, 2, 3, N-1, N, N+1, K*N-1 from one start), the first and last legal offsets, and random ones."""
    hi = NOISE_COUNT - P
    a = int(rs.randint(0, hi // 4))
    b = int(rs.randint(hi // 4, hi // 2))
    pidx = [a, a, a, b] + [b + d for d in (1, 2, 3, N_ - 1, N_, N_ + 1, K * N_ - 1)] + [0, hi]
    pidx += rs.randint(0, hi + 1, size=16 - len(pidx)).tolist()
    assert max(pidx) <= hi
    return np.repeat(np.array(pidx, dtype=np.int64), 2)


def _crowded_table(rs, P, n_pairs=16):
    """12 pairs on one region (more covering groups than one pass takes) + random pairs."""
    hi = NOISE_COUNT - P
    c = int(rs.randint(0, hi - 2000))
    pidx = [c + 7 * i for i in range(12)] + rs.randint(0, hi + 1, size=n_pairs - 12).tolist()
    return np.repeat(np.array(pidx, dtype=np.int64), 2)


def _check_vs_simt_and_oracle(ctx, host_noise, net_name, idx, paired, active=None, parents=None, theta_idx=None,
                              n_oracle=6, seed=0):
    net, net_o = N.make_net(net_name), O.make_net(net_name)
    P = net.num_params
    rs = np.random.RandomState(seed)
    n = len(idx)
    mlp = net.ob_kind == F.OB_VECTOR
    if parents is None:
        theta_h = (rs.randn(P) * 0.05).astype(np.float32)
        scale = np.tile([SIGMA, -SIGMA], n // 2).astype(np.float32)
    else:
        theta_h = parents
        scale = np.full(n, 0.002, dtype=np.float32)
    obs = ((rs.randn(n, 376) * 2).astype(np.float32) if mlp else
           rs.randint(0, 256, size=(n, 84, 84, 4)).astype(np.uint8))
    ob = {}
    if mlp:
        ob = dict(ob_mean=rs.randn(376).astype(np.float32), ob_std=(np.abs(rs.randn(376)) + 0.1).astype(np.float32))
    d_ob = {k: cuda(v) for k, v in ob.items()}
    d_theta, d_obs = cuda(theta_h), cuda(obs)
    lu, again = _forward(ctx, net, d_theta, idx, scale, d_obs, paired, active, theta_idx, 1, **d_ob)
    np.testing.assert_array_equal(lu, again)                       # rerun: bit-identical
    ls, _ = _forward(ctx, net, d_theta, idx, scale, d_obs, paired, active, theta_idx, 0, **d_ob)
    on = np.arange(n) if active is None else np.flatnonzero(active)
    if active is not None:
        off = np.flatnonzero(active == 0)
        assert (lu[off] == 123.0).all()                            # inactive slots untouched
    tol = 2e-4 if mlp else 2e-5
    bound = 2 * _row_bound(ls[on], tol)
    err = np.abs(lu[on] - ls[on]).max(axis=1)
    assert (err <= bound).all(), (err.max(), on[err > bound])
    rows = sorted(set(rs.choice(on, size=min(n_oracle, len(on)), replace=False).tolist()) | {int(on[0]), int(on[-1])})
    ref = []
    for s in rows:
        base = theta_h if theta_idx is None else theta_h[theta_idx[s]]
        th = (base + np.float32(scale[s]) * host_noise[idx[s]:idx[s] + P]).astype(np.float32)
        ref.append(O.forward(net_o, th, obs[s:s + 1], **ob)[0][0])
    ref = np.stack(ref)
    err = np.abs(lu[rows] - ref).max(axis=1)
    assert (err <= _row_bound(ref, tol)).all(), (err.max(), np.array(rows)[err > _row_bound(ref, tol)])


def test_largemodel_overlapping_touching_and_edge_slices(ctx, host_noise):
    net = N.make_net("LargeModel")
    K, N_ = _fc_dims(net)
    idx = _es_table(np.random.RandomState(1), net.num_params, K, N_)
    active = np.ones(len(idx), dtype=np.uint8)
    active[2:4] = 0                                                # a pair whose slice the pairs around it cover
    _check_vs_simt_and_oracle(ctx, host_noise, "LargeModel", idx, True, active=active, seed=11)


def test_largemodel_more_covering_groups_than_one_pass(ctx, host_noise):
    net = N.make_net("LargeModel")
    idx = _crowded_table(np.random.RandomState(2), net.num_params)
    _check_vs_simt_and_oracle(ctx, host_noise, "LargeModel", idx, True, seed=12)
    _check_vs_simt_and_oracle(ctx, host_noise, "LargeModel", idx, False, seed=13)    # unpaired: G = 1, 24 groups


def test_largemodel_unpaired_edges(ctx, host_noise):
    net = N.make_net("LargeModel")
    K, N_ = _fc_dims(net)
    idx = _es_table(np.random.RandomState(3), net.num_params, K, N_)
    idx[1::2] += np.arange(len(idx) // 2) % 5                      # members of a pair no longer share the slice
    idx = np.minimum(idx, NOISE_COUNT - net.num_params)
    _check_vs_simt_and_oracle(ctx, host_noise, "LargeModel", idx, False, seed=14)


def test_largemodel_ga_shared_parents(ctx, host_noise):
    """GA: siblings (2p, 2p+1) share a parent row, and cousins share it too, so the parent-row GEMV dedupes them."""
    net = N.make_net("LargeModel")
    P = net.num_params
    rs = np.random.RandomState(4)
    parents = (rs.randn(3, P) * 0.05).astype(np.float32)
    n = 24
    theta_idx = np.repeat(np.array([0, 0, 0, 1, 2, 2, 0, 1, 1, 2, 0, 2], dtype=np.int32), 2)
    idx = rs.randint(0, NOISE_COUNT - P + 1, size=n).astype(np.int64)
    _check_vs_simt_and_oracle(ctx, host_noise, "LargeModel", idx, 2, parents=parents, theta_idx=theta_idx, seed=15)


def test_mlp_overlapping_slices(ctx, host_noise):
    net = N.make_net("MujocoPolicy")
    P = net.num_params
    rs = np.random.RandomState(5)
    hi = NOISE_COUNT - P
    c = int(rs.randint(0, hi - 100_000))
    pidx = [c, c, c + 1, c + 255, c + 256, c + 257, c + 376 * 256 - 1, 0, hi] + [c + 3 * i for i in range(12)]
    pidx += rs.randint(0, hi + 1, size=24 - len(pidx)).tolist()
    idx = np.repeat(np.array(pidx, dtype=np.int64), 2)
    _check_vs_simt_and_oracle(ctx, host_noise, "MujocoPolicy", idx, True, seed=16)
    _check_vs_simt_and_oracle(ctx, host_noise, "MujocoPolicy", idx, False, seed=17)


def test_graph_replay_is_bit_identical(ctx, host_noise):
    """A captured tick (bench.py's DNE_BENCH_GRAPH=1 mode) replayed twice gives the eager tick's logits bit for bit."""
    net = N.make_net("LargeModel")
    P = net.num_params
    rs = np.random.RandomState(6)
    idx = _crowded_table(rs, P, n_pairs=64)
    scale = np.tile([SIGMA, -SIGMA], len(idx) // 2).astype(np.float32)
    theta = cuda((rs.randn(P) * 0.05).astype(np.float32))
    obs = cuda(rs.randint(0, 256, size=(len(idx), 84, 84, 4)).astype(np.uint8))
    sf = SlotForward(ctx, net, len(idx))
    sf.set_slots(idx, scale)
    sf.forward(theta, obs, paired=True)
    torch.cuda.synchronize()
    eager = sf.logits.clone()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            sf.forward(theta, obs, paired=True)
    torch.cuda.current_stream().wait_stream(s)
    outs = []
    for _ in range(2):
        sf.logits.fill_(0.0)
        g.replay()
        torch.cuda.synchronize()
        outs.append(sf.logits.clone())
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0], eager)
