"""Every dense-layer forward path of dne_launch_dense_layer (csrc/forward_kernels.cu) against a float64 referee.

The dispatch picks a kernel from the layer shape, the slot-table mode and the process-wide options: the union GEMV
(gemv_bulk.cu) for 64 <= N <= 1024 with N/4 dividing 256, the plain SIMT GEMV and theta GEMM otherwise, the fused
combine+head kernel (register and streamed head rows), and dense_small_kernel for every layer the split does not take
(fan-in or width not a multiple of 4, K*N < 16384, width > 1024, wide heads).  Each shape below names the branch it
exists to reach; each runs five slot tables (antithetic pairs at every slice alignment, unpaired slots with a zero and a
large scale, GA siblings on three parent rows, per-slot parent rows, a single slot).

The referee builds every member's weights exactly as the engine does, w = fl32(theta[row] + fl32(s * noise)), normalises
observations in float32 in the kernel's operation order, then runs the layers in float64.  The allowed error of every
output comes from a magnitude forward of the same net on |x|, |theta| + |s * noise| and |b| (see referee()).  The
bound is checked to be sharp: on every shape's data the comparison must reject a referee with the noise index off by
one, one with the last weight row (k = K-1) of the first layer dropped, and (GA tables) one that reads the wrong parent
row.
"""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from oracle import oracle as O            # noqa: E402  (noise table only)
from dne import _ffi as F                 # noqa: E402
from dne import nets as N                 # noqa: E402
from dne.engine import SlotForward, make_context   # noqa: E402
from dne.noise import SharedNoiseTable    # noqa: E402

DEV = torch.device("cuda", 0)
NOISE_COUNT = 6_000_000
SIGMA = 0.02
U = 2.0 ** -24                            # float32 unit roundoff
f32, f64 = np.float32, np.float64

# every option of dne_set_option (include/dne.h) with its default
DEFAULTS = dict(conv_tc=2, theta_tma=1, theta_mc=0, fuse_head=1, fold_theta=1, pdl=1, chain_ticks=0, gemv_bulk=1,
                gemv_ctas_per_sm=2, gemv_stages=5, gemv_grid=0)


def set_option(name, value):
    F.check(F.lib().dne_set_option(name.encode(), int(value)))


@pytest.fixture(autouse=True)
def restore_options():
    yield
    for k, v in DEFAULTS.items():
        set_option(k, v)


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def ctx(host_noise):
    return make_context(0, SharedNoiseTable(host_noise=host_noise, device=DEV))


def cuda(x):
    return torch.as_tensor(np.ascontiguousarray(x)).to(DEV).contiguous()


# ---- the float64 referee -------------------------------------------------------------------------------------------
def normalise(obs, mean, std):
    """ob_norm_kernel: fl32(fl32(o - mean) / std) clipped to [-5, 5]; without statistics the observation unchanged."""
    obs = obs.astype(f32)
    if mean is None:
        return obs
    return np.minimum(np.maximum((obs - mean.astype(f32)) / std.astype(f32), f32(-5)), f32(5))


def member(theta_rows, row, noise, idx, s, P):
    """(w, |theta| + |s * noise|): the member's float32 weights as the engine builds them, and their magnitudes."""
    th = theta_rows[row]
    sn = (f32(s) * noise[idx:idx + P]).astype(f32)
    return (th + sn).astype(f32), np.abs(th).astype(f64) + np.abs(sn).astype(f64)


def referee(net, w, wmag, x0, drop_last_row_of=None):
    """float64 forward of one member on float32 input x0 -> (outputs, per-output error bound).

    Per layer: A = sum_k mag_k |W_kn| + |b_n| is the magnitude of everything the kernel adds (mag = |x| + the input's
    bound; |W| = |theta| + |s * noise|: the split layers add x.theta and s * (x.noise) separately), and the sum may be
    off by u * (4 sqrt(K) + 16) * A: the random-walk growth of K float32 roundings, plus the roundings of w = theta +
    s * noise, of the theta / noise split and of the partial sums.  The input's error reaches the output through W as a
    root-sum-square (the hidden units' errors come from independent roundings), never more than the worst case
    sum_k e_k |W_kn|: the worst case alone compounds by sum_k |W_kn| per layer, which in an eight-layer stack outgrows
    what an off-by-one noise slice changes.  tanh passes an error on with its largest slope over [z - e, z + e] and adds
    tanhf's 2 ulp; ReLU passes it on where z + e > 0."""
    x = x0.astype(f64)
    err = np.zeros_like(x)
    for li, l in enumerate(net.layers):
        K, Nn = l.cin, l.cout
        W = w[l.off_w:l.off_w + K * Nn].astype(f64).reshape(K, Nn)
        Wm = wmag[l.off_w:l.off_w + K * Nn].reshape(K, Nn)
        b = w[l.off_b:l.off_b + Nn].astype(f64)
        if drop_last_row_of == li:
            W, Wm, x, err = W[:-1], Wm[:-1], x[:-1], err[:-1]
        z = x @ W + b
        A = (np.abs(x) + err) @ Wm + np.abs(b)
        e = np.minimum(err @ np.abs(W), np.sqrt(np.square(err) @ np.square(W))) + U * (4.0 * np.sqrt(K) + 16.0) * A
        if l.act == F.ACT_TANH:
            x = np.tanh(z)
            slope = np.where(np.abs(z) > e, 1.0 - np.square(np.tanh(np.abs(z) - e)), 1.0)
            err = slope * e + 4.0 * U * np.minimum(np.abs(x) + slope * e, 1.0)
        elif l.act == F.ACT_RELU:
            x, err = np.maximum(z, 0.0), np.where(z + e > 0.0, e, 0.0)
        else:
            x, err = z, e
    return x, err


def referee_table(net, theta_rows, noise, tab, x0, *, idx_shift=0, row_shift=0, drop=None):
    P = net.num_params
    ref, bound = [], []
    for s in range(len(tab["idx"])):
        i = int(tab["idx"][s]) + idx_shift
        if i + P > len(noise):
            i -= 2 * idx_shift
        row = 0 if tab["theta_idx"] is None else (int(tab["theta_idx"][s]) + row_shift) % len(theta_rows)
        w, wm = member(theta_rows, row, noise, i, tab["scale"][s], P)
        r, e = referee(net, w, wm, x0[s], drop)
        ref.append(r)
        bound.append(e)
    return np.array(ref), np.array(bound)


def violations(out, ref, bound, rows):
    """Number of outputs of the listed slots outside the bound."""
    return int((np.abs(out[rows].astype(f64) - ref[rows]) > bound[rows]).sum())


# ---- slot tables ---------------------------------------------------------------------------------------------------
def tables(rs, P):
    hi = NOISE_COUNT - P
    out = {}
    # paired = 1: 13 antithetic pairs -- slice starts at every alignment mod 4, the first and last legal offsets, two
    # pairs on one index, one inactive pair (left untouched)
    q = 4 * int(rs.randint(1, hi // 4 - 4))
    pidx = [q, q + 1, q + 2, q + 3, 0, hi, q + 7, q + 7] + rs.randint(0, hi + 1, size=5).tolist()
    active = np.ones(26, np.uint8)
    active[18:20] = 0
    out["paired"] = dict(idx=np.repeat(np.array(pidx, np.int64), 2), scale=np.tile([SIGMA, -SIGMA], 13).astype(f32),
                         paired=1, theta_idx=None, active=active, n_theta=1)
    # paired = 0: 7 slots, scales with a zero and a large one
    out["unpaired"] = dict(idx=rs.randint(0, hi + 1, size=7).astype(np.int64),
                           scale=np.array([SIGMA, -SIGMA, 0.0, 0.5, 0.01, -0.03, SIGMA], f32),
                           paired=0, theta_idx=None, active=None, n_theta=1)
    # paired = 2: GA siblings (2p, 2p+1) share one of 3 parent rows (rows start unaligned when P % 4 != 0)
    out["ga_pairs"] = dict(idx=rs.randint(0, hi + 1, size=10).astype(np.int64),
                           scale=np.full(10, 0.01, f32), paired=2,
                           theta_idx=np.repeat(np.array([0, 1, 2, 2, 1], np.int32), 2), active=None, n_theta=3)
    # paired = 0 with per-slot parent rows
    out["ga_rows"] = dict(idx=rs.randint(0, hi + 1, size=6).astype(np.int64),
                          scale=np.array([0.01, -0.02, 0.0, 0.01, 0.03, -0.01], f32), paired=0,
                          theta_idx=np.array([2, 0, 1, 1, 2, 0], np.int32), active=None, n_theta=3)
    out["single"] = dict(idx=np.array([rs.randint(0, hi + 1)], np.int64), scale=np.array([SIGMA], f32), paired=0,
                         theta_idx=None, active=None, n_theta=1)
    return out


def init_theta(rs, net, n_rows):
    """Weights ~ N(0, 1/K) per layer, biases ~ N(0, 0.1): pre-activations of order one."""
    rows = np.zeros((n_rows, net.num_params), f32)
    for r in range(n_rows):
        for l in net.layers:
            rows[r, l.off_w:l.off_w + l.cin * l.cout] = rs.randn(l.cin * l.cout) / np.sqrt(l.cin)
            rows[r, l.off_b:l.off_b + l.cout] = 0.1 * rs.randn(l.cout)
    return rows


def run_mlp(ctx, net, theta_rows, tab, obs, ob_mean, ob_std):
    n = len(tab["idx"])
    sf = SlotForward(ctx, net, n)
    sf.set_slots(tab["idx"], tab["scale"], active=tab["active"], theta_idx=tab["theta_idx"])
    sf.logits.fill_(123.0)
    d_theta = cuda(theta_rows if tab["theta_idx"] is not None else theta_rows[0])
    kw = {} if ob_mean is None else dict(ob_mean=cuda(ob_mean), ob_std=cuda(ob_std))
    sf.forward(d_theta, cuda(obs), paired=tab["paired"], **kw)
    torch.cuda.synchronize()
    return sf.logits.cpu().numpy()


# (ob_dim, hidden, ac_dim, nonlin) -> the branch it exists to reach
SHAPES = {
    "humanoid": (376, (256, 256), 17, "tanh"),          # union GEMV N = 256, fused head, register branch
    "humanoid_uniform5": (376, (256, 256), 85, "tanh"),  # fused head, streamed (non-register) head rows
    "humanoid_uniform16": (376, (256, 256), 272, "tanh"),  # head wider than 256 columns (dense_small_kernel tiles)
    "hopper": (11, (64, 64), 3, "tanh"),                # every layer in dense_small_kernel
    "wide_odd_fanin": (17, (300, 300), 6, "relu"),      # 17x300 in dense_small_kernel; N = 300: SIMT GEMV + theta GEMM, no
                                                        # fold; fused head with N1 = 300
    "ant_1024": (111, (1024, 1024), 8, "tanh"),         # 111x1024 in dense_small_kernel; union N = 1024; the fused head's
                                                        # hidden loop runs twice
    "wider_than_1024": (64, (2048,), 4, "tanh"),        # 64x2048 in dense_small_kernel; unfused head with K = 2048
    "union_512_64": (376, (512, 64), 17, "tanh"),       # union N = 512 and N = 64
    "kn_16384": (4096, (4,), 2, "tanh"),                # K*N = 16384: decomposed, N = 4 SIMT GEMV
    "kn_16368": (4092, (4,), 2, "tanh"),                # K*N < 16384: dense_small_kernel with K = 4092
    "eight_layers": (376, (256,) * 7, 17, "tanh"),      # DNE_MAX_LAYERS layers in one tick
    "simple_classifier": None,                          # no normalisation: observations unclipped
    "linear_classifier": None,
}


def make_shape(name):
    if name == "simple_classifier":
        return N.make_net("SimpleClassifier", num_actions=2, ob_dim=4)
    if name == "linear_classifier":
        return N.make_net("LinearClassifier", num_actions=2, ob_dim=4)
    ob, hidden, ac, nl = SHAPES[name]
    return N.make_net("MujocoPolicy", ob_dim=ob, hidden=hidden, ac_dim=ac, nonlin=nl)


def shape_data(rs, net):
    """Observations (z-scores past +-5 where normalised, values well beyond +-5 for the classifiers) and statistics."""
    d = net.ob_dim
    if net.name == "MujocoPolicy":
        mean = rs.randn(d).astype(f32)
        std = (np.abs(rs.randn(d)) + 0.2).astype(f32)
        z = 2.5 * rs.randn(32, d)
        return (mean + std * z).astype(f32), mean, std
    return (12.0 * rs.randn(32, d)).astype(f32), None, None


def check_table(net, out, theta_rows, noise, tab, x0, what):
    """out within the referee bound on the active slots, untouched elsewhere; the three wrong referees rejected."""
    n = len(tab["idx"])
    on = np.arange(n) if tab["active"] is None else np.flatnonzero(tab["active"])
    if tab["active"] is not None:
        assert (out[tab["active"] == 0] == 123.0).all(), f"{what}: inactive slot written"
    ref, bound = referee_table(net, theta_rows, noise, tab, x0)
    bad = violations(out, ref, bound, on)
    worst = (np.abs(out[on] - ref[on]) / bound[on]).max()
    assert bad == 0, f"{what}: {bad} outputs outside the bound (worst error / bound = {worst:.3g})"
    # sharpness: the same comparison rejects deliberately wrong referees
    wrong = {"noise index + 1": dict(idx_shift=1), "last row of the first layer dropped": dict(drop=0)}
    if tab["n_theta"] > 1:
        wrong["wrong parent row"] = dict(row_shift=1)
    for why, kw in wrong.items():
        r, b = referee_table(net, theta_rows, noise, tab, x0, **kw)
        assert violations(out, r, b, on) > 0, f"{what}: the bound does not reject a referee with the {why}"
    return worst


@pytest.mark.parametrize("shape", list(SHAPES))
def test_shape_sweep_against_float64_referee(ctx, host_noise, shape):
    net = make_shape(shape)
    rs = np.random.RandomState(1000 + list(SHAPES).index(shape))
    obs_all, mean, std = shape_data(rs, net)
    worst = {}
    for tname, tab in tables(rs, net.num_params).items():
        n = len(tab["idx"])
        theta_rows = init_theta(rs, net, tab["n_theta"])
        obs = obs_all[:n]
        x0 = normalise(obs, mean, std)
        out = run_mlp(ctx, net, theta_rows, tab, obs, mean, std)
        worst[tname] = check_table(net, out, theta_rows, host_noise, tab, x0, f"{shape}/{tname}")
        if tname == "paired":
            # reruns are bit-identical; the unfused head and the unfolded theta partials stay within the bound
            np.testing.assert_array_equal(run_mlp(ctx, net, theta_rows, tab, obs, mean, std), out)
            for opt in ("fuse_head", "fold_theta"):
                set_option(opt, 0)
                alt = run_mlp(ctx, net, theta_rows, tab, obs, mean, std)
                set_option(opt, 1)
                check_table(net, alt, theta_rows, host_noise, tab, x0, f"{shape}/{tname}/{opt}=0")
    print(shape, {k: f"{v:.2g}" for k, v in worst.items()})


def test_classifier_observations_are_not_clipped(ctx, host_noise):
    """Without statistics the engine feeds observations as they are (models/simple.py has no normalisation)."""
    net = make_shape("linear_classifier")
    rs = np.random.RandomState(3)
    theta = init_theta(rs, net, 1)
    obs = np.array([[7.0, -9.5, 0.25, 40.0], [-6.0, 5.5, -100.0, 1.0]], f32)
    tab = dict(idx=np.zeros(2, np.int64), scale=np.zeros(2, f32), paired=0, theta_idx=None, active=None, n_theta=1)
    out = run_mlp(ctx, net, theta, tab, obs, None, None)
    W = theta[0, :8].astype(f64).reshape(4, 2)
    want = obs.astype(f64) @ W + theta[0, 8:10]
    np.testing.assert_allclose(out, want, rtol=1e-5)


# ---- argmax rule of both head kernels ------------------------------------------------------------------------------
def _argmax_rows(rs, A):
    nan, inf = f32(np.nan), f32(np.inf)
    rows = []
    rows.append(np.full(A, 0.7, f32))                                        # all equal
    r = rs.uniform(-1, 0, A).astype(f32)
    r[A // 3] = r[A - 1] = 2.0                                               # a tie for the maximum
    rows.append(r)
    r = rs.uniform(-1, 1, A).astype(f32)
    r[A // 2] = nan                                                          # one NaN
    rows.append(r)
    r = rs.uniform(-1, 1, A).astype(f32)
    r[A - 1] = nan
    r[A // 2] = nan                                                          # two NaNs
    rows.append(r)
    r = rs.uniform(-1, 1, A).astype(f32)
    r[0] = inf
    r[A - 1] = nan                                                           # +inf, then NaN
    rows.append(r)
    r = rs.uniform(-1, 1, A).astype(f32)
    r[A - 1] = inf
    r[A // 2] = nan                                                          # NaN, then +inf
    rows.append(r)
    rows.append(np.full(A, -inf, f32))                                       # all -inf
    r = rs.uniform(-1, 1, A).astype(f32)
    r[: A // 2] = -inf                                                       # -inf before finite values
    rows.append(r)
    return np.stack(rows)


@pytest.mark.parametrize("fuse_head", [1, 0])
@pytest.mark.parametrize("A", [1, 3, 4, 18])
def test_argmax_rule_of_both_head_kernels(ctx, A, fuse_head):
    """Model (Atari): zero head weights, per-row head biases => logits == biases exactly; actions == np.argmax (first
    maximum, the first NaN counts as the maximum)."""
    net = N.make_net("Model", num_actions=A)
    P = net.num_params
    head = net.layers[-1]
    rs = np.random.RandomState(A)
    biases = _argmax_rows(rs, A)
    n = len(biases)
    theta = (rs.randn(n, P) * 0.05).astype(f32)
    theta[:, head.off_w:head.off_w + head.cin * A] = 0.0
    theta[:, head.off_b:head.off_b + A] = biases
    set_option("fuse_head", fuse_head)
    sf = SlotForward(ctx, net, n)
    sf.set_slots(rs.randint(0, NOISE_COUNT - P + 1, size=n).astype(np.int64), np.zeros(n, f32),
                 theta_idx=np.arange(n, dtype=np.int32))
    sf.actions.fill_(-7)
    obs = cuda(rs.randint(0, 256, size=(n, 84, 84, 4)).astype(np.uint8))
    actions = sf.forward(cuda(theta), obs, paired=False).cpu().numpy()
    logits = sf.logits.cpu().numpy()
    np.testing.assert_array_equal(np.isnan(logits), np.isnan(biases))
    fin = ~np.isnan(biases)
    np.testing.assert_array_equal(logits[fin].view(np.uint32), biases[fin].view(np.uint32))
    np.testing.assert_array_equal(actions, np.argmax(biases, axis=1))


def test_head_wider_than_256_with_argmax_is_unsupported(ctx):
    net = N.make_net("Model", num_actions=300)
    sf = SlotForward(ctx, net, 2)
    with pytest.raises(F.DneError, match="not supported"):
        sf.forward(cuda(np.zeros(net.num_params, f32)), cuda(np.zeros((2, 84, 84, 4), np.uint8)), paired=False)


# ---- options that must not change a bit ------------------------------------------------------------------------------
def _largemodel_table(rs, P, n_slots=256, n_pairs=125):
    pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots // 2).astype(np.int64)
    for a in range(4):
        pidx[a] = (pidx[a] // 4) * 4 + a
    active = np.zeros(n_slots, np.uint8)
    active[:2 * n_pairs] = 1
    return np.repeat(pidx, 2), np.tile([0.005, -0.005], n_slots // 2).astype(f32), active


def _crowded(rs, P, n_pairs=12):
    hi = NOISE_COUNT - P
    c = int(rs.randint(0, hi - 2000))
    pidx = [c + 7 * i for i in range(n_pairs - 4)] + rs.randint(0, hi + 1, size=4).tolist()
    return np.repeat(np.array(pidx, np.int64), 2), np.tile([0.005, -0.005], n_pairs).astype(f32), None


@pytest.fixture(scope="module")
def option_tables():
    out = {}
    rs = np.random.RandomState(77)
    net = N.make_net("LargeModel")
    idx, scale, active = _largemodel_table(rs, net.num_params)
    out["LargeModel"] = dict(net=net, idx=idx, scale=scale, active=active,
                             theta=(rs.randn(net.num_params) * 0.05).astype(f32),
                             obs=rs.randint(0, 256, size=(256, 84, 84, 4)).astype(np.uint8), kw={})
    net = N.make_net("Model")
    idx, scale, active = _crowded(rs, net.num_params)
    out["Model"] = dict(net=net, idx=idx, scale=scale, active=active,
                        theta=(rs.randn(net.num_params) * 0.05).astype(f32),
                        obs=rs.randint(0, 256, size=(24, 84, 84, 4)).astype(np.uint8), kw={})
    net = make_shape("humanoid")
    tab = tables(rs, net.num_params)["paired"]
    obs, mean, std = shape_data(rs, net)
    out["Humanoid"] = dict(net=net, idx=tab["idx"], scale=tab["scale"], active=tab["active"],
                           theta=init_theta(rs, net, 1)[0], obs=obs[:26], kw=dict(ob_mean=mean, ob_std=std))
    return out


def _run(ctx, t):
    net, n = t["net"], len(t["idx"])
    sf = SlotForward(ctx, net, n)
    sf.set_slots(t["idx"], t["scale"], active=t["active"])
    sf.logits.fill_(123.0)
    sf.actions.fill_(-7)
    sf.forward(cuda(t["theta"]), cuda(t["obs"]), paired=True, **{k: cuda(v) for k, v in t["kw"].items()})
    torch.cuda.synchronize()
    return sf.logits.cpu().numpy(), sf.actions.cpu().numpy()


OPTION_SETS = [
    dict(gemv_ctas_per_sm=1, gemv_stages=8),      # 8 ring stages fit only at 1 CTA per SM
    dict(gemv_ctas_per_sm=2, gemv_stages=2),
    dict(gemv_ctas_per_sm=2, gemv_stages=3),
    dict(gemv_grid=7),
    dict(gemv_grid=1),
    dict(pdl=0),
]


@pytest.mark.parametrize("table", ["LargeModel", "Model", "Humanoid"])
def test_scheduling_options_are_bit_identical(ctx, option_tables, table):
    t = option_tables[table]
    base_logits, base_actions = _run(ctx, t)
    for opts in OPTION_SETS:
        if opts.get("gemv_grid") == 1 and table == "LargeModel":
            continue                                  # one CTA streaming 125 slices: covered by the smaller tables
        for k, v in opts.items():
            set_option(k, v)
        logits, actions = _run(ctx, t)
        for k in opts:
            set_option(k, DEFAULTS[k])
        np.testing.assert_array_equal(logits, base_logits, err_msg=str(opts))
        np.testing.assert_array_equal(actions, base_actions, err_msg=str(opts))


@pytest.mark.parametrize("table", ["LargeModel", "Model"])
def test_unfused_head_and_unfolded_theta_stay_within_the_forward_bound(ctx, option_tables, table):
    """fuse_head = 0 (dense_small_kernel head) and fold_theta = 0 add the same products in another order: within the
    forward tolerance of the conv policies (tests/test_gpu_scale.py), actions equal wherever the top two logits are
    apart by more than that.  (The MLP shapes check both options against the float64 referee.)"""
    t = option_tables[table]
    base_logits, base_actions = _run(ctx, t)
    on = np.arange(len(t["idx"])) if t["active"] is None else np.flatnonzero(t["active"])
    bl = base_logits[on]
    bound = 2e-5 * np.maximum(1.0, np.abs(bl).max(axis=1))
    srt = np.sort(bl, axis=1)
    decided = (srt[:, -1] - srt[:, -2]) > 2 * bound
    for opt in ("fuse_head", "fold_theta"):
        set_option(opt, 0)
        logits, actions = _run(ctx, t)
        set_option(opt, 1)
        assert (np.abs(logits[on] - bl).max(axis=1) <= bound).all(), opt
        np.testing.assert_array_equal(actions[on][decided], base_actions[on][decided], err_msg=opt)


@pytest.mark.parametrize("n_slots", [256, 128])
def test_theta_multicast_is_bit_identical(ctx, option_tables, n_slots):
    """theta_mc = 1: the TMA-fed theta GEMM (prepared theta) with the cluster-multicast A operand."""
    t = dict(option_tables["LargeModel"])
    t["idx"], t["scale"], t["obs"] = t["idx"][:n_slots], t["scale"][:n_slots], t["obs"][:n_slots]
    t["active"] = t["active"][:n_slots]
    base = _run(ctx, t)
    set_option("theta_mc", 1)
    got = _run(ctx, t)
    np.testing.assert_array_equal(got[0], base[0])
    np.testing.assert_array_equal(got[1], base[1])


def _four_ticks(ctx, t, chain):
    """4 ticks back to back on one stream after one dne_theta_prepare, through the raw C ABI: a distinct observation
    buffer and a distinct logits / actions buffer per tick, no other work on the stream in between."""
    net, n = t["net"], len(t["idx"])
    L = F.lib()
    sf = SlotForward(ctx, net, n)
    sf.set_slots(t["idx"], t["scale"], active=t["active"])
    theta = cuda(t["theta"])
    rs = np.random.RandomState(5)
    obs = [cuda(t["obs"])] + [cuda(rs.randint(0, 256, size=(n, 84, 84, 4)).astype(np.uint8)) for _ in range(3)]
    logits = [torch.full((n, net.n_out), 123.0, device=DEV) for _ in range(4)]
    actions = [torch.full((n,), -7, dtype=torch.int32, device=DEV) for _ in range(4)]
    set_option("chain_ticks", chain)
    sf.prepare(theta, n)
    torch.cuda.synchronize()
    for k in range(4):
        F.check(L.dne_perturb_forward_conv(
            ctx.handle, C.byref(net.desc), F.ptr(theta), F.ptr(sf.noise_idx), F.ptr(sf.scale), None, F.ptr(sf.active), n, 1,
            F.ptr(obs[k]), None, F.ptr(actions[k]), F.ptr(logits[k]), F.ptr(sf.ws), sf.ws.numel(), F.stream_ptr()))
    torch.cuda.synchronize()
    set_option("chain_ticks", 0)
    return [x.cpu().numpy() for x in logits], [a.cpu().numpy() for a in actions]


def test_chained_ticks_are_bit_identical(ctx, option_tables):
    t = option_tables["LargeModel"]
    base_l, base_a = _four_ticks(ctx, t, 0)
    got_l, got_a = _four_ticks(ctx, t, 1)
    for k in range(4):
        np.testing.assert_array_equal(got_l[k], base_l[k], err_msg=f"tick {k}")
        np.testing.assert_array_equal(got_a[k], base_a[k], err_msg=f"tick {k}")
    assert not np.array_equal(base_l[0], base_l[1])          # the ticks really saw different observations


# ---- the policy classes end to end -----------------------------------------------------------------------------------
def test_mujoco_policy_uniform16_head_acts_like_the_referee(ctx, host_noise):
    """Humanoid-sized MujocoPolicy with 'uniform:16' bins: a 256 x 272 head, per action dimension the argmax bin."""
    from dne.envs import Box
    from es_distributed import policies
    ob = Box(-np.inf, np.inf, (376,))
    ac = Box(-0.4, 0.4, (17,))
    pol = policies.MujocoPolicy(ob, ac, ac_bins="uniform:16", ac_noise_std=0.0, nonlin_type="tanh", hidden_dims=[256, 256],
                                connection_type="ff", ctx=ctx, seed=1)
    assert pol.net.n_out == 272
    rs = np.random.RandomState(9)
    mean, std = rs.randn(376).astype(f32), (np.abs(rs.randn(376)) + 0.2).astype(f32)
    obs = (mean + std * 2.5 * rs.randn(6, 376)).astype(f32)
    pol.set_ob_stat(mean, std)
    theta = pol.get_trainable_flat()
    w, wm = member(theta[None, :], 0, host_noise, 0, 0.0, pol.num_params)
    x0 = normalise(obs, mean, std)
    scores = pol._forward_noiseless(obs)
    for s in range(len(obs)):
        ref, bound = referee(pol.net, w, wm, x0[s])
        assert (np.abs(scores[s] - ref) <= bound).all()
        ref_b = ref.reshape(17, 16)
        srt = np.sort(ref_b, axis=1)
        decided = srt[:, -1] - srt[:, -2] > 2 * bound.reshape(17, 16).max(axis=1)
        want = pol._bin_values[np.arange(17), np.argmax(ref_b, axis=1)]
        got = pol.act(obs[s:s + 1])[0]
        np.testing.assert_array_equal(got[decided], want[decided])
        assert decided.mean() > 0.5


def test_mujoco_policy_clips_before_its_first_set_ob_stat(ctx):
    from dne.envs import Box
    from es_distributed import policies
    pol = policies.MujocoPolicy(Box(-np.inf, np.inf, (11,)), Box(-1.0, 1.0, (3,)), ac_bins="continuous:", ac_noise_std=0.0,
                                nonlin_type="tanh", hidden_dims=[64, 64], connection_type="ff", ctx=ctx, seed=2)
    np.testing.assert_array_equal(pol.ob_mean.cpu().numpy(), np.zeros(11, f32))
    np.testing.assert_array_equal(pol.ob_std.cpu().numpy(), np.ones(11, f32))
    obs = (9.0 * np.random.RandomState(4).randn(4, 11)).astype(f32)
    np.testing.assert_array_equal(pol.act(obs), pol.act(np.clip(obs, -5, 5)))
    assert not np.array_equal(pol.act(obs), pol.act(obs * 0.5))


def test_simple_classifier_policy_acts_on_unclipped_observations(ctx, host_noise):
    from dne.envs import Box, Discrete
    from es_distributed import policies
    pol = policies.SimpleClassifierPolicy(Box(-np.inf, np.inf, (4,)), Discrete(2), ctx=ctx, seed=5)
    rs = np.random.RandomState(6)
    obs = (12.0 * rs.randn(64, 4)).astype(f32)
    theta = pol.get_trainable_flat()
    w, wm = member(theta[None, :], 0, host_noise, 0, 0.0, pol.num_params)
    logits = pol._forward_noiseless(obs)
    ref, bound = zip(*[referee(pol.net, w, wm, o) for o in obs])
    ref, bound = np.array(ref), np.array(bound)
    assert (np.abs(logits - ref) <= bound).all(), np.abs(logits - ref).max()
    decided = np.abs(ref[:, 0] - ref[:, 1]) > 2 * bound.max(axis=1)
    np.testing.assert_array_equal(pol.act(obs)[decided], np.argmax(ref, axis=1)[decided])
