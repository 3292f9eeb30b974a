"""The once-per-generation kernels at the sizes production runs them, against float64 referees: the ES gradient on both
of its template paths and through its tile remainder (csrc/update_kernels.cu), the Adam / SGD steps past their
grid-stride boundary and their update ratio over more than 256 block partials, k-NN novelty on vector and uint8
behaviour characterisations (BCs) with archives past one CTA's width (csrc/ga_ns_kernels.cu), and the observation
statistics (csrc/forward_kernels.cu).  The C ABI is called directly, so t, denom, accumulate and the workspace pointer
are the test's choice.

Dispatch boundaries come from the device's SM count (printed by test_dispatch_boundaries and shown in the test ids):
  * dne_es_grad runs es_grad_kernel<4,4> when cdiv(P, 1024) >= 16 * SMs, so P_THR = (16 * SMs - 1) * 1024 is the
    largest P on <1,8> and P_THR + 1 the smallest on <4,4>;
  * dne_adam_step / dne_sgd_step launch at most 8 * SMs blocks of 256, so P > C = 8 * SMs * 256 runs the grid-stride
    loop, and ratio_finalize_kernel reduces 8 * SMs > 256 partials from P > 256 * 256 on.

Bounds (stated once):
  * ES gradient: |g_j - r_j| <= 2^-24 |r_j| + 1e-12 S_j, r_j = sum_i w_i eps[idx_i + j] / denom in float64 and
    S_j = sum_i |w_i eps[idx_i + j]| / |denom|: one float32 rounding plus float64 reassociation slack;
  * optimizer theta, m, v: bit-exact against the float32 oracle; update ratio within 2 float32 ulp of
    sqrt(sum step^2) / sqrt(sum theta_old^2) in float64;
  * novelty: within 1 float32 ulp of a float64 referee, NaN and inf in the same places;
  * observation sums: bit-exact (float64 adds in slot order); sums of squares rtol 1e-13 (v * v may be fused).
"""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from oracle import oracle as O            # noqa: E402  (checker only)
from dne import _ffi as F                 # noqa: E402
from dne.engine import make_context       # noqa: E402
from dne.noise import SharedNoiseTable    # noqa: E402

DEV = torch.device("cuda", 0)
NOISE_COUNT = 12_000_000
SMS = torch.cuda.get_device_properties(0).multi_processor_count
P_THR = (16 * SMS - 1) * 1024             # largest P on es_grad_kernel<1,8>
OPT_C = 8 * SMS * 256                     # largest P the optimizer grid covers with one element per thread
P_LARGE = 4_052_658                       # LargeModel, the benchmarked net
L2 = 0.005


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def table(host_noise):
    return SharedNoiseTable(host_noise=host_noise, device=DEV)


@pytest.fixture(scope="module")
def ctx(table):
    return make_context(0, table)


def cuda(x):
    return torch.as_tensor(np.ascontiguousarray(x)).to(DEV).contiguous()


def _cdiv(a, b):
    return -(-a // b)


def test_dispatch_boundaries():
    print(f"SMs={SMS} P_thr={P_THR} C={OPT_C}")
    assert _cdiv(P_THR, 1024) < 16 * SMS <= _cdiv(P_THR + 1, 1024)
    assert P_LARGE > P_THR + 1 and P_LARGE > OPT_C + 1          # the benchmark net is on <4,4> and the stride loop
    assert 8 * SMS > 256                                         # ratio_finalize: several partials per thread


# ---- ES gradient -----------------------------------------------------------------------------------------------------
def _grad_jpt(P):
    return 4 if _cdiv(P, 1024) >= 16 * SMS else 1


def _proc(rs, n):
    """Processed returns [n, 2] whose float32 differences w include zeros and magnitudes 1e-3 .. 1e3 of both signs."""
    base = rs.randn(n).astype(np.float32)
    w = (np.where(rs.rand(n) < 0.5, -1.0, 1.0) * 10.0 ** rs.uniform(-3, 3, n)).astype(np.float32)
    w[rs.rand(n) < 0.1] = 0
    w[:4] = [0, 1e-3, -1e3, 1][:min(n, 4)]
    return np.stack([base + w, base], axis=1).astype(np.float32)


def _slots(rs, n, P):
    """Noise offsets: the first and last legal ones, repeats (also across the 512-slice tile boundary), and starts of
    every alignment."""
    hi = NOISE_COUNT - P
    r = int(rs.randint(0, hi - 2)) // 4 * 4
    idx = rs.randint(0, hi + 1, size=n).astype(np.int64)
    special = [0, hi, r, r, r + 1, r + 3, hi, r + 2]
    idx[:min(n, len(special))] = special[:n]
    if n > 600:
        idx[511] = idx[512] = r + 1
    return idx


def _es_grad(ctx, proc, idx, P, denom, g, accumulate=0):
    n = len(idx)
    d_proc = cuda(proc if n else np.zeros((1, 2), np.float32))      # n = 0 still passes valid pointers
    d_idx = cuda(idx if n else np.zeros(1, np.int64))
    F.check(F.lib().dne_es_grad(ctx.handle, F.ptr(d_proc, torch.float32), F.ptr(d_idx, torch.int64), n, P,
                                float(denom), F.ptr(g, torch.float32), int(accumulate), F.stream_ptr()))
    torch.cuda.synchronize()
    return g


def _referee(table, proc, idx, P):
    """(sum_i w_i eps[idx_i + j], sum_i |w_i eps[idx_i + j]|) over all j, in float64 with torch's own elementwise ops,
    one slice at a time in index order."""
    noise = table.device_tensor
    w = (proc[:, 0] - proc[:, 1]).astype(np.float32)                # es.py:292, float32
    r = torch.zeros(P, dtype=torch.float64, device=DEV)
    s = torch.zeros_like(r)
    for wi, i in zip(w.tolist(), idx.tolist()):
        x = noise[i:i + P].double()
        r.add_(x, alpha=wi)
        s.add_(x.abs_(), alpha=abs(wi))
    return r, s


def _check_grad(g, r, s, denom, g0=None):
    """Every column within one float32 rounding of the referee (two when adding onto g0) plus reassociation slack."""
    ref = r / denom
    slack = 1e-12 * (s / abs(denom))
    got = g.double()
    if g0 is None:
        bound = 2.0 ** -24 * ref.abs() + slack
    else:
        bound = 2.0 ** -24 * ((g0.double() + ref).abs() + ref.abs()) + slack
        ref = g0.double() + ref
    err = (got - ref).abs()
    bad = ~(err <= bound)                                            # NaN (a column never written) is bad too
    if bool(bad.any()):
        j = int(bad.nonzero()[0, 0])
        raise AssertionError(f"{int(bad.sum())} columns out of bound; first j={j}: g={float(got[j])!r} "
                             f"ref={float(ref[j])!r} bound={float(bound[j])!r}")


def _pin_ranges(P):
    """Column ranges pinned on the host: the first CTA, the whole last CTA, and the columns == 0, 255 (mod 256) of three
    CTAs in between."""
    W = 256 * _grad_jpt(P)
    nct = _cdiv(P, W)
    ranges = [(0, min(P, W)), ((nct - 1) * W, P)]
    for c in sorted({nct // 3, nct // 2, 2 * nct // 3} - {0, nct - 1}):
        for b in range(c * W, (c + 1) * W, 256):
            ranges += [(b, b + 1), (b + 255, b + 256)]
    return ranges


def _pin_referee(host_noise, proc, idx, P, r, s):
    """The device referee against the oracle's float64 es_gradient (es.py:291-296, denom = 2n) on sampled columns: the
    oracle of a column range [a, b) is es_gradient over the slices shifted by a."""
    denom = proc.size
    for a, b in _pin_ranges(P):
        ref = O.es_gradient(proc, host_noise, idx + a, b - a, dtype=np.float64)
        got = r[a:b].cpu().numpy() / denom
        tol = 1e-12 * s[a:b].cpu().numpy() / denom
        assert (np.abs(got - ref) <= tol).all(), (a, b, np.abs(got - ref).max())


def _grad_case(ctx, table, host_noise, P, n, seed):
    rs = np.random.RandomState(seed)
    proc, idx = _proc(rs, n), _slots(rs, n, P)
    g = _es_grad(ctx, proc, idx, P, 2 * n, torch.full((P,), float("nan"), device=DEV))
    r, s = _referee(table, proc, idx, P)
    _check_grad(g, r, s, 2 * n)
    _pin_referee(host_noise, proc, idx, P, r, s)
    again = _es_grad(ctx, proc, idx, P, 2 * n, torch.full((P,), float("nan"), device=DEV))
    assert torch.equal(g, again)                                     # fixed summation order: bit-identical


@pytest.mark.parametrize("n", [7, 513, 2500])
@pytest.mark.parametrize("P", [pytest.param(P_THR, id=f"P_thr={P_THR}"),
                               pytest.param(P_THR + 1, id=f"P_thr+1={P_THR + 1}"),
                               pytest.param(P_LARGE, id=f"P={P_LARGE}")])
def test_es_grad_wide_vs_float64_referee(ctx, table, host_noise, P, n):
    """Both template paths at and around their boundary and at LargeModel's width.  n = 7 is all remainder,
    513 one full 512-slice tile plus one, 2500 five tiles with a tail of 452."""
    _grad_case(ctx, table, host_noise, P, n, seed=P % 997 + n)


@pytest.mark.parametrize("P", [1, 255, 257])
def test_es_grad_narrow_vs_float64_referee(ctx, table, host_noise, P):
    _grad_case(ctx, table, host_noise, P, 1203, seed=P)


@pytest.mark.parametrize("P", [pytest.param(P_THR, id=f"P_thr={P_THR}"),
                               pytest.param(P_THR + 1, id=f"P_thr+1={P_THR + 1}")])
def test_es_grad_shard_denominator_and_accumulate(ctx, table, P):
    """A shard's partial gradient: denom is the whole generation's returns_n2.size, not 2n, and accumulate = 1 adds it
    onto a non-zero g."""
    rs = np.random.RandomState(P % 991)
    n, n_global = 600, 1500
    proc, idx = _proc(rs, n), _slots(rs, n, P)
    r, s = _referee(table, proc, idx, P)
    g = _es_grad(ctx, proc, idx, P, 2 * n_global, torch.full((P,), float("nan"), device=DEV))
    _check_grad(g, r, s, 2 * n_global)
    g0 = cuda((rs.randn(P) * 0.1).astype(np.float32))
    g = _es_grad(ctx, proc, idx, P, 2 * n_global, g0.clone(), accumulate=1)
    _check_grad(g, r, s, 2 * n_global, g0=g0)


@pytest.mark.parametrize("P", [257, pytest.param(P_THR + 1, id=f"P_thr+1={P_THR + 1}")])
def test_es_grad_no_slices(ctx, P):
    """n = 0 writes zeros, or leaves g as it was with accumulate."""
    g0 = cuda((np.random.RandomState(3).randn(P) * 0.1 + 1.0).astype(np.float32))
    g = _es_grad(ctx, np.zeros((0, 2), np.float32), np.zeros(0, np.int64), P, 2.0, g0.clone(), accumulate=1)
    assert torch.equal(g, g0)
    g = _es_grad(ctx, np.zeros((0, 2), np.float32), np.zeros(0, np.int64), P, 2.0, g0.clone())
    assert bool((g == 0).all())


# ---- Adam / SGD --------------------------------------------------------------------------------------------------------
class _Opt:
    """One optimizer on the device beside its float32 oracle (optimizers.py), stepped through the C ABI."""

    def __init__(self, ctx, kind, theta, **kw):
        self.ctx, self.kind, self.kw = ctx, kind, kw
        self.orc = O.Adam(theta, **kw) if kind == "adam" else O.SGD(theta, **kw)
        self.theta = cuda(theta)
        self.m = torch.zeros_like(self.theta) if kind == "adam" else None
        self.v = torch.zeros_like(self.theta)
        self.ratio = torch.full((1,), float("nan"), device=DEV)

    def device_step(self, d_g, t, with_ratio=True):
        L, P, kw = F.lib(), self.theta.numel(), self.kw
        ratio = F.ptr(self.ratio) if with_ratio else None
        if self.kind == "adam":
            F.check(L.dne_adam_step(self.ctx.handle, F.ptr(self.theta), F.ptr(self.m), F.ptr(self.v), F.ptr(d_g), P, L2,
                                    kw["stepsize"], kw.get("beta1", 0.9), kw.get("beta2", 0.999),
                                    kw.get("epsilon", 1e-8), t, ratio, F.stream_ptr()))
        else:
            F.check(L.dne_sgd_step(self.ctx.handle, F.ptr(self.theta), F.ptr(self.v), F.ptr(d_g), P, L2,
                                   kw["stepsize"], kw.get("momentum", 0.9), ratio, F.stream_ptr()))
        torch.cuda.synchronize()
        return float(self.ratio.cpu()[0])

    def oracle_step(self, g):
        """The oracle's update; returns its float32 step (optimizers.py:31 / :49, restated on the oracle's new state) and
        the float64 referee of the update ratio."""
        orc = self.orc
        theta_old = orc.theta.copy()
        orc.update(O.es_update_direction(g, orc.theta, L2))
        if self.kind == "adam":
            step = (-np.float32(orc.step_scale())) * orc.m / (np.sqrt(orc.v) + np.float32(orc.epsilon))
        else:
            step = np.float32(-orc.stepsize) * orc.v
        np.testing.assert_array_equal((theta_old + step).astype(np.float32), orc.theta)   # the restatement is the oracle's
        s64, t64 = step.astype(np.float64), theta_old.astype(np.float64)
        return math.sqrt(float(np.dot(s64, s64))) / math.sqrt(float(np.dot(t64, t64)))

    def assert_state_equal(self):
        np.testing.assert_array_equal(self.theta.cpu().numpy(), self.orc.theta)
        np.testing.assert_array_equal(self.v.cpu().numpy(), self.orc.v)
        if self.kind == "adam":
            np.testing.assert_array_equal(self.m.cpu().numpy(), self.orc.m)


def _nonzero(x):
    x = x.astype(np.float32)
    x[x == 0] = 0.25
    return x


def _assert_ratio(got, ref):
    ulp = float(np.spacing(np.float32(ref)))
    assert abs(got - ref) <= 2 * ulp, (got, ref, (got - ref) / ulp)


def _run_steps(opt, rs, P, steps=3):
    for _ in range(steps):
        g = _nonzero(rs.randn(P) * 0.01)
        ref = opt.oracle_step(g)
        got = opt.device_step(cuda(g), opt.orc.t)
        opt.assert_state_equal()
        _assert_ratio(got, ref)


OPT_SIZES = [1, 257, pytest.param(OPT_C, id=f"C={OPT_C}"), pytest.param(OPT_C + 1, id=f"C+1={OPT_C + 1}"),
             pytest.param(P_LARGE, id=f"P={P_LARGE}")]


@pytest.mark.parametrize("P", OPT_SIZES)
@pytest.mark.parametrize("kind", ["adam", "sgd"])
def test_optimizer_bit_exact_and_ratio(ctx, kind, P):
    rs = np.random.RandomState(P % 983)
    kw = dict(stepsize=0.01) if kind == "adam" else dict(stepsize=0.01, momentum=0.9)
    _run_steps(_Opt(ctx, kind, _nonzero(rs.randn(P) * 0.1), **kw), rs, P)


def test_adam_bias_correction_underflow(ctx):
    """t = 10^6: beta1^t and beta2^t underflow to 0 in float64, so the step scale is the step size itself."""
    P = OPT_C + 1
    rs = np.random.RandomState(5)
    opt = _Opt(ctx, "adam", _nonzero(rs.randn(P) * 0.1), stepsize=0.01)
    opt.orc.t = 10 ** 6 - 1
    _run_steps(opt, rs, P, steps=2)
    assert opt.orc.step_scale() == 0.01


@pytest.mark.parametrize("kind,kw", [("adam", dict(stepsize=0.03, beta1=0.8, beta2=0.95, epsilon=1e-5)),
                                     ("sgd", dict(stepsize=0.03, momentum=0.5))])
def test_optimizer_non_default_hyperparameters(ctx, kind, kw):
    P = OPT_C + 1
    rs = np.random.RandomState(6)
    _run_steps(_Opt(ctx, kind, _nonzero(rs.randn(P) * 0.1), **kw), rs, P)


@pytest.mark.parametrize("kind", ["adam", "sgd"])
def test_optimizer_rerun_bit_identical_and_ratio_optional(ctx, kind):
    """Two steps from the same state give the same theta and the same ratio bit for bit (fixed reduction order); a
    NULL update-ratio pointer is accepted and changes nothing else."""
    P = P_LARGE
    rs = np.random.RandomState(7)
    kw = dict(stepsize=0.01) if kind == "adam" else dict(stepsize=0.01, momentum=0.9)
    opt = _Opt(ctx, kind, _nonzero(rs.randn(P) * 0.1), **kw)
    _run_steps(opt, rs, P, steps=1)
    saved = [t.clone() for t in (opt.theta, opt.m, opt.v) if t is not None]
    g = cuda(_nonzero(rs.randn(P) * 0.01))
    outs = []
    for with_ratio in (True, True, False):
        for t, s in zip([t for t in (opt.theta, opt.m, opt.v) if t is not None], saved):
            t.copy_(s)
        opt.ratio.fill_(float("nan"))
        ratio = opt.device_step(g, 2, with_ratio=with_ratio)
        outs.append((ratio, [t.clone() for t in (opt.theta, opt.m, opt.v) if t is not None]))
    assert np.float32(outs[0][0]).tobytes() == np.float32(outs[1][0]).tobytes()
    assert math.isnan(outs[2][0])                                    # nothing written through a NULL ratio
    for a, b in zip(outs[0][1], outs[1][1]):
        assert torch.equal(a, b)
    for a, b in zip(outs[0][1], outs[2][1]):
        assert torch.equal(a, b)
    opt.oracle_step(g.cpu().numpy())
    opt.assert_state_equal()


# ---- k-NN novelty ------------------------------------------------------------------------------------------------------
def _assert_novelty(got, ref):
    """Within 1 float32 ulp of the float64 referee; NaN and inf exactly where the referee has them."""
    got, ref = np.asarray(got), np.asarray(ref, dtype=np.float64)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(ref))
    inf = np.isinf(ref)
    np.testing.assert_array_equal(got[inf], ref[inf])
    fin = np.isfinite(ref)
    ulp = np.spacing(np.abs(ref[fin]).astype(np.float32)).astype(np.float64)
    err = np.abs(got[fin].astype(np.float64) - ref[fin])
    assert (err <= ulp).all(), (np.flatnonzero(fin)[err > ulp], (err / ulp).max())


def _knn_ref(dist, k):
    """nses.py:28-32: mean of the first k of a stable ascending sort (numpy sorts NaN last)."""
    return np.sort(dist, axis=1, kind="stable")[:, :k].mean(axis=1)


def _vec_dist(bc, ar):
    return np.sqrt(((bc[:, None, :] - ar[None, :, :]) ** 2).sum(axis=-1))


class _GuardedWs:
    """A k-NN workspace at a 256-byte-aligned interior offset of a larger buffer filled with a sentinel byte."""
    PAD = 512

    def __init__(self, q, A):
        nb = C.c_size_t()
        F.check(F.lib().dne_knn_ws_bytes(q, A, C.byref(nb)))
        self.nbytes, self.used = nb.value, q * A * 8
        self.buf = torch.full((self.PAD + nb.value + self.PAD,), 0xA5, dtype=torch.uint8, device=DEV)
        self.ptr = C.c_void_p(self.buf.data_ptr() + self.PAD)
        assert self.ptr.value % 256 == 0

    def assert_sentinel_intact(self):
        torch.cuda.synchronize()
        b = self.buf.cpu().numpy()
        assert (b[:self.PAD] == 0xA5).all(), "bytes before the workspace were written"
        assert (b[self.PAD + self.used:] == 0xA5).all(), "bytes after the workspace were written"


def _knn_vec(bc, ar, k, ws=None):
    """dne_knn_novelty_vec on a guarded workspace.  Checks that nothing outside the workspace was written, unless the
    caller passes its own ws and checks it later."""
    q, D = bc.shape
    A = ar.shape[0]
    own = ws is None
    ws = _GuardedWs(q, A) if own else ws
    d_bc, d_ar = cuda(bc), cuda(ar)
    nov = torch.full((q,), -7.0, device=DEV)
    F.check(F.lib().dne_knn_novelty_vec(F.ptr(d_bc, torch.float64), q, F.ptr(d_ar, torch.float64), A, D, k, F.ptr(nov),
                                        ws.ptr, ws.nbytes, F.stream_ptr()))
    if own:
        ws.assert_sentinel_intact()
    return nov.cpu().numpy()


def _vec_case(rs, q, A, D, with_inf=True):
    """Archive and queries with exact duplicates, integer-grid points (many equal distances), queries that are archive
    entries, and (with_inf) +-inf coordinates that give inf distances (never inf - inf)."""
    ar = rs.randn(A, D) * 3
    ar[A // 2:] = np.round(ar[A // 2:])
    if A >= 3:
        ar[1] = ar[A - 1] = ar[0]
    if with_inf and A >= 6:                                          # rows no query copies
        ar[3, D - 1] = np.inf
        ar[4, 0] = -np.inf
    bc = rs.randn(q, D) * 3
    bc[q // 2:] = np.round(bc[q // 2:])
    bc[0] = ar[0]
    if q > 3:
        bc[1] = ar[A - 1]
        bc[2] = ar[A // 2]
        if with_inf and D >= 2:
            bc[3, 0] = np.inf                                       # inf - (-inf): every distance is inf
    return bc, ar


@pytest.mark.parametrize("A", [1, 5, 255, 256, 257, 1000])
@pytest.mark.parametrize("D", [1, 2, 3, 17])
def test_knn_novelty_vec_vs_oracle(D, A):
    rs = np.random.RandomState(100 * D + A)
    for q in (1, 64):
        bc, ar = _vec_case(rs, q, A, D)
        dist = _vec_dist(bc, ar)
        for k in (1, 3, 10, A, A + 5):
            ref = _knn_ref(dist, k)
            for i in {0, q - 1}:                                     # the vectorised referee is the oracle's
                np.testing.assert_allclose(ref[i], O.compute_novelty_vs_archive(list(ar), bc[i], k), rtol=1e-13)
            _assert_novelty(_knn_vec(bc, ar, k), ref)


def test_knn_novelty_vec_nan_query():
    """A query BC with a NaN coordinate has novelty NaN.  Its selection stays inside its own row of the workspace: the
    sentinel around the workspace is unchanged, and every other query's novelty equals a run without the NaN rows bit
    for bit, including a neighbouring query whose nearest archive entry is the last one of its row."""
    rs = np.random.RandomState(21)
    q, A, D = 64, 300, 3
    bc, ar = _vec_case(rs, q, A, D)
    nan_rows = [0, 17, 40, 63]
    for r in nan_rows:
        if r > 0:
            bc[r - 1] = ar[A - 1]
        bc[r, r % D] = np.nan
    keep = np.setdiff1d(np.arange(q), nan_rows)
    for k in (1, 10, A):
        ws = _GuardedWs(q, A)
        got = _knn_vec(bc, ar, k, ws)
        assert np.isnan(got[nan_rows]).all(), got[nan_rows]
        ws.assert_sentinel_intact()
        clean = _knn_vec(bc[keep], ar, k)
        assert got[keep].tobytes() == clean.tobytes()
        _assert_novelty(got, _knn_ref(_vec_dist(bc, ar), k))


@pytest.mark.parametrize("A,nan_rows", [(5, [1, 4]), (300, [0, 1, 150, 255, 256, 298, 299])])
def test_knn_novelty_vec_nan_archive_entries_sort_last(A, nan_rows):
    """m archive entries with a NaN coordinate: the novelty is finite and equals a run without them bit for bit when
    A - m >= min(k, A), and NaN otherwise (numpy's sort puts NaN after every number)."""
    rs = np.random.RandomState(22 + A)
    q, D = 64, 2
    bc, ar = _vec_case(rs, q, A, D, with_inf=False)
    bc[0] = ar[nan_rows[0]]                                          # a query that was an archive entry before it broke
    for r in nan_rows:
        ar[r, r % D] = np.nan
    m = len(nan_rows)
    clean_ar = np.delete(ar, nan_rows, axis=0)
    dist = _vec_dist(bc, ar)
    for k in sorted({1, 3, A - m, A - m + 1, A, A + 5}):
        ws = _GuardedWs(q, A)
        got = _knn_vec(bc, ar, k, ws)
        if A - m >= min(k, A):
            assert np.isfinite(got).all(), (k, got)
            assert got.tobytes() == _knn_vec(bc, clean_ar, k).tobytes()
        else:
            assert np.isnan(got).all(), (k, got)
        ws.assert_sentinel_intact()
        _assert_novelty(got, _knn_ref(dist, k))
        for i in (0, q - 1):
            np.testing.assert_allclose(_knn_ref(dist[i:i + 1], k)[0], O.compute_novelty_vs_archive(list(ar), bc[i], k),
                                       rtol=1e-13)


def _u8_sqdist(qp, ql, ap, al):
    """Exact int64 sum over rows t < max(len_q, len_a) and all columns of (q - a)^2 on last-row-padded sequences."""
    t_max = qp.shape[1]
    qi, ai = qp.astype(np.int64), ap.astype(np.int64)
    rows = np.minimum(t_max, np.maximum(ql[:, None], al[None, :]))
    qsq, asq = (qi ** 2).sum(-1), (ai ** 2).sum(-1)
    total = np.zeros(rows.shape, dtype=np.int64)
    for t in range(t_max):
        d2 = qsq[:, t, None] + asq[None, :, t] - 2 * (qi[:, t] @ ai[:, t].T)
        total += np.where(t < rows, d2, 0)
    return total


def _u8_seqs(rs, n, t_max, D):
    lens = rs.randint(1, t_max + 1, size=n).astype(np.int32)
    lens[:2] = [1, t_max][:n]
    seqs = [rs.randint(0, 256, size=(t, D)).astype(np.uint8) for t in lens]
    return lens, seqs


def _pad(seqs, t_max):
    return np.stack([np.concatenate([s, np.repeat(s[-1:], t_max - len(s), 0)]) for s in seqs])


@pytest.mark.parametrize("A", [255, 256, 257, 1000])
def test_knn_novelty_u8_large_archive(A):
    """dne_knn_novelty with archives where each selection thread scans one or several entries; ragged lengths from 1 to
    t_max, an archive entry duplicated, and a query that is itself in the archive."""
    rs = np.random.RandomState(30 + A)
    q, t_max, D = 64, 60, 128
    ql, qs = _u8_seqs(rs, q, t_max, D)
    al, as_ = _u8_seqs(rs, A, t_max, D)
    al[A - 1], as_[A - 1] = ql[5], qs[5]
    al[A // 2], as_[A // 2] = al[7], as_[7]
    qp, ap = _pad(qs, t_max), _pad(as_, t_max)
    dist = np.sqrt(_u8_sqdist(qp, ql, ap, al).astype(np.float64))
    assert dist[5, A - 1] == 0 and dist[:, A // 2].tobytes() == dist[:, 7].tobytes()
    L = F.lib()
    ws = _GuardedWs(q, A)
    d_qp, d_ql, d_ap, d_al = cuda(qp), cuda(ql), cuda(ap), cuda(al)
    nov = torch.empty(q, dtype=torch.float32, device=DEV)
    for k in (1, 10, A):
        ref = _knn_ref(dist, k)
        for i in (0, 5, q - 1):
            np.testing.assert_allclose(ref[i], O.compute_novelty_vs_archive(as_, qs[i], k), rtol=1e-13)
        F.check(L.dne_knn_novelty(F.ptr(d_qp), F.ptr(d_ql), q, F.ptr(d_ap), F.ptr(d_al), A, t_max, D, k, F.ptr(nov),
                                  ws.ptr, ws.nbytes, F.stream_ptr()))
        torch.cuda.synchronize()
        _assert_novelty(nov.cpu().numpy(), ref)
        ws.assert_sentinel_intact()


# ---- observation statistics --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ob_dim", [1, 3, 376])
def test_ob_stat_accumulate_vs_float64(ob_dim):
    """Sums of listed observation rows (out of order, repeated) added onto preset non-zero float64 sums over successive
    calls; m = 0 leaves them untouched."""
    rs = np.random.RandomState(40 + ob_dim)
    n_rows = 512
    obs = (rs.randn(n_rows, ob_dim) * 10.0 ** rs.uniform(-2, 2, size=ob_dim)).astype(np.float32)
    ref_sum = rs.randn(ob_dim) * 100
    ref_sumsq = np.abs(rs.randn(ob_dim)) * 1e4 + 1e-2
    d_obs, d_sum, d_sumsq = cuda(obs), cuda(ref_sum), cuda(ref_sumsq)
    L = F.lib()
    for m in (0, 1, 300, 300):
        slots = rs.randint(0, n_rows, size=max(m, 1)).astype(np.int32)
        if m == 300:
            slots[:6] = [511, 3, 3, 0, 511, 3]
        d_slots = cuda(slots)
        F.check(L.dne_ob_stat_accumulate(F.ptr(d_obs), ob_dim, F.ptr(d_slots), m, F.ptr(d_sum), F.ptr(d_sumsq),
                                         F.stream_ptr()))
        a, b = np.zeros(ob_dim), np.zeros(ob_dim)
        for s in slots[:m]:
            v = obs[s].astype(np.float64)
            a += v
            b += v * v
        ref_sum, ref_sumsq = ref_sum + a, ref_sumsq + b
        got_sum, got_sumsq = d_sum.cpu().numpy(), d_sumsq.cpu().numpy()
        np.testing.assert_array_equal(got_sum, ref_sum)
        np.testing.assert_allclose(got_sumsq, ref_sumsq, rtol=1e-13, atol=0)
        if m == 0:
            np.testing.assert_array_equal(got_sumsq, ref_sumsq)
