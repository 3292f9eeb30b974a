"""GPU tests of the tensor-core (wgmma, 3xTF32 / 2 x fp16) convolution path against the oracle and against the
fp32 SIMT path, plus GA slots (per-slot parent rows) and a self-test of the wgmma plumbing."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
if not torch.cuda.is_available():
    pytest.skip("needs a CUDA device", allow_module_level=True)

from oracle import oracle as O            # noqa: E402
from dne import _ffi as F                 # noqa: E402
from dne import nets as N                 # noqa: E402
from dne.engine import SlotForward, make_context   # noqa: E402
from dne.noise import SharedNoiseTable    # noqa: E402

DEV = torch.device("cuda", 0)
NOISE_COUNT = 6_000_000


@pytest.fixture(scope="module")
def host_noise():
    return O.noise_table(NOISE_COUNT)


@pytest.fixture(scope="module")
def ctx(host_noise):
    return make_context(0, SharedNoiseTable(host_noise=host_noise, device=DEV))


def cuda(x):
    return torch.as_tensor(np.ascontiguousarray(x)).to(DEV).contiguous()


@pytest.mark.parametrize("n,k", [(32, 256), (64, 512), (64, 576), (16, 256), (32, 32)])
def test_tcgen05_gemm_selftest(n, k):
    """C = A B^T through the hand-written wgmma path (smem descriptors, register accumulators, wgmma fence / commit /
    wait) with the 3xTF32 split: must be fp32-accurate, not TF32-accurate."""
    rs = np.random.RandomState(n * 1000 + k)
    A = rs.randn(128, k).astype(np.float32)
    B = rs.randn(n, k).astype(np.float32)
    dA, dB = cuda(A), cuda(B)
    dC = torch.full((128, n), float("nan"), dtype=torch.float32, device=DEV)
    F.check(F.dev_lib().dne_test_tc_gemm(F.ptr(dA), F.ptr(dB), F.ptr(dC), k, n, F.stream_ptr()))
    got = dC.cpu().numpy()
    ref = A.astype(np.float64) @ B.astype(np.float64).T
    scale = np.abs(ref).max()
    err = np.abs(got - ref).max()
    # plain TF32 would be ~1e-3 * scale; 3xTF32 leaves the tensor core's own fp32 accumulation error (not IEEE
    # round-to-nearest; measured 2e-6 * scale at K = 256), an order of magnitude inside the forward tolerance
    assert err <= 1e-5 * scale, (err, scale)


def _forward(ctx, net, theta, idx, scale, obs, paired, conv_tc, theta_idx=None):
    F.check(F.lib().dne_set_option(b"conv_tc", conv_tc))
    try:
        sf = SlotForward(ctx, net, len(idx))
        sf.set_slots(idx, scale, theta_idx=theta_idx)
        d_theta, d_obs = cuda(theta), cuda(obs)
        actions = sf.forward(d_theta, d_obs, paired=paired).cpu().numpy()
        return sf.logits.cpu().numpy(), actions
    finally:
        F.check(F.lib().dne_set_option(b"conv_tc", 2))


@pytest.mark.parametrize("name", ["LargeModel", "Model"])
def test_conv_tc_vs_simt_vs_oracle(ctx, host_noise, name):
    net, net_o = N.make_net(name), O.make_net(name)
    P = net.num_params
    rs = np.random.RandomState(5)
    theta = (rs.randn(P) * 0.05).astype(np.float32)
    n_slots = 6
    pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots // 2).astype(np.int64)
    idx, scale = np.repeat(pidx, 2), np.tile([0.02, -0.02], n_slots // 2).astype(np.float32)
    obs = rs.randint(0, 256, size=(n_slots, 84, 84, 4)).astype(np.uint8)
    l2, a2 = _forward(ctx, net, theta, idx, scale, obs, 1, 2)        # shifted-window wgmma + TMA (default)
    lt, at = _forward(ctx, net, theta, idx, scale, obs, 1, 1)        # im2col-staged wgmma
    ls, as_ = _forward(ctx, net, theta, idx, scale, obs, 1, 0)       # fp32 SIMT
    ref = np.stack([O.forward(net_o, O.perturb(theta, host_noise, int(idx[s]), 0.02, 1 if scale[s] > 0 else -1),
                              obs[s:s + 1])[0][0] for s in range(n_slots)])
    bound = 2e-5 * max(1.0, float(np.abs(ref).max()))
    assert np.abs(ls - ref).max() <= bound
    assert np.abs(lt - ref).max() <= bound, np.abs(lt - ref).max()
    assert np.abs(l2 - ref).max() <= bound, np.abs(l2 - ref).max()
    srt = np.sort(ref, axis=1)
    decided = (srt[:, -1] - srt[:, -2]) > 2 * bound
    np.testing.assert_array_equal(at[decided], np.argmax(ref, axis=1)[decided])
    np.testing.assert_array_equal(a2[decided], np.argmax(ref, axis=1)[decided])


def _s2d_geom(l):
    """Image geometry of a conv layer's INPUT on the shifted-window path (csrc/conv_s2d.cu: s2d_geom): planes of 8 fp16
    channels per pixel, groups of 16 channels = [h0 plane 0, h0 plane 1, h1 plane 0, h1 plane 1]."""
    hp = (l.hout - 1) * l.stride + l.ksize
    W = hp // l.stride
    cp = l.stride * l.stride * l.cin
    pixp = (W * W + 7) // 8 * 8
    return dict(S=l.stride, pad=l.pad, W=W, NG=cp // 16, PIXP=pixp, floats=(cp // 16) * 4 * pixp * 4)


def _decode_image(buf, l):
    """[NG][h0 / h1][2 channel octets][PIXP][8 x fp16] -> the NHWC activation [hin, hin, cin] it encodes
    (h0 + h1 * 2^-11), and the largest magnitude in the zero padding it must carry."""
    g = _s2d_geom(l)
    raw = buf[:g["floats"]].view(np.float16).reshape(g["NG"], 2, 2, g["PIXP"], 8).astype(np.float64)
    full = raw[:, 0] + raw[:, 1] / 2048.0                            # [NG][2][PIXP][8]
    chans = full.transpose(2, 0, 1, 3).reshape(g["PIXP"], g["NG"] * 16)[:g["W"] * g["W"]]     # [pixel][s2d channel]
    S, W = g["S"], g["W"]
    grid = chans.reshape(W, W, S, S, l.cin).transpose(0, 2, 1, 3, 4).reshape(W * S, W * S, l.cin)   # padded NHWC
    inner = grid[g["pad"]:g["pad"] + l.hin, g["pad"]:g["pad"] + l.hin]
    border = grid.copy()
    border[g["pad"]:g["pad"] + l.hin, g["pad"]:g["pad"] + l.hin] = 0
    return inner, float(np.abs(border).max())


@pytest.mark.parametrize("conv_tc", [2, 1])
def test_conv_tc_intermediate_activations(ctx, host_noise, conv_tc):
    """Layer-by-layer check of the tensor-core convolutions (conv3 output = the 7744-vector fed to the fc layer).
    conv_tc = 2: shifted-window kernels -- conv1 / conv2 write the NEXT layer's space-to-depth image (fp16 h0/h1 planes,
    zero padded), decoded here; conv_tc = 1: NHWC activations of the im2col-staged kernels."""
    net, net_o = N.make_net("LargeModel"), O.make_net("LargeModel")
    P = net.num_params
    rs = np.random.RandomState(8)
    theta = (rs.randn(P) * 0.05).astype(np.float32)
    idx = np.array([17, 17], dtype=np.int64)
    scale = np.array([0.02, -0.02], dtype=np.float32)
    obs = rs.randint(0, 256, size=(2, 84, 84, 4)).astype(np.uint8)
    F.check(F.lib().dne_set_option(b"conv_tc", conv_tc))
    try:
        sf = SlotForward(ctx, net, 2)
        sf.set_slots(idx, scale)
        d_theta, d_obs = cuda(theta), cuda(obs)
        sf.forward(d_theta, d_obs, paired=True)
        torch.cuda.synchronize()
    finally:
        F.check(F.lib().dne_set_option(b"conv_tc", 2))
    ws = sf.ws.view(torch.float32)
    off = 0
    for li, l in enumerate(net.layers[:3]):
        nxt = net.layers[li + 1]
        per_slot = max(l.out_elems, _s2d_geom(nxt)["floats"]) if nxt.kind == F.CONV else l.out_elems
        raw = ws[off:off + 2 * per_slot].cpu().numpy().reshape(2, per_slot)
        off += ((2 * per_slot * 4 + 255) // 256 * 256) // 4
        for s in range(2):
            th = O.perturb(theta, host_noise, 17, 0.02, 1 if s == 0 else -1)
            want = O.forward(net_o, th, obs[s:s + 1], return_all=True)[2][li][0]
            if conv_tc == 2 and nxt.kind == F.CONV:
                got, border = _decode_image(raw[s], nxt)
                assert border == 0.0, (li, s, border)
            else:
                got = raw[s][:l.out_elems].reshape(l.hout, l.hout, l.cout)
            assert np.abs(got - want).max() <= 2e-5 * max(1.0, np.abs(want).max()), (li, s, np.abs(got - want).max())


@pytest.mark.parametrize("paired", [0, 2])
def test_ga_slots_parent_rows(ctx, host_noise, paired):
    """GA offspring: theta[parent(slot)] + power*noise[seed(slot)] (models/base.py:148-156), per-slot parent rows.
    paired=2: slots (2p,2p+1) share the parent row (read once)."""
    net, net_o = N.make_net("LargeModel"), O.make_net("LargeModel")
    P = net.num_params
    rs = np.random.RandomState(31)
    parents = (rs.randn(3, P) * 0.05).astype(np.float32)
    n_slots = 6
    tidx = np.array([2, 2, 0, 0, 1, 1], dtype=np.int32) if paired == 2 else np.array([2, 0, 1, 1, 0, 2], dtype=np.int32)
    idx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots).astype(np.int64)
    scale = np.full(n_slots, 0.002, dtype=np.float32)
    obs = rs.randint(0, 256, size=(n_slots, 84, 84, 4)).astype(np.uint8)
    logits, actions = _forward(ctx, net, parents, idx, scale, obs, paired, 1, theta_idx=tidx)
    ref = np.stack([O.forward(net_o, (parents[tidx[s]] + np.float32(0.002) * host_noise[idx[s]:idx[s] + P]).astype(np.float32),
                              obs[s:s + 1])[0][0] for s in range(n_slots)])
    bound = 2e-5 * max(1.0, float(np.abs(ref).max()))
    assert np.abs(logits - ref).max() <= bound, np.abs(logits - ref).max()


def test_two_tables_with_phase_events_match_single_table(ctx, host_noise):
    """Two slot tables on two streams with phase events (both modes) compute exactly what one table computes."""
    net = N.make_net("Model")
    P = net.num_params
    rs = np.random.RandomState(77)
    theta = cuda((rs.randn(P) * 0.05).astype(np.float32))
    n = 8
    pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n // 2).astype(np.int64)
    idx, scale = np.repeat(pidx, 2), np.tile([0.02, -0.02], n // 2).astype(np.float32)
    obs = cuda(rs.randint(0, 256, size=(n, 84, 84, 4)).astype(np.uint8))
    whole = SlotForward(ctx, net, n)
    whole.set_slots(idx, scale)
    whole.forward(theta, obs, paired=1)
    ref_logits, ref_actions = whole.logits.clone(), whole.actions.clone()
    half = n // 2
    tabs = [SlotForward(ctx, net, half) for _ in range(2)]
    streams = [torch.cuda.Stream() for _ in range(2)]
    evs = [torch.cuda.Event() for _ in range(2)]
    for e in evs:
        e.record()
    for h in range(2):
        tabs[h].set_slots(idx[h * half:(h + 1) * half], scale[h * half:(h + 1) * half])
    torch.cuda.synchronize()
    for mode in (0, 1):
        for rep in range(3):
            for h in range(2):
                with torch.cuda.stream(streams[h]):
                    F.check(F.lib().dne_set_phase_events(ctx.handle, C.c_void_p(evs[1 - h].cuda_event),
                                                         C.c_void_p(evs[h].cuda_event), mode))
                    tabs[h].forward(theta, obs[h * half:(h + 1) * half], paired=1)
        torch.cuda.synchronize()
        got = torch.cat([tabs[0].logits, tabs[1].logits])
        assert torch.equal(got, ref_logits), mode
        assert torch.equal(torch.cat([tabs[0].actions, tabs[1].actions]), ref_actions)


@pytest.mark.parametrize("use_tma", [0, 1])
@pytest.mark.parametrize("C_,pixp,W,taps,N,row0", [
    (16, 144, 12, [(0, 0), (0, 1), (1, 0), (1, 1)], 64, 0),      # conv2 geometry: 12-wide s2d grid, LBO 2304 B
    (16, 144, 12, [(0, 0), (0, 1), (1, 0), (1, 1)], 128, 3),     # second tile starting at an arbitrary (16 B aligned) row
    (16, 176, 13, [(dy, dx) for dy in range(3) for dx in range(3)], 128, 0),   # conv3 geometry: 13-wide grid, 9 taps
    (8, 169, 13, [(dy, dx) for dy in range(3) for dx in range(3)], 64, 13),    # LBO 2704 B: NOT a multiple of 128 B
    (16, 488, 22, [(0, 0), (0, 1), (1, 0), (1, 1)], 64, 256),    # conv1 geometry: 22-wide grid, third M tile
])
def test_tcgen05_shifted_window_operand(C_, pixp, W, taps, N, row0, use_tma):
    """The A operand of the convolution kernels: channel-quad planes of an activation image addressed through a
    descriptor whose start address is shifted by (dy*W + dx) pixels (16 bytes each) per filter tap -- no im2col copy.
    Exact integer data, so the tensor-core result must equal the reference bit for bit."""
    rs = np.random.RandomState(C_ * 1000 + pixp + N + row0)
    img = rs.randint(-8, 9, size=(C_ // 4, pixp, 4)).astype(np.float32)
    K = len(taps) * C_
    Bw = rs.randint(-4, 5, size=(N, K)).astype(np.float32)
    off = np.array([dy * W + dx for dy, dx in taps], dtype=np.int32)
    d_img, d_B = cuda(img), cuda(Bw)
    d_D = torch.full((128, N), float("nan"), dtype=torch.float32, device=DEV)
    F.check(F.dev_lib().dne_dev_tc_window(F.ptr(d_img), F.ptr(d_B), F.ptr(d_D), C_, len(taps),
                                          off.ctypes.data_as(C.POINTER(C.c_int)), pixp, N, row0, use_tma, F.stream_ptr()))
    got = d_D.cpu().numpy()
    flat = img.transpose(1, 0, 2).reshape(pixp, C_)                  # [pixel][channel]
    ref = np.zeros((128, N), dtype=np.float64)
    valid = np.ones(128, dtype=bool)
    for t, o in enumerate(off):
        rows = row0 + np.arange(128) + o
        ok = rows < pixp                                            # rows past the image read other planes / slack: ignored
        valid &= ok
        ref[ok] += flat[rows[ok]].astype(np.float64) @ Bw[:, t * C_:(t + 1) * C_].astype(np.float64).T
    assert valid.sum() >= 32
    np.testing.assert_array_equal(got[valid], ref[valid].astype(np.float32))


def test_theta_gemm_tma_vs_thread_staged_and_invalidation(ctx, host_noise):
    """The TMA-fed shared-theta GEMM (dne_theta_prepare + Xc written by the conv3 epilogue) against the thread-staged GEMM
    on 256 and 128 slots, and the staleness rule: after dne_adam_step rewrote theta through the same context the prepared
    entry is dropped, so the next forward must see the NEW weights (with and without a fresh prepare)."""
    from dne.engine import ESUpdate
    net, net_o = N.make_net("LargeModel"), O.make_net("LargeModel")
    P = net.num_params
    rs = np.random.RandomState(123)
    theta0 = (rs.randn(P) * 0.05).astype(np.float32)
    L = F.lib()
    for n_slots in (256, 128, 6):
        pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots // 2).astype(np.int64)
        idx, scale = np.repeat(pidx, 2), np.tile([0.005, -0.005], n_slots // 2).astype(np.float32)
        obs = cuda(rs.randint(0, 256, size=(n_slots, 84, 84, 4)).astype(np.uint8))
        d_theta = cuda(theta0)
        out = {}
        try:
            for tma in (1, 0):
                F.check(L.dne_set_option(b"theta_tma", tma))
                sf = SlotForward(ctx, net, n_slots)
                sf.set_slots(idx, scale)
                a = sf.forward(d_theta, obs, paired=True).cpu().numpy()
                out[tma] = (sf.logits.cpu().numpy(), a)
        finally:
            F.check(L.dne_set_option(b"theta_tma", 1))
        bound = 2e-5 * np.maximum(1.0, np.abs(out[0][0]).max(axis=1))
        assert (np.abs(out[1][0] - out[0][0]).max(axis=1) <= bound).all(), n_slots
    # staleness: one Adam step through the same context, then forward again on the same workspace
    upd = ESUpdate(ctx, theta0, "adam", stepsize=0.05)
    n_slots = 128
    pidx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots // 2).astype(np.int64)
    idx, scale = np.repeat(pidx, 2), np.tile([0.005, -0.005], n_slots // 2).astype(np.float32)
    obs_h = rs.randint(0, 256, size=(n_slots, 84, 84, 4)).astype(np.uint8)
    obs = cuda(obs_h)
    sf = SlotForward(ctx, net, n_slots)
    sf.set_slots(idx, scale)
    sf.forward(upd.theta, obs, paired=True)
    before = sf.logits.clone()
    upd.step(0.005, cuda((rs.randn(P)).astype(np.float32)))                 # theta rewritten in place (same pointer)
    # raw C-ABI forward WITHOUT a new prepare: must not use the stale operand (falls back to the thread-staged GEMM)
    F.check(L.dne_perturb_forward_conv(ctx.handle, C.byref(net.desc), F.ptr(upd.theta), F.ptr(sf.noise_idx), F.ptr(sf.scale),
                                       None, None, n_slots, 1, F.ptr(obs), None, F.ptr(sf.actions), F.ptr(sf.logits),
                                       F.ptr(sf.ws), sf.ws.numel(), F.stream_ptr()))
    raw = sf.logits.cpu().numpy()
    sf.forward(upd.theta, obs, paired=True)                                   # engine path: re-prepares (epoch changed)
    eng = sf.logits.cpu().numpy()
    th = upd.theta.cpu().numpy()
    rows = [0, 1, 64, 127]
    ref = np.stack([O.forward(net_o, (th + np.float32(scale[s]) * host_noise[idx[s]:idx[s] + P]).astype(np.float32),
                              obs_h[s:s + 1])[0][0] for s in rows])
    bound = 2e-5 * np.maximum(1.0, np.abs(ref).max(axis=1))
    assert (np.abs(raw[rows] - ref).max(axis=1) <= bound).all()
    assert (np.abs(eng[rows] - ref).max(axis=1) <= bound).all()
    assert float((before - torch.from_numpy(eng).to(DEV)).abs().max()) > 1e-3       # the step really changed the outputs


@pytest.mark.parametrize("name", ["ESAtariPolicy", "ModelVirtualBN"])
def test_vbn_reference_pass_tensor_core_paths_match_simt(ctx, host_noise, name):
    """The virtual-batch-norm reference pass (policies.py:322-328,399) three ways: conv_tc = 2 (shifted-window wgmma
    convolutions over n_slots * n_ref virtual slots + fp16-split images + tensor-core member GEMM), conv_tc = 1 (r01
    tensor-core kernels) and conv_tc = 0 (fp32 SIMT referee): same statistics, and the tick on those statistics gives the
    same logits.  Ragged sizes: n_ref not a multiple of anything, an inactive slot in the middle, unpaired scales."""
    net = N.make_net(name)
    P = net.num_params
    rs = np.random.RandomState(77)
    theta = (rs.randn(P) * 0.05).astype(np.float32)
    n_slots, n_ref = 10, 21
    idx = rs.randint(0, NOISE_COUNT - P + 1, size=n_slots).astype(np.int64)
    scale = (0.005 * rs.randn(n_slots)).astype(np.float32)
    active = np.ones(n_slots, dtype=np.uint8)
    active[3] = 0
    ref_batch = cuda(rs.randint(0, 256, size=(n_ref, 84, 84, 4)).astype(np.uint8))
    obs = cuda(rs.randint(0, 256, size=(n_slots, 84, 84, 4)).astype(np.uint8))
    d_theta = cuda(theta)
    res = {}
    try:
        for mode in (2, 1, 0):
            F.check(F.lib().dne_set_option(b"conv_tc", mode))
            sf = SlotForward(ctx, net, n_slots, n_ref=n_ref)
            sf.set_slots(idx, scale, active=active)
            sf.vbn.fill_(float("nan"))
            sf.vbn_reference_pass(d_theta, ref_batch, active=sf.active)
            sf.forward(d_theta, obs, paired=False)
            torch.cuda.synchronize()
            res[mode] = (sf.vbn.cpu().numpy().copy(), sf.logits.cpu().numpy().copy())
    finally:
        F.check(F.lib().dne_set_option(b"conv_tc", 2))
    live = active.astype(bool)
    for mode in (2, 1):
        vbn, logits = res[mode]
        assert np.isnan(vbn[~live]).all()                        # inactive slots are not touched
        assert np.isfinite(vbn[live]).all()
        np.testing.assert_allclose(vbn[live], res[0][0][live], rtol=3e-4, atol=3e-5)
        np.testing.assert_allclose(logits[live], res[0][1][live], rtol=0, atol=5e-4 * max(1.0, np.abs(res[0][1][live]).max()))
