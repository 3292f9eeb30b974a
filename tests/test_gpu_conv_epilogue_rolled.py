"""The staged conv epilogue (registers -> shared-memory tile -> rolled store loop) on every compiled conv shape, against the
fp32 SIMT convolutions (conv_tc = 0, the referee of bench.py's parity check), and bit-identical reruns.

Output modes: the next layer's image at space-to-depth stride 2 (conv1 -> conv2) and stride 1 (conv2 -> conv3 of
LargeModel), NHWC floats + the Xc copy (the last conv layer).  Epilogue flavours: ReLU, tanh and identity without batch
norm, and both batch-norm flavours (ESAtariPolicy: BN_TF, ModelVirtualBN: BN_GPU), whose statistics come from the
virtual-batch-norm reference pass (n_slots * n_ref virtual slots, vdiv > 1, over shared frames, in_mod > 0).  Slots:
an inactive slot in the middle and an inactive tail."""
import numpy as np
import pytest
import torch

from dne import _ffi as F, nets
from dne.engine import SlotForward, make_context
from dne.noise import SharedNoiseTable

pytestmark = pytest.mark.gpu

COUNT = 6_000_000
N_SLOTS = 150                    # more than one member per CTA on a 132-SM card


def act_mix_net():
    """LargeModel's conv shapes with tanh, identity and tanh on conv1 .. conv3."""
    layers = [nets._conv(4, 32, 8, 4, 84, act=F.ACT_TANH), nets._conv(32, 64, 4, 2, 21, act=F.ACT_NONE),
              nets._conv(64, 64, 3, 1, 11, act=F.ACT_TANH), nets._dense(11 * 11 * 64, 512), nets._dense(512, 18, act=F.ACT_NONE)]
    return nets._finish(nets.NetSpec("act_mix", layers, F.OB_ATARI_U8, 84 * 84 * 4))


NETS = {"LargeModel": lambda: nets.make_net("LargeModel"), "GAAtariPolicy": lambda: nets.make_net("GAAtariPolicy"),
        "act_mix": act_mix_net, "ESAtariPolicy": lambda: nets.make_net("ESAtariPolicy"),
        "ModelVirtualBN": lambda: nets.make_net("ModelVirtualBN")}


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    return make_context(0, SharedNoiseTable(count=COUNT, device="cuda:0"))


def run(ctx, net, theta, obs, idx, scale, active, ref_batch, conv_tc):
    L = F.lib()
    F.check(L.dne_set_option(b"conv_tc", conv_tc))
    try:
        n_ref = 0 if ref_batch is None else ref_batch.shape[0]
        sf = SlotForward(ctx, net, len(idx), **({"n_ref": n_ref} if n_ref else {}))
        sf.set_slots(idx, scale, active=active)
        vbn = None
        if n_ref:
            sf.vbn.fill_(float("nan"))
            sf.vbn_reference_pass(theta, ref_batch, active=sf.active)
            vbn = sf.vbn.clone()
        sf.logits.fill_(0)
        acts = sf.forward(theta, obs, paired=False).clone()
        torch.cuda.synchronize()
        return sf.logits.clone(), acts, vbn
    finally:
        F.check(L.dne_set_option(b"conv_tc", 2))


@pytest.mark.parametrize("name", list(NETS))
def test_staged_epilogue_matches_simt(ctx, name):
    net = NETS[name]()
    rs = np.random.RandomState(31)
    theta = torch.from_numpy((rs.randn(net.num_params) * 0.05).astype(np.float32)).cuda()
    n = N_SLOTS
    idx = rs.randint(0, COUNT - net.num_params + 1, size=n).astype(np.int64)
    scale = (rs.randn(n) * 0.01).astype(np.float32)
    active = np.ones(n, np.uint8)
    active[[5, 70, 71]] = 0
    active[137:] = 0
    obs = torch.randint(0, 256, (n, 84, 84, 4), dtype=torch.uint8, device="cuda")
    bn = any(l.bn != F.BN_NONE for l in net.layers)
    ref_batch = torch.randint(0, 256, (13, 84, 84, 4), dtype=torch.uint8, device="cuda") if bn else None
    lf, af, vf = run(ctx, net, theta, obs, idx, scale, active, ref_batch, 2)
    lr, ar, vr = run(ctx, net, theta, obs, idx, scale, active, ref_batch, 0)
    on = torch.from_numpy(active.astype(bool)).cuda()
    if bn:
        assert bool(vf[~on].isnan().all())                       # inactive members are not touched
        assert bool(vf[on].isfinite().all())
        torch.testing.assert_close(vf[on], vr[on], rtol=3e-4, atol=3e-5)
    lf, lr, af, ar = lf[on], lr[on], af[on], ar[on]
    # the forward bound of the tensor-core paths against the SIMT referee (BN: statistics from the reference pass too)
    bound = (5e-4 if bn else 4e-5) * torch.clamp(lr.abs().max(dim=1).values, min=1.0)
    assert bool(((lf - lr).abs().max(dim=1).values <= bound).all())
    srt = lr.sort(dim=1).values
    decided = (srt[:, -1] - srt[:, -2]) > 2 * bound
    assert torch.equal(af[decided], ar[decided])
    lf2, af2, vf2 = run(ctx, net, theta, obs, idx, scale, active, ref_batch, 2)
    assert torch.equal(lf2[on], lf) and torch.equal(af2[on], af)
    if bn:
        assert torch.equal(vf2[on], vf[on])
