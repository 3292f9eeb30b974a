"""The conv epilogue's short variant (ReLU, no batch norm: conv2 and conv3 of LargeModel) against the fp32 SIMT
convolutions (conv_tc = 0, the referee of bench.py's parity check) at the benchmarked 256 slots, with an inactive tail
and with unpaired scales; and bit-identical reruns."""
import numpy as np
import pytest
import torch

from dne import _ffi as F, nets
from dne.engine import SlotForward, make_context
from dne.noise import SharedNoiseTable

pytestmark = pytest.mark.gpu

COUNT = 6_000_000


@pytest.fixture(scope="module")
def setup():
    if not torch.cuda.is_available():
        pytest.skip("needs a GPU")
    ctx = make_context(0, SharedNoiseTable(count=COUNT, device="cuda:0"))
    net = nets.make_net("LargeModel")
    rs = np.random.RandomState(7)
    theta = torch.from_numpy((rs.randn(net.num_params) * 0.05).astype(np.float32)).cuda()
    return ctx, net, theta, rs


def run(ctx, net, theta, obs, idx, scale, active, paired, conv_tc):
    L = F.lib()
    F.check(L.dne_set_option(b"conv_tc", conv_tc))
    try:
        sf = SlotForward(ctx, net, len(idx))
        sf.set_slots(idx, scale, active=active)
        sf.logits.fill_(0)
        acts = sf.forward(theta, obs, paired=paired).clone()
        torch.cuda.synchronize()
        return sf.logits.clone(), acts
    finally:
        F.check(L.dne_set_option(b"conv_tc", 2))


@pytest.mark.parametrize("case", ["full", "inactive_tail", "unpaired"])
def test_epilogue_variant_matches_simt(setup, case):
    ctx, net, theta, rs = setup
    n = 256
    pidx = rs.randint(0, COUNT - net.num_params + 1, size=n // 2).astype(np.int64)
    if case == "unpaired":
        idx = rs.randint(0, COUNT - net.num_params + 1, size=n).astype(np.int64)
        scale = (rs.randn(n) * 0.01).astype(np.float32)
    else:
        idx, scale = np.repeat(pidx, 2), np.tile([0.005, -0.005], n // 2).astype(np.float32)
    active = np.ones(n, np.uint8)
    if case == "inactive_tail":
        active[232:] = 0
    paired = case != "unpaired"
    obs = torch.randint(0, 256, (n, 84, 84, 4), dtype=torch.uint8, device="cuda")
    lf, af = run(ctx, net, theta, obs, idx, scale, active, paired, 2)
    lr, ar = run(ctx, net, theta, obs, idx, scale, active, paired, 0)
    on = torch.from_numpy(active.astype(bool)).cuda()
    lf, lr, af, ar = lf[on], lr[on], af[on], ar[on]
    bound = 4e-5 * torch.clamp(lr.abs().max(dim=1).values, min=1.0)
    assert bool(((lf - lr).abs().max(dim=1).values <= bound).all())
    srt = lr.sort(dim=1).values
    decided = (srt[:, -1] - srt[:, -2]) > 2 * bound
    assert torch.equal(af[decided], ar[decided])
    lf2, af2 = run(ctx, net, theta, obs, idx, scale, active, paired, 2)
    assert torch.equal(lf2[on], lf) and torch.equal(af2[on], af)
