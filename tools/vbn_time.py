"""Dev tool (GPU box): time of the virtual-batch-norm reference pass (256 members x 128 reference observations) per
conv_tc mode (2 = shifted-window wgmma convs over virtual slots + tensor-core member GEMM, 1 = r01 tensor-core kernels,
0 = fp32 SIMT).  Not a bench."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-neuroevolution_b200")]
import numpy as np, torch
from dne import _ffi as F, nets
from dne.engine import SlotForward, make_context
from dne.noise import SharedNoiseTable
count = int(os.environ.get("NOISE_COUNT", 50_000_000))
ctx = make_context(0, SharedNoiseTable(count=count, device="cuda:0"))
rs = np.random.RandomState(0)
n_slots, n_ref = int(os.environ.get("SLOTS", 256)), int(os.environ.get("NREF", 128))
for name in ("ESAtariPolicy", "ModelVirtualBN"):
    net = nets.make_net(name); P = net.num_params
    theta = torch.from_numpy((rs.randn(P) * 0.05).astype(np.float32)).cuda()
    ref = torch.randint(0, 256, (n_ref, 84, 84, 4), dtype=torch.uint8, device="cuda")
    pidx = rs.randint(0, count - P + 1, size=n_slots // 2).astype(np.int64)
    flops = 0
    for L in net.desc.layers[:net.desc.n_layers]:
        if L.kind == F.CONV: flops += 2 * L.hout * L.hout * L.cout * L.ksize * L.ksize * L.cin
        elif L.bn != 0: flops += 2 * L.cin * L.cout
    for mode in [int(x) for x in os.environ.get("MODES", "2,1").split(",")]:
        F.check(F.lib().dne_set_option(b"conv_tc", mode))
        sf = SlotForward(ctx, net, n_slots, n_ref=n_ref)
        sf.set_slots(np.repeat(pidx, 2), np.tile([0.005, -0.005], n_slots // 2).astype(np.float32))
        for _ in range(2): sf.vbn_reference_pass(theta, ref)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(True), torch.cuda.Event(True)
        a.record()
        for _ in range(5): sf.vbn_reference_pass(theta, ref)
        b.record(); torch.cuda.synchronize()
        ms = a.elapsed_time(b) / 5
        print(json.dumps(dict(net=name, conv_tc=mode, slots=n_slots, n_ref=n_ref, ms=round(ms, 3),
                              tflops_fp32_equiv=round(flops * n_slots * n_ref / ms / 1e9, 1))), flush=True)
        del sf
    F.check(F.lib().dne_set_option(b"conv_tc", 2))
