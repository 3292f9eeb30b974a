"""Dev tool (GPU box): interleaved A/B of dne_set_option variants on the warm tick (kernel-by-kernel launches, CUDA events over
blocks of ticks, variants alternated inside one process so that clock / thermal drift hits them equally).  Not a bench.
VARIANTS="name:opt=v,opt=v;name2:..."  SLOTS_LIST=124,256"""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-neuroevolution_b200")]
import numpy as np, torch
from dne import _ffi as F, nets
from dne.engine import SlotForward, make_context
from dne.noise import SharedNoiseTable
count = int(os.environ.get("NOISE_COUNT", 250_000_000))
ctx = make_context(0, SharedNoiseTable(count=count, device="cuda:0"))
net = nets.make_net("LargeModel"); P = net.num_params
rs = np.random.RandomState(0)
theta = torch.from_numpy((rs.randn(P) * 0.05).astype(np.float32)).cuda()
variants = []
for v in os.environ.get("VARIANTS", "base:").split(";"):
    name, _, spec = v.partition(":")
    variants.append((name, [kv.split("=") for kv in spec.split(",") if kv]))
keys = sorted({k for _, kv in variants for k, _ in kv})
defaults = {"chain_ticks": 0, "fold_theta": 1, "pdl": 1, "fuse_head": 1, "theta_tma": 1, "gemv_stages": 5, "gemv_ctas_per_sm": 2, "gemv_grid": 0}
ROUNDS, TICKS = int(os.environ.get("ROUNDS", 7)), int(os.environ.get("TICKS", 150))
for slots in [int(x) for x in os.environ.get("SLOTS_LIST", "124,256").split(",")]:
    pidx = rs.randint(0, count - P + 1, size=slots // 2).astype(np.int64)
    sf = SlotForward(ctx, net, slots)
    sf.set_slots(np.repeat(pidx, 2), np.tile([0.005, -0.005], slots // 2).astype(np.float32))
    pool = torch.randint(0, 256, (4, slots, 84, 84, 4), dtype=torch.uint8, device="cuda")
    times = {name: [] for name, _ in variants}
    for r in range(ROUNDS):
        for name, kv in variants:
            for k in keys: F.check(F.lib().dne_set_option(k.encode(), defaults[k]))
            for k, v in kv: F.check(F.lib().dne_set_option(k.encode(), int(v)))
            for t in range(10): sf.forward(theta, pool[t & 3], paired=True)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(True), torch.cuda.Event(True)
            a.record()
            for t in range(TICKS): sf.forward(theta, pool[t & 3], paired=True)
            b.record(); torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b) / TICKS * 1e3)
    for k in keys: F.check(F.lib().dne_set_option(k.encode(), defaults[k]))
    print(slots, json.dumps({n: dict(median=round(float(np.median(t)), 2), min=round(min(t), 2), max=round(max(t), 2)) for n, t in times.items()}), flush=True)
