"""Dev tool (GPU box): forward-tick throughput of the LargeModel hot path for different slot-table / stream /
phase-event schedules (the knobs bench.py exposes as DNE_BENCH_STREAMS, DNE_GEMV_CTAS, DNE_PHASE_MODE)."""
import ctypes as C, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-neuroevolution_b200")]
import numpy as np, torch
from dne import _ffi as F, nets
from dne.engine import SlotForward, make_context
from dne.noise import SharedNoiseTable, generate_host
count = int(os.environ.get("NOISE_COUNT", 120_000_000))
ctx = make_context(0, SharedNoiseTable(host_noise=generate_host(count), device="cuda:0"))
net = nets.make_net("LargeModel"); P = net.num_params
rs = np.random.RandomState(0)
theta = torch.from_numpy((rs.randn(P) * 0.05).astype(np.float32)).cuda()
L = F.lib()
net_ref = C.byref(net.desc)
R = 4

def run(total, NS, gemv_ctas, mode, stages=5, ticks=300):
    F.check(L.dne_set_option(b"gemv_ctas_per_sm", gemv_ctas))
    F.check(L.dne_set_option(b"gemv_stages", stages))
    part = (total // NS) // 2 * 2
    sfs = [SlotForward(ctx, net, part) for _ in range(NS)]
    for sf in sfs:
        pidx = rs.randint(0, count - P + 1, size=part // 2).astype(np.int64)
        sf.set_slots(np.repeat(pidx, 2), np.tile([0.02, -0.02], part // 2).astype(np.float32))
    pool = torch.randint(0, 256, (R, NS * part, 84, 84, 4), dtype=torch.uint8, device="cuda")
    streams = [torch.cuda.Stream() for _ in range(NS)]
    evs = [torch.cuda.Event() for _ in range(max(NS, 2))]
    for e in evs: e.record()
    args = [(F.ptr(sf.noise_idx), F.ptr(sf.scale), F.ptr(sf.actions), F.ptr(sf.logits), F.ptr(sf.ws), sf.ws.numel()) for sf in sfs]
    obs = [[F.ptr(pool[r][h * part:(h + 1) * part]) for h in range(NS)] for r in range(R)]
    sp = [C.c_void_p(s.cuda_stream) for s in streams]
    ep = [C.c_void_p(e.cuda_event) for e in evs]
    th = F.ptr(theta)
    cur = torch.cuda.current_stream()
    def loop(n):
        for s in streams: s.wait_stream(cur)
        for t in range(n):
            for h in range(NS):
                if NS >= 2 and mode >= 0:
                    L.dne_set_phase_events(ctx.handle, ep[(h - 1) % NS], ep[h], mode)
                a = args[h]
                rc = L.dne_perturb_forward_conv(ctx.handle, net_ref, th, a[0], a[1], None, None, part, 1, obs[t % R][h], None,
                                                a[2], a[3], a[4], a[5], sp[h])
                if rc: F.check(rc)
        for s in streams: cur.wait_stream(s)
    loop(30); torch.cuda.synchronize()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True)
    a.record(); loop(ticks); b.record(); torch.cuda.synchronize()
    L.dne_set_phase_events(ctx.handle, None, None, 0)
    us = a.elapsed_time(b) * 1e3 / ticks
    print(f"slots={NS * part:4d} tables={NS} gemv_ctas/SM={gemv_ctas} stages={stages} phase_mode={mode:2d}: tick {us:7.1f} us  -> {NS * part / us * 1e6 / 1e3:7.1f}K env-steps/s", flush=True)

CFGS = eval(os.environ["SWEEP"]) if os.environ.get("SWEEP") else None
for cfg in CFGS or [(256, 1, 2, -1, 5), (256, 1, 1, -1, 8), (256, 1, 1, -1, 4), (512, 2, 2, -1, 5), (512, 2, 1, 1, 4),
            (512, 4, 1, 1, 4), (512, 2, 2, -1, 3)]:
    try:
        run(*cfg)
    except Exception as e:
        print(cfg, "failed:", e, flush=True)
