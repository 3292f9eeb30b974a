"""Per-kernel split of the chained LargeModel tick (GPU box).  Not a bench.

Builds the workload bench.py's `value` leg runs (make_context, SlotForward(ctx, LargeModel, 256), ESUpdate, the seeded
theta0 / observation pool / index stream, a full 128-pair wave, chain_ticks = 1, ticks issued by the same raw
dne_perturb_forward_conv call on one stream) and measures one window of ticks three ways:

  split    torch.profiler with CUDA activities, no event records in the chain.  Per kernel: mean duration, and its
           critical-path share = its end minus the previous kernel's end (under PDL a kernel is resident early, so its
           duration includes the time spent in griddepcontrol.wait); the gap = its start minus the previous kernel's end.
  plain    the same window unprofiled, CUDA events only at its two ends: ms per tick.  The shares add up to the
           profiled window's end-to-end time per tick, which is compared with this figure.
  gemv_ev  the fc noise GEMV timed with CUDA events around every 16th tick's launch (dne_profile_enable, as bench.py's
           roofline), next to its in-chain duration and share.

    python tools/tick_split.py --out result.json [--ticks 300] [--plain-ticks 2000]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-neuroevolution_b200")]
import numpy as np  # noqa: E402
import torch  # noqa: E402
from dne import _ffi as F, nets  # noqa: E402
from dne.engine import ESUpdate, SlotForward, make_context  # noqa: E402
from dne.noise import SharedNoiseTable  # noqa: E402

SIGMA, LR = 0.005, 0.01            # bench.py
ORDER = ["conv1", "conv2", "conv3", "theta_gemm", "noise_gemv", "head"]


def kernel_name(raw):
    """Stable short name of a tick kernel from its demangled name (None: not a tick kernel)."""
    if "conv_s2d_kernel" in raw:
        if "true>" in raw or ", true" in raw:
            return "conv1"
        return "conv3" if "<64, 64, 3" in raw else "conv2"
    if "theta_gemm_tma_kernel" in raw:
        return "theta_gemm"
    if "gemv_union_kernel" in raw:
        return "noise_gemv"
    if "dense_combine_head_kernel" in raw:
        return "head"
    return None


def gpu_info():
    q = "name,power.limit,enforced.power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=20).stdout.strip()
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:  # the numbers are still worth having without it
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--ticks", type=int, default=300, help="profiled window (ticks)")
    ap.add_argument("--plain-ticks", type=int, default=2000, help="unprofiled window (ticks)")
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--noise-count", type=int, default=250_000_000)
    a = ap.parse_args()
    assert a.ticks >= 200 and torch.cuda.is_available()

    dev = torch.device("cuda", 0)
    L = F.lib()
    noise = SharedNoiseTable(count=a.noise_count, device=dev)
    ctx = make_context(0, noise)
    net = nets.make_net("LargeModel")
    P = net.num_params
    rs = np.random.RandomState(0)
    theta0 = (rs.randn(P) * 0.05).astype(np.float32)
    upd = ESUpdate(ctx, theta0, "adam", stepsize=LR)
    slots = 256
    sf = SlotForward(ctx, net, slots)
    stream = torch.cuda.Stream(device=dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(1234)
    R = 4
    pool = torch.randint(0, 256, (R, slots, 84, 84, 4), dtype=torch.uint8, device=dev, generator=gen)
    idx_stream = np.random.RandomState(1)
    wave = np.array([noise.sample_index(idx_stream, P) for _ in range(slots // 2)], dtype=np.int64)
    sf.set_slots(np.zeros(slots, np.int64), np.zeros(slots, np.float32), active=np.ones(slots, np.uint8))
    sf.set_slots(np.repeat(wave, 2), np.tile([SIGMA, -SIGMA], slots // 2).astype(np.float32),
                 active=np.ones(slots, np.uint8))
    with torch.cuda.stream(stream):
        sf.prepare(upd.theta, slots)
    torch.cuda.synchronize()

    net_ref = C.byref(net.desc)
    theta_p = F.ptr(upd.theta)
    args = (F.ptr(sf.noise_idx), F.ptr(sf.scale), F.ptr(sf.active), F.ptr(sf.actions), F.ptr(sf.logits), F.ptr(sf.ws),
            sf.ws.numel())
    obs_ptr = [F.ptr(pool[r]) for r in range(R)]
    sp = C.c_void_p(stream.cuda_stream)
    fwd = L.dne_perturb_forward_conv

    def ticks(n, prof_every=0):
        for t in range(n):
            if prof_every and t % prof_every == 0:
                L.dne_profile_enable(ctx.handle, 2, 0)
            F.check(fwd(ctx.handle, net_ref, theta_p, args[0], args[1], None, args[2], slots, 1, obs_ptr[t % R], None,
                        args[3], args[4], args[5], args[6], sp))
            if prof_every and t % prof_every == 0:
                L.dne_profile_enable(ctx.handle, 0, 0)

    F.check(L.dne_set_option(b"chain_ticks", 1))
    try:
        ticks(a.warmup)
        torch.cuda.synchronize()

        # ---- plain: events at the window's two ends only ----
        plain = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            ticks(a.plain_ticks)
            e1.record(stream)
            torch.cuda.synchronize()
            plain.append(e0.elapsed_time(e1) / a.plain_ticks)
        info = gpu_info()                                   # right after a busy window: the clock under load

        # ---- split: torch.profiler, no event records in the chain ----
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ticks(a.ticks)
            torch.cuda.synchronize()
        with tempfile.TemporaryDirectory() as td:
            path = os.path.join(td, "trace.json")
            prof.export_chrome_trace(path)
            with open(path) as f:
                trace = json.load(f)

        # ---- gemv_ev: CUDA events around every 16th tick's GEMV launch ----
        F.check(L.dne_profile_enable(ctx.handle, 1, 16384))
        F.check(L.dne_profile_enable(ctx.handle, 0, 0))
        ticks(a.plain_ticks, prof_every=16)
        torch.cuda.synchronize()
        n, tot = C.c_int(), C.c_double()
        F.check(L.dne_profile_read(ctx.handle, C.byref(n), C.byref(tot)))
        F.check(L.dne_profile_enable(ctx.handle, 0, 0))
        gemv_ev_ms = tot.value / max(n.value, 1)
    finally:
        F.check(L.dne_set_option(b"chain_ticks", 0))

    ks = []
    for ev in trace.get("traceEvents", []):
        if ev.get("cat") != "kernel":
            continue
        nm = kernel_name(ev.get("name", ""))
        if nm is None:
            raise RuntimeError(f"unexpected kernel in the tick window: {ev.get('name')}")
        ks.append((float(ev["ts"]), float(ev["ts"]) + float(ev["dur"]), nm))
    ks.sort()
    names = [k[2] for k in ks]
    per_tick = len(set(names))
    assert len(ks) == per_tick * a.ticks, f"{len(ks)} kernels for {a.ticks} ticks of {per_tick}"
    dur, share, gap = {}, {}, {}
    for i in range(1, len(ks)):             # the first kernel has no predecessor in the window
        s, e, nm = ks[i]
        pe = ks[i - 1][1]
        dur.setdefault(nm, []).append(e - s)
        share.setdefault(nm, []).append(e - pe)
        gap.setdefault(nm, []).append(s - pe)
    n_win = len(ks) - 1
    span_ms = (ks[-1][1] - ks[0][1]) / 1e3
    kernels = {}
    for nm in [x for x in ORDER if x in dur]:
        kernels[nm] = {"duration_ms": float(np.mean(dur[nm])) / 1e3, "share_ms": float(np.mean(share[nm])) / 1e3,
                       "gap_ms": float(np.mean(gap[nm])) / 1e3, "share_median_ms": float(np.median(share[nm])) / 1e3}
    tick_split_ms = span_ms / (n_win / per_tick)
    out = {
        "gpu": info, "ticks_profiled": a.ticks, "ticks_plain": a.plain_ticks, "slots": slots, "pairs": slots // 2,
        "kernels_per_tick": per_tick, "kernels": kernels,
        "tick_ms_profiled": tick_split_ms, "sum_of_shares_ms": float(sum(v["share_ms"] for v in kernels.values())),
        "tick_ms_plain": plain, "tick_ms_plain_median": float(np.median(plain)),
        "gemv_event_timed_ms": gemv_ev_ms, "gemv_event_timed_launches": n.value,
        "non_gemv_share_ms": float(sum(v["share_ms"] for k, v in kernels.items() if k != "noise_gemv")),
    }
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
