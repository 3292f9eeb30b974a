"""GPU-box measurement of the other BASELINE.json configurations' device hot paths (configs 1, 3, 4, 5): per-tick /
per-call kernel-path timings with inputs resident in HBM.  Not the headline bench (bench.py = config 2); results go to
other_configs.json in the output directory."""
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "deep-neuroevolution_b200")]
import numpy as np
import torch
from dne import _ffi as F, nets
from dne.engine import SlotForward, ESUpdate, make_context
from dne.noise import SharedNoiseTable, generate_host


def timeit(fn, n=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(True), torch.cuda.Event(True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


count = int(os.environ.get("NOISE_COUNT", 250_000_000))
noise = SharedNoiseTable(host_noise=generate_host(count), device="cuda:0")
ctx = make_context(0, noise)
L = F.lib()
rs = np.random.RandomState(0)
out = {}

# ---- config 5: MLP 376-256-256-17, ES pop 10000 (5000 pairs), env stubbed -------------------------------------
net = nets.make_net("MujocoPolicy")
P = net.num_params
slots = 10000
theta = torch.from_numpy((rs.randn(P) * 0.1).astype(np.float32)).cuda()
pidx = rs.randint(0, count - P + 1, size=slots // 2).astype(np.int64)
sf = SlotForward(ctx, net, slots)
sf.set_slots(np.repeat(pidx, 2), np.tile([0.02, -0.02], slots // 2).astype(np.float32))
obs = torch.randn(slots, 376, device="cuda")
mean, std = torch.zeros(376, device="cuda"), torch.ones(376, device="cuda")
ms = timeit(lambda: sf.forward(theta, obs, paired=True, ob_mean=mean, ob_std=std))
upd = ESUpdate(ctx, theta, "adam", stepsize=0.01)
gi = torch.from_numpy(rs.randint(0, count - P + 1, size=5000).astype(np.int64)).cuda()
proc = torch.randn(5000, 2, device="cuda")
ms_g = timeit(lambda: upd.gradient(proc, gi, 10000), n=5, warm=1)
ms_r = timeit(lambda: upd.centered_ranks(proc), n=5, warm=1)
ms_a = timeit(lambda: upd.step(0.005), n=10)
out["config5_mlp_pop10000"] = {
    "slots": slots, "ms_per_tick": ms, "env_steps_per_s": slots / ms * 1e3,
    "noise_GBs_pair_shared": slots / 2 * 4 * P / ms / 1e6, "noise_GBs_survey(4P per env-step)": slots * 4 * P / ms / 1e6,
    "update": {"rank_ms(20000 values)": ms_r, "grad_ms(n=5000)": ms_g, "grad_GBs": 5000 * 4 * P / ms_g / 1e6, "adam_ms": ms_a}}
print("config5", json.dumps(out["config5_mlp_pop10000"]), flush=True)
del sf, obs

# ---- config 3: Deep GA, LargeModel, pop 1000 offspring over 256 slots, T = 20 cached parents -------------------
net = nets.make_net("LargeModel")
P = net.num_params
slots, T = 256, 20
parents = torch.from_numpy((rs.randn(T, P) * 0.05).astype(np.float32)).cuda()
obs = torch.randint(0, 256, (slots, 84, 84, 4), dtype=torch.uint8, device="cuda")
seeds = rs.randint(0, count - P + 1, size=slots).astype(np.int64)
res = {}
for label, tidx, paired in (("unsorted_parents", rs.randint(0, T, size=slots).astype(np.int32), 0),
                            ("sibling_pairs_share_parent", np.repeat(rs.randint(0, T, size=slots // 2), 2).astype(np.int32), 2)):
    sf = SlotForward(ctx, net, slots)
    sf.set_slots(seeds, np.full(slots, 0.002, np.float32), theta_idx=tidx)
    ms = timeit(lambda: sf.forward(parents, obs, paired=paired))
    res[label] = {"ms_per_tick": ms, "env_steps_per_s": slots / ms * 1e3,
                  "weight_GBs(noise + parent rows)": (slots * 4 * P + (slots if paired == 0 else slots / 2) * 4 * P) / ms / 1e6}
    del sf
# genome materialisation + one mutation + truncation select
std = (C.c_double * len(net.layers))(*net.init_std())
chain = 256
d_seeds = torch.from_numpy(rs.randint(0, count - P + 1, size=chain).astype(np.int64)).cuda()
d_pow = torch.full((chain,), 0.002, dtype=torch.float32, device="cuda")
outp = torch.empty(P, dtype=torch.float32, device="cuda")
for ln in (1, 16, 256):
    res[f"materialize_chain{ln}_ms"] = timeit(lambda: F.check(L.dne_ga_materialize(
        ctx.handle, C.byref(net.desc), F.ptr(d_seeds), F.ptr(d_pow), ln, std, 0, F.ptr(outp), F.stream_ptr())), n=5, warm=1)
res["mutate_ms"] = timeit(lambda: F.check(L.dne_ga_mutate(ctx.handle, F.ptr(parents[0]), int(seeds[0]), 0.002, P,
                                                         F.ptr(outp), F.stream_ptr())), n=20)
fit = torch.rand(1000, device="cuda")
sel = torch.empty(20, dtype=torch.int32, device="cuda")
res["truncate_pop1000_T20_ms"] = timeit(lambda: F.check(L.dne_ga_truncate(F.ptr(fit), 1000, 20, F.ptr(sel), F.stream_ptr())), n=20)
out["config3_deep_ga_largemodel"] = res
print("config3", json.dumps(res), flush=True)

# ---- config 1/4: ESAtariPolicy (virtual batch norm) tick + reference pass; k-NN novelty ------------------------
net = nets.make_net("ESAtariPolicy")
P = net.num_params
slots = 256
theta = torch.from_numpy((rs.randn(P) * 0.05).astype(np.float32)).cuda()
pidx = rs.randint(0, count - P + 1, size=slots // 2).astype(np.int64)
sf = SlotForward(ctx, net, slots)
sf.set_slots(np.repeat(pidx, 2), np.tile([0.005, -0.005], slots // 2).astype(np.float32))
ref = torch.randint(0, 256, (128, 84, 84, 4), dtype=torch.uint8, device="cuda")
ms_v = timeit(lambda: sf.vbn_reference_pass(theta, ref), n=3, warm=1)
ms_t = timeit(lambda: sf.forward(theta, obs, paired=True))
out["config1_es_atari_policy_vbn"] = {"slots": slots, "ms_per_tick": ms_t, "env_steps_per_s": slots / ms_t * 1e3,
                                      "vbn_reference_pass_ms(256 members x 128 obs)": ms_v,
                                      "vbn_GFLOPs": slots * 128 * 7.6e6 / ms_v / 1e6}
print("config1", json.dumps(out["config1_es_atari_policy_vbn"]), flush=True)
del sf
knn = {}
q, t_max, D, k = 1000, 1000, 128, 10
bc = torch.randint(0, 256, (q, t_max, D), dtype=torch.uint8, device="cuda")
bl = torch.full((q,), t_max, dtype=torch.int32, device="cuda")
for A in (8, 256, 4096):
    ar = torch.randint(0, 256, (A, t_max, D), dtype=torch.uint8, device="cuda")
    al = torch.full((A,), t_max, dtype=torch.int32, device="cuda")
    nb = C.c_size_t()
    F.check(L.dne_knn_ws_bytes(q, A, C.byref(nb)))
    ws = torch.empty(max(nb.value, 256), dtype=torch.uint8, device="cuda")
    nov = torch.empty(q, dtype=torch.float32, device="cuda")
    ms = timeit(lambda: F.check(L.dne_knn_novelty(F.ptr(bc), F.ptr(bl), q, F.ptr(ar), F.ptr(al), A, t_max, D, k,
                                                  F.ptr(nov), F.ptr(ws), ws.numel(), F.stream_ptr())), n=2, warm=1)
    knn[f"archive_{A}"] = {"ms": ms, "pair_distances_per_s": q * A / ms * 1e3, "byte_pairs_GBs": q * A * t_max * D * 2 / ms / 1e6}
    del ar
out["config4_knn_novelty_q1000_t1000"] = knn
print("config4", json.dumps(knn), flush=True)
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "gpurun_out", "other_configs.json"), "w"), indent=1)
