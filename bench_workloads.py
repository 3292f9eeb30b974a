"""bench.py --workload {mlp, ga, nsr}: BASELINE.json configs[4], [2] and [3] on the same JSON contract as the default
(`es` = configs[1]) line: metric env-steps/s, device-timed `value` with inputs resident in HBM, `e2e` through the
reference-facing driver with a host environment, clocks, launches, and a roofline object for the dominant HBM-bound work.

  mlp  configs[4]: MLP 376-256-256-17 tanh (MujocoPolicy), ES pop 10000 (5000 antithetic pairs), env step stubbed
       (float32 observations regenerated on the device), T ticks per generation + update (ranks over 20000 returns,
       gradient over 5000 slices, Adam).  Roofline: the whole tick -- 6 small kernels, 0.67 MB of noise per pair.
  ga   configs[2]: Deep GA, LargeModel, pop 1000 offspring per generation, truncation T = 20, parents cached in HBM; an
       offspring = theta[parent] + power * noise[seed] evaluated straight from the slot table (per-slot parent row:
       the fc layer streams the parent's weights AND the noise slice).  Generation = rollouts + dne_ga_truncate + the
       new parents' dne_ga_mutate.  Roofline: the two GEMV launches per tick (noise + parent rows).
  nsr  configs[3]: NSR-ES, pop 1000 (500 pairs), LargeModel forward as in `es` + per generation the k-NN novelty of the
       1000 episodes' behaviour characterisations ([T, 128] uint8 RAM traces, synthetic) against an on-device archive
       (256 entries), reward-rank / novelty-rank blend, gradient, Adam.  Roofline: the fc noise GEMV (as `es`).
Population sharded over the ranks exactly like `es` (all_gather of returns / fitness / novelty + one all_reduce of g)."""
from __future__ import annotations

import ctypes as C
import json
import os
import time

import numpy as np


def run(args, emit, ClockSampler, load_peaks):
    import torch
    import torch.distributed as dist
    from dne import _ffi as F, nets, shard
    from dne.engine import ESUpdate, SlotForward, make_context
    from dne.noise import SharedNoiseTable

    wl = args.workload
    rank, world, local = shard.init_from_env("nccl")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}"
    peaks, peak_src = load_peaks()
    L = F.lib()
    noise = SharedNoiseTable(count=args.noise_count, device=dev)
    ctx = make_context(local, noise)
    rs = np.random.RandomState(0)
    T = args.episode_len
    SIGMA, L2, LR = 0.02, 0.005, 0.01
    tally = {"ticks": 0, "pairs": 0, "gemv_bytes": 0.0}

    # ------------------------------------------------------------------------------------------------ workload set-up
    if wl == "mlp":
        net = nets.make_net("MujocoPolicy")
        pop = args.pop if args.pop != 1000 else 10000
        n_units, G = pop // 2, 2
        slots_cap = 10000
        label = f"humanoid_mlp_es_pop{pop}_T{T}"
        policy_desc = "MujocoPolicy 376-256-256-17 tanh (P=166673)"
    elif wl == "ga":
        net = nets.make_net("LargeModel")
        pop = args.pop
        n_units, G = pop, 1
        slots_cap = args.slots
        label = f"frostbite_deepga_pop{pop}_T20parents_LargeModel_T{T}"
        policy_desc = "LargeModel (P=4052658, 18 actions)"
    else:
        net = nets.make_net("LargeModel")
        pop = args.pop
        n_units, G = pop // 2, 2
        slots_cap = args.slots
        label = f"frostbite_nsres_pop{pop}_LargeModel_T{T}_archive256"
        policy_desc = "LargeModel (P=4052658, 18 actions)"
    P = net.num_params
    lo, hi = shard.shard_bounds(n_units, rank, world)
    n_local = hi - lo
    slots = max(G, min(slots_cap, G * n_local))
    slots -= slots % G
    theta0 = (rs.randn(P) * 0.05).astype(np.float32)
    upd = ESUpdate(ctx, theta0, "adam", stepsize=LR)
    sf = SlotForward(ctx, net, slots)
    idx_stream = np.random.RandomState(1)
    if net.ob_kind == F.OB_ATARI_U8:
        pool = torch.randint(0, 256, (4, slots, 84, 84, 4), dtype=torch.uint8, device=dev)
        ob_mean = ob_std = None
    else:
        pool = torch.randn(4, slots, net.ob_dim, device=dev)
        ob_mean, ob_std = torch.zeros(net.ob_dim, device=dev), torch.ones(net.ob_dim, device=dev)
    rew_pool = (torch.rand(64, slots, device=dev) < 0.05).float() * 10.0
    ret_acc = torch.zeros(slots, device=dev)
    if wl == "ga":
        TP = 20
        parents = torch.from_numpy((rs.randn(TP, P) * 0.05).astype(np.float32)).to(dev)
        new_parents = torch.empty_like(parents)
        fit_all = torch.zeros(pop, device=dev)
        sel = torch.empty(TP, dtype=torch.int32, device=dev)
    if wl == "nsr":
        A, k, D = 256, 10, 128
        bc_pool = torch.randint(0, 256, (min(2 * n_local, 64), T, D), dtype=torch.uint8, device=dev)     # synthetic RAM traces
        arch = torch.randint(0, 256, (A, T, D), dtype=torch.uint8, device=dev)
        arch_len = torch.full((A,), T, dtype=torch.int32, device=dev)
        nb = C.c_size_t()
        F.check(L.dne_knn_ws_bytes(2 * max(n_local, 1), A, C.byref(nb)))
        knn_ws = torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)

    def rollout_wave(theta, unit_idx, scales, theta_idx, paired):
        """T ticks for one wave of units resident in the slot table; returns the per-slot returns."""
        n = len(unit_idx) * G
        act = np.zeros(slots, dtype=np.uint8)
        act[:n] = 1
        ii = np.zeros(slots, dtype=np.int64)
        ii[:n] = np.repeat(unit_idx, G)
        sf.set_slots(ii, scales, active=act if n < slots else None, theta_idx=theta_idx)
        ret_acc.zero_()
        for t in range(T):
            sf.forward(theta, pool[t & 3], paired=paired, ob_mean=ob_mean, ob_std=ob_std)
            ret_acc.add_(rew_pool[t & 63])
        tally["ticks"] += T
        tally["pairs"] += T * len(unit_idx)
        return ret_acc[:n].clone()

    def generation():
        if wl == "ga":
            seeds = np.array([noise.sample_index(idx_stream, P) for _ in range(pop)], dtype=np.int64)
            par = idx_stream.randint(0, TP, size=pop).astype(np.int32)
            my_s, my_p = seeds[lo:hi], par[lo:hi]
            fit = torch.zeros(n_local, device=dev)
            scales = np.full(slots, 0.002, dtype=np.float32)                      # ga_atari_config.json mutation_power
            for w0 in range(0, n_local, slots):
                w = my_s[w0:w0 + slots]
                tix = np.zeros(slots, dtype=np.int32)
                tix[:len(w)] = my_p[w0:w0 + slots]
                fit[w0:w0 + len(w)] = rollout_wave(parents, w, scales, tix, 0)
            allfit = shard.all_gather_rows(fit.view(-1, 1), pop).view(-1)
            F.check(L.dne_ga_truncate(F.ptr(allfit.contiguous()), pop, TP, F.ptr(sel), F.stream_ptr()))   # ga.py:145-149
            chosen = sel.cpu().numpy()
            for j, c in enumerate(chosen):                                         # new parents = parent + power * noise[seed]
                F.check(L.dne_ga_mutate(ctx.handle, F.ptr(parents[int(par[c])]), int(seeds[c]), 0.002, P,
                                        F.ptr(new_parents[j]), F.stream_ptr()))
            parents.copy_(new_parents)
            return
        idx_all = np.array([noise.sample_index(idx_stream, P) for _ in range(n_units)], dtype=np.int64)
        my = idx_all[lo:hi]
        returns = torch.zeros(n_local, 2, device=dev)
        sc = np.tile([SIGMA, -SIGMA], slots // 2).astype(np.float32)
        for w0 in range(0, n_local, slots // 2):
            w = my[w0:w0 + slots // 2]
            returns[w0:w0 + len(w)] = rollout_wave(upd.theta, w, sc, None, True).view(-1, 2)
        if wl == "nsr":
            q = 2 * n_local
            nov = torch.empty(max(q, 1), dtype=torch.float32, device=dev)
            if q:
                bc = bc_pool[torch.arange(q, device=dev) % bc_pool.shape[0]].contiguous()
                bl = torch.full((q,), T, dtype=torch.int32, device=dev)
                F.check(L.dne_knn_novelty(F.ptr(bc), F.ptr(bl), q, F.ptr(arch), F.ptr(arch_len), A, T, D, k, F.ptr(nov),
                                          F.ptr(knn_ws), knn_ws.numel(), F.stream_ptr()))
            pack = torch.cat([returns, nov[:q].view(-1, 2)], dim=1)
            allp = shard.all_gather_rows(pack, n_units)
            rew_rank, _ = upd.centered_ranks(allp[:, 0:2].contiguous())
            nov_rank, _ = upd.centered_ranks(allp[:, 2:4].contiguous())
            proc = (rew_rank + nov_rank) / 2.0                                     # nses.py:226-228
        else:
            allret = shard.all_gather_rows(returns, n_units)
            proc, _ = upd.centered_ranks(allret)
        g = upd.gradient(proc[lo:hi].contiguous(), torch.from_numpy(my).to(dev), denom=2 * n_units)
        shard.all_reduce_sum_(g)
        upd.step(L2)

    # ------------------------------------------------------------------------------------------------ timed region
    for _ in range(args.warmup):
        generation()
    torch.cuda.synchronize()
    shard.barrier()
    torch.cuda.synchronize()
    F.check(L.dne_profile_enable(ctx.handle, 1, 16384))
    L.dne_launch_count(1)
    tally.update(ticks=0, pairs=0)
    sampler = ClockSampler(local)
    if rank == 0:
        sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        generation()
    e1.record()
    torch.cuda.synchronize()
    shard.barrier()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    clocks = sampler.stop() if rank == 0 else None
    launches = L.dne_launch_count(0)
    n_t, tot = C.c_int(), C.c_double()
    F.check(L.dne_profile_enable(ctx.handle, 0, 0))
    F.check(L.dne_profile_read(ctx.handle, C.byref(n_t), C.byref(tot)))
    tt = torch.tensor([ms], dtype=torch.float64, device=dev)
    if world > 1:
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
    ms = float(tt.item())
    env_steps = args.steps * pop * T
    value = env_steps / (ms / 1e3)

    # roofline: the noise GEMV launches timed with CUDA events on their stream (dne_profile_*): algorithmic bytes = one
    # slice of every decomposed dense layer per launch group (pair-shared for ES; per offspring for GA, plus the parent rows
    # that the GA GEMV streams in a second launch -- not timed by the profile hook, so GA reports the noise launches only)
    dense = [l for l in net.layers[:-1] if l.kind == F.DENSE and l.cin * l.cout >= 16384]
    groups_per_tick = tally["pairs"] / max(tally["ticks"], 1)
    bytes_per_tick = groups_per_tick * sum(4.0 * l.cin * l.cout for l in dense)
    launches_per_tick = max(len(dense), 1)
    avg_ms = tot.value / max(n_t.value, 1)
    achieved = (bytes_per_tick / launches_per_tick) / (avg_ms * 1e-3) / 1e9 if n_t.value else None
    roofline = {"bound": "hbm", "kernel": "gemv_union_kernel (noise GEMV of the decomposed dense layers)",
                "achieved": achieved, "peak": peaks["hbm_gbs"], "peak_source": peak_src, "unit": "GB/s",
                "frac": achieved / peaks["hbm_gbs"] if achieved else None, "traffic": None,
                "launches_timed": n_t.value, "avg_launch_ms": avg_ms,
                "algorithmic_bytes_per_launch": bytes_per_tick / launches_per_tick,
                "whole_run_frac": args.steps * (tally["pairs"] / max(args.steps, 1)) * sum(4.0 * l.cin * l.cout for l in dense)
                                  / (ms * 1e-3) / 1e9 / peaks["hbm_gbs"],
                "note": "bytes = one noise slice of every decomposed dense layer per antithetic pair (es/nsr/mlp) or per "
                        "offspring (ga; the parent-row stream of the same size is a second, untimed launch)"}

    # ------------------------------------------------------------------------------------------------ e2e through the driver
    e2e = None
    if not args.no_e2e:
        from es_distributed import es as ES, ga as GA, nses as NS, tabular_logger
        from dne.envs import SyntheticAtariEnv, SyntheticVectorEnv
        tabular_logger.set_quiet(True)
        ES.set_default_noise(noise)
        ES._STATE["ctx"] = ctx
        cfg = {"calc_obstat_prob": 0.0, "episodes_per_batch": pop, "eval_prob": 0.0, "l2coeff": L2, "noise_stdev": SIGMA,
               "snapshot_freq": 0, "timesteps_per_batch": 1, "return_proc_mode": "centered_rank", "episode_cutoff_mode": T}
        s4 = max(4, -(-slots // 4) * 4)
        marks, io = {}, {"ticks": 0}

        def on_it(it, stats, extra):
            if it == args.warmup or it == args.warmup + args.steps:
                torch.cuda.synchronize()
                shard.barrier()
                torch.cuda.synchronize()
                marks[it] = time.perf_counter()
        kw = dict(max_iterations=args.warmup + args.steps, n_slots=s4, noise=noise, seed=0, on_iteration=on_it)
        if args.warmup == 0:         # run_master numbers its iterations from 1: without warm-up the window opens here
            on_it(0, None, None)
        if wl == "mlp":
            exp = {"config": cfg, "env_id": "SyntheticVectorHumanoid", "optimizer": {"args": {"stepsize": LR}, "type": "adam"},
                   "policy": {"args": {"ac_bins": "continuous:", "ac_noise_std": 0.0, "connection_type": "ff",
                                       "hidden_dims": [256, 256], "nonlin_type": "tanh"}, "type": "MujocoPolicy"}}
            ES.run_master(None, None, exp, env=SyntheticVectorEnv(s4, episode_len=T, seed=rank), **kw)
            ob_bytes, api = net.ob_dim * 4, "es_distributed.es.run_master + SyntheticVectorEnv"
        elif wl == "ga":
            exp = {"config": cfg, "env_id": "SyntheticAtari", "population_size": 20, "num_elites": 1, "ga_mode": "gpu",
                   "policy": {"args": {}, "type": "LargeModelPolicy"}}
            GA.run_master(None, None, exp, env=SyntheticAtariEnv(s4, episode_len=T, seed=rank), **kw)
            ob_bytes, api = 84 * 84 * 4, "es_distributed.ga.run_master + SyntheticAtariEnv"
        else:
            exp = {"config": dict(cfg, return_proc_mode="centered_sign_rank"), "env_id": "SyntheticAtari", "algo_type": "nsr",
                   "novelty_search": {"k": 10, "population_size": 1, "num_rollouts": 1, "selection_method": "round_robin"},
                   "optimizer": {"args": {"stepsize": LR}, "type": "adam"}, "policy": {"args": {}, "type": "LargeModelPolicy"}}
            NS.run_master(None, None, exp, env=SyntheticAtariEnv(s4, episode_len=T, seed=rank), **kw)
            ob_bytes, api = 84 * 84 * 4, "es_distributed.nses.run_master + SyntheticAtariEnv (RAM-trace BCs, archive grows from 1)"
        dt = marks[args.warmup + args.steps] - marks[args.warmup]
        t2 = torch.tensor([dt], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t2, op=dist.ReduceOp.MAX)
        dt = float(t2.item())
        per_rank_steps = pop * T / world
        e2e = {"value": env_steps / dt, "unit": "env-steps/s", "ms_per_step": dt * 1e3 / args.steps,
               "h2d_bytes_per_step": int(per_rank_steps * ob_bytes), "d2h_bytes_per_step": int(per_rank_steps * 4 * (17 if wl == "mlp" else 1)),
               "bytes_scope": "one rank's copies per generation", "api": api}

    if rank == 0:
        emit({"metric": "env-steps/sec across the population (whole box)", "value": value, "unit": "env-steps/s",
              "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps,
              "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
              "config": {"workload": label, "population": pop, "policy": policy_desc, "env_slots_per_gpu": slots,
                         "episode_len": T, "noise_table": args.noise_count,
                         "sharding": f"population over {world} rank(s)",
                         "l2": "inputs larger than L2 (every tick streams the population's noise slices)",
                         "step": "one generation (rollouts + selection / update)"},
              "generation_wall_clock_s": ms / args.steps / 1e3, "e2e": e2e, "gpu_launches": int(launches), "clocks": clocks,
              "roofline": roofline, "cpu_baseline": None})
    if world > 1:
        dist.destroy_process_group()


def run_gpu_ref_proxy(args, emit, ClockSampler):
    """--impl gpu-ref-proxy: a PROXY of the reference's GPU schedule (gpu_implementation/) on this GPU, for the
    north_star's "vs gpu_implementation" denominator.  TensorFlow, the gym_tensorflow ops and ALE are absent, so this is not
    the reference itself; it reproduces the schedule's data movement with library kernels (torch -> cuBLAS batched GEMM):
      * every member's FULL weight vector is materialised in device memory and (re)loaded by a 4*P-byte host->device copy
        per member and episode (neuroevolution/models/base.py:158-192 `load` -> scatter_update; concurrent_worker.py:72-102),
      * per tick one batched matmul per layer over all resident members -- the conv layers as extract_image_patches +
        batched matmul, the dense layers as batched mat-vec (gym_tensorflow/ops/indexedmatmul.cpp:169-202: SgemmBatched over
        host-built pointer arrays; models/base.py:54-99) -- i.e. every member streams its own 16.2 MB of weights per tick
        (no antithetic sharing, no split of theta and noise),
      * argmax on the device, synthetic observations / rewards resident in HBM (as in the gpu arm's `value`).
    What it leaves out (all in the reference's disfavour): TF op dispatch, the per-call host pointer-array build + H2D,
    the CPU env thread pool, the master's numpy update.  So it is a LOWER bound on the reference schedule's time here."""
    import torch
    import torch.nn.functional as Fn
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    T, pop, slots = args.episode_len, args.pop, args.slots
    shapes = [(8, 4, 32, 4, 2, 2), (4, 32, 64, 2, 1, 2), (3, 64, 64, 1, 1, 1)]       # k, cin, cout, stride, pad_before, pad_after
    sizes = [8 * 8 * 4 * 32, 32, 4 * 4 * 32 * 64, 64, 3 * 3 * 64 * 64, 64, 7744 * 512, 512, 512 * 18, 18]
    P = sum(sizes)
    W = torch.randn(slots, P, device=dev) * 0.05                                     # [members, P]: materialised weights
    host = [torch.randn(P).pin_memory() for _ in range(8)]                          # rotating pinned sources of the member loads
    offs = np.cumsum([0] + sizes)
    pool = torch.randint(0, 256, (4, slots, 84, 84, 4), dtype=torch.uint8, device=dev)
    rew = (torch.rand(64, slots, device=dev) < 0.05).float() * 10.0
    ret = torch.zeros(slots, device=dev)

    def view(i, *shape):
        return W[:, offs[i]:offs[i + 1]].view(slots, *shape)

    def tick(t):
        x = pool[t & 3].permute(0, 3, 1, 2).float() / 255.0                          # NCHW
        for li, (k, cin, cout, s, pb, pa) in enumerate(shapes):
            xp = Fn.pad(x, (pb, pa, pb, pa))
            patches = Fn.unfold(xp, k, stride=s)                                     # [B, cin*k*k, L]  (extract_image_patches)
            L_ = patches.shape[-1]
            patches = patches.view(slots, cin, k * k, L_).permute(0, 3, 2, 1).reshape(slots, L_, k * k * cin)   # (ky,kx,ci) order
            y = torch.baddbmm(view(2 * li + 1, 1, cout), patches, view(2 * li, k * k * cin, cout))             # batched matmul
            h = int(round(L_ ** 0.5))
            x = torch.relu(y).view(slots, h, h, cout).permute(0, 3, 1, 2)
        f = x.permute(0, 2, 3, 1).reshape(slots, 1, 7744)
        hdn = torch.relu(torch.baddbmm(view(7, 1, 512), f, view(6, 7744, 512)))
        logits = torch.baddbmm(view(9, 1, 18), hdn, view(8, 512, 18))
        return logits.argmax(dim=-1)

    def generation():
        for w0 in range(0, pop, slots):
            n = min(slots, pop - w0)
            for m in range(n):                                                       # models/base.py:158-192: one load per member
                W[m].copy_(host[m & 7], non_blocking=True)
            ret.zero_()
            for t in range(T):
                tick(t)
                ret.add_(rew[t & 63])

    for _ in range(args.warmup):
        generation()
    torch.cuda.synchronize()
    sampler = ClockSampler(0)
    sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        generation()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    clocks = sampler.stop()
    v = args.steps * pop * T / (ms / 1e3)
    emit({"impl": "gpu-ref-proxy", "metric": "env-steps/sec across ES population (whole box)", "value": v, "unit": "env-steps/s",
          "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True,
          "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
          "config": {"workload": f"frostbite_es_pop{pop}_LargeModel_T{T}", "population": pop, "env_slots_per_gpu": slots,
                     "policy": "LargeModel (P=4052658, 18 actions)", "episode_len": T,
                     "schedule": "reference GPU path proxy: materialised per-member weights, 4*P-byte H2D per member-episode, "
                                 "5 cuBLAS batched matmuls per tick (torch.baddbmm), no update step"},
          "clocks": clocks, "weights_streamed_per_tick_GB": slots * P * 4 / 1e9,
          "note": "PROXY, not the reference (TensorFlow / gym_tensorflow / ALE absent): lower bound of the reference GPU "
                  "schedule's time on this GPU; see bench_workloads.run_gpu_ref_proxy"})
