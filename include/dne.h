/* dne.h -- C ABI of libdne.so: the sm_90a ES/GA rollout-and-update engine.
 *
 * The reference (uber-research/deep-neuroevolution) is Python and has no C ABI for this path; its
 * "plugin boundary" is (a) the Python API es_distributed.{es,ga,nses}.run_master/run_worker +
 * policies.Policy + SharedNoiseTable and (b) on its GPU path the TF custom-op registry
 * (gpu_implementation/gym_tensorflow/ops/indexedmatmul.cpp:303-344).  Each entry point below names the
 * reference code it replaces (paths relative to the reference root).  The Python host side
 * (deep-neuroevolution_b200/dne/_ffi.py) binds exactly these symbols through ctypes; INTEGRATION.md shows
 * the stub a reference maintainer would add.
 *
 * Conventions
 *   - every call returns int: 0 = ok, <0 = error (text via dne_last_error(), thread-local); never throws,
 *     never aborts.
 *   - device pointers are BORROWED (the caller -- torch -- owns and frees them).  Kernels are enqueued
 *     on the caller's cudaStream_t (passed as void*) and the call returns without synchronising.
 *   - no hidden allocation on the hot path: workspaces are passed in; sizes come from the *_ws_bytes
 *     queries.  A dne_ctx owns only a small fixed scratch buffer allocated at creation.
 *   - one host thread per context; handles are not thread-safe.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails with
 *     DNE_ERR_CUDA.
 */
#ifndef DNE_H_
#define DNE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DNE_OK            0
#define DNE_ERR_ARG      -1
#define DNE_ERR_CUDA     -2
#define DNE_ERR_WS       -3   /* workspace too small */
#define DNE_ERR_UNSUP    -4   /* layer shape not supported by the compiled kernels */

#define DNE_MAX_LAYERS    8

/* layer kinds / activations / batch-norm flavours */
#define DNE_CONV   0
#define DNE_DENSE  1
#define DNE_ACT_NONE 0
#define DNE_ACT_RELU 1
#define DNE_ACT_TANH 2
#define DNE_BN_NONE 0
#define DNE_BN_TF   1          /* contrib.layers.batch_norm(scale=True, decay=0, eps=1e-3): policies.py:322 */
#define DNE_BN_GPU  2          /* ModelVirtualBN (gpu_implementation/neuroevolution/models/batchnorm.py:64-93): layer without
                                  bias, (x - mean) / sqrt(var + 1e-3) + b, no gamma; off_b is that post-normalisation bias */

/* observation kinds */
#define DNE_OB_ATARI_U8 0      /* uint8 [slots,84,84,4], scaled by 1/255 (atari_wrappers.py:186) */
#define DNE_OB_VECTOR   1      /* float32 [slots,ob_dim], clip((o-mean)/std,-5,5) (policies.py:151); without
                                  statistics (d_ob_mean NULL) used as given, unclipped */

typedef struct dne_layer_desc {
    int32_t kind;              /* DNE_CONV | DNE_DENSE */
    int32_t cin, cout;         /* conv: channels; dense: fan-in / fan-out */
    int32_t ksize, stride;     /* conv only (square kernel) */
    int32_t hin, hout, pad;    /* conv only: square input/output size, TF-SAME pad_before */
    int32_t act;               /* DNE_ACT_* */
    int32_t bn;                /* DNE_BN_* */
    int32_t bn_off;            /* offset of this layer's (mean[cout], var[cout]) in a slot's vbn stats vector */
    int32_t _pad;
    int64_t off_w, off_b;      /* element offsets into the flat parameter vector; off_b < 0: no bias */
    int64_t off_beta, off_gamma; /* bn == DNE_BN_TF only */
} dne_layer_desc;

/* Flat layout = variable creation order of the reference policy (tf_util.py:224-246;
 * gpu_implementation/neuroevolution/models/base.py:165-192). */
typedef struct dne_net_desc {
    int32_t n_layers;
    int32_t ob_kind;           /* DNE_OB_* */
    int32_t ob_dim;            /* DNE_OB_VECTOR: observation length; ATARI: 84*84*4 */
    int32_t n_out;             /* logits / action dimension */
    int32_t vbn_len;           /* floats of virtual-batch-norm statistics per slot (0 if none) */
    int32_t _pad;
    int64_t num_params;
    dne_layer_desc layers[DNE_MAX_LAYERS];
} dne_net_desc;

typedef struct dne_ctx dne_ctx;

/* ---- context ------------------------------------------------------------------------------------ */
int         dne_ctx_create(int device, dne_ctx** out);
int         dne_ctx_destroy(dne_ctx* ctx);
const char* dne_last_error(void);
int         dne_version(void);
/* ABI self-check for FFI bindings: sizeof(dne_layer_desc), sizeof(dne_net_desc). */
int         dne_abi_sizes(int* layer_desc_bytes, int* net_desc_bytes);
/* The same for sizeof(dne_maze_desc). */
int         dne_abi_maze_size(int* maze_desc_bytes);

/* ---- measurement hooks (bench.py) -------------------------------------------------------------------
 * dne_launch_count: kernels launched by this library in this process so far (reset != 0 zeroes it).
 * dne_profile_enable/read: CUDA-event timing of every launch of the dominant HBM-bound kernel
 * (dense_noise_gemv) on the stream it is launched on; read() synchronises the device. */
long long   dne_launch_count(int reset);
/* Runtime switches (process-wide; A/B measurement and referee paths only):
 *   "conv_tc" = 2 (default): shifted-window wgmma convolutions, images / weights by TMA (conv_s2d.cu), also used by the
 *               virtual-batch-norm reference pass; 1: im2col-staged wgmma tf32 convolutions (tc_conv.cu); 0: fp32 SIMT
 *               kernels everywhere (the parity referee).
 *   "theta_tma" = 1 (default): TMA-fed shared-theta GEMM when a prepared region is current (dne_theta_prepare).
 *   "theta_mc" = 0 (default): cluster-multicast variant of it (measured slower).
 *   "fuse_head" = 1 (default): combine + output head + argmax in one kernel.
 *   "fold_theta" = 1 (default): the theta GEMM's split-K partials are folded into the noise GEMV's output.
 *   "pdl" = 1 (default): the tick's kernels are chained by programmatic dependent launch (griddepcontrol).
 *   "chain_ticks" = 0 (default): 1 = the tick's first convolution is a dependent launch too; only valid when the stream's
 *               previous kernel is the previous tick's last kernel (nothing that writes theta / the noise table / the slot table).
 *   "gemv_bulk" = 1 (default): the dense layers' GEMV streams the union of the slot table's slices once, through the
 *               cp.async.bulk shared-memory ring; 0 = plain-LDG kernel, one slice per group (the parity referee).
 *   "gemv_ctas_per_sm" = 1|2 (default 2), "gemv_stages" = 2..8 (default 5, upper bound on the ring depth that fits),
 *   "gemv_grid" (default 0 = no cap). */
int         dne_set_option(const char* name, int value);
int         dne_profile_enable(dne_ctx* ctx, int on, int capacity);
int         dne_profile_read(dne_ctx* ctx, int* n_launches, double* total_ms);

/* Replaces SharedNoiseTable (es_distributed/es.py:51-67): the table lives in HBM; `count` floats, the
 * allocation must extend at least 8 floats past `count` (aligned vector loads of unaligned slices). */
int dne_noise_bind(dne_ctx* ctx, const float* d_noise, int64_t count);

/* ---- rollout side ------------------------------------------------------------------------------- */
/* Bytes of workspace dne_perturb_forward_* needs for `n_slots` slots of `net`. */
int dne_forward_ws_bytes(const dne_net_desc* net, int n_slots, size_t* out_bytes);

/* Replaces, per env tick and for all slots at once:
 *   v = noise_stdev*noise.get(idx,P); policy.set_trainable_flat(theta +/- v)   (es.py:412-419)
 *   policy.act(ob)  -> conv/dense forward + argmax                              (policies.py:319-330,403,449-459;
 *                                                                                models/dqn.py:25-47; indexedmatmul.cpp:148-213)
 * Slot s evaluates weights theta + d_scale[s]*noise[d_noise_idx[s] : +P] (never materialised in HBM).
 * paired == 1 asserts slots (2p, 2p+1) share d_noise_idx (antithetic pair): the slice is then read once.
 * paired == 2 asserts slots (2p, 2p+1) share d_theta_idx (GA siblings of one parent): the parent row is read once.
 * d_theta_idx (nullable): per-slot row into d_theta [n_theta, P] (GA parents); NULL = row 0 for every slot.
 * d_active (nullable): uint8 per slot; inactive slots are skipped and their outputs left untouched.
 * d_vbn: per-slot virtual-batch-norm statistics from dne_vbn_reference_pass (NULL if the net has none).
 * Outputs: d_actions int32[n_slots] (argmax, first max on ties), d_logits float[n_slots, n_out] (nullable). */
int dne_perturb_forward_conv(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                             const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                             const uint8_t* d_active, int n_slots, int paired,
                             const uint8_t* d_obs, const float* d_vbn,
                             int32_t* d_actions, float* d_logits,
                             void* d_ws, size_t ws_bytes, void* stream);

/* Optional, once per generation: relays out the shared weight matrices of the net's large dense layers
 * (theta_w[K, N] of the fc layer: the x . theta_w half of x . (theta_w + s*noise), policies.py:327 / dqn.py:46) into the
 * workspace in the tensor-core operand layout (TF32 hi / lo planes), so that the following dne_perturb_forward_conv calls
 * on the SAME (d_ws, d_theta, n_slots) feed that GEMM by TMA instead of staging it through threads.  The entry stays
 * current until dne_adam_step / dne_sgd_step on this context rewrite d_theta (they drop it themselves); after any OTHER
 * write to d_theta call it again.  Without a current entry the forward is still correct (thread-staged GEMM). */
int dne_theta_prepare(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta, int n_slots, void* d_ws, size_t ws_bytes,
                      void* stream);
/* Entries are keyed by the workspace ADDRESS: forget them when a workspace is allocated or freed (an allocator may hand a
 * freed workspace's address to a new one).  d_ws == NULL forgets every entry of the context. */
int dne_theta_forget(dne_ctx* ctx, const void* d_ws);

/* Phase-shifted double buffering of two slot tables on two CUDA streams: the NEXT dne_perturb_forward_* call on ctx
 * makes its stream wait for wait_event (cudaEvent_t, nullable) before its first kernel and records record_event
 * (nullable) right before its first HBM-bound noise GEMV.  Table A: (wait eB, record eA); table B: (wait eA, record eB):
 * the tensor-core conv phase of one table then runs under the HBM-bound phase of the other (mode 0).
 * mode 1 instead waits right before the GEMV and records right after it: the tables take turns on the memory system
 * while their conv chains free-run (use with >= 3 tables). */
int dne_set_phase_events(dne_ctx* ctx, void* wait_event, void* record_event, int mode);

/* MujocoPolicy variant (policies.py:150-162,195-196,202-206): float observations, ob normalisation, tanh MLP,
 * continuous head.  d_actions_out float[n_slots, n_out] (action noise is added by the caller's stream).
 * d_ob_mean / d_ob_std (both or neither): the layer input is clip((o - mean) / std, -5, 5).  Both NULL: the
 * observations are fed as they are, NOT clipped (SimpleClassifier / LinearClassifier, models/simple.py: no
 * normalisation).  A MujocoPolicy always passes statistics (mean 0 / std 1 before its first set_ob_stat).
 * Dense layers of any width run; an output wider than 256 has no argmax (dne_perturb_forward_conv: DNE_ERR_UNSUP). */
int dne_perturb_forward_mlp(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                            const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                            const uint8_t* d_active, int n_slots, int paired,
                            const float* d_obs, const float* d_ob_mean, const float* d_ob_std,
                            float* d_actions_out, void* d_ws, size_t ws_bytes, void* stream);

/* CartPole-v1 (gym classic_control) episodes run entirely on the device, one per member:
 * weights theta[d_theta_idx[m] or 0] + d_scale[m]*noise[d_noise_idx[m] : +P], initial state d_init_state[m][4] (float64),
 * at most max_steps steps.  Outputs d_returns float[n], d_lengths int32[n], d_final_state double[n][4] (nullable:
 * state after the last step -- the 'final' behaviour characterisation).  Enqueued on `stream`, no host sync.
 * Supported nets (SimpleClassifier / LinearClassifier shapes): 1..4 dense layers of width <= 32, DNE_OB_VECTOR with
 * ob_dim 4, n_out 2, ReLU hidden layers, linear head, no batch norm; anything else returns DNE_ERR_UNSUP.
 * Observation = (float)state; action = argmax of the logits (first max on ties, NaN counts as the maximum); the
 * environment step is float64 in gym's operation order; return = length (reward 1 per step). */
int dne_cartpole_episodes(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                          const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                          int n_members, const double* d_init_state, int max_steps,
                          float* d_returns, int32_t* d_lengths, double* d_final_state, void* stream);

/* gym's discrete-action classic_control tasks, whole episodes on the device (DESIGN.md 3.5) */
#define DNE_EPISODE_CARTPOLE    0      /* CartPole-v1:    state (x, x_dot, theta, theta_dot), ob_dim 4, 2 actions, 500 steps */
#define DNE_EPISODE_ACROBOT     1      /* Acrobot-v1:     state (theta1, theta2, dtheta1, dtheta2), ob_dim 6, 3 actions, 500 */
#define DNE_EPISODE_MOUNTAINCAR 2      /* MountainCar-v0: state (position, velocity), ob_dim 2, 3 actions, 200 */

/* dne_cartpole_episodes for any DNE_EPISODE_* task `env`: the same arguments, with d_init_state / d_final_state
 * double[n][state_dim] (4, 4, 2) and 1 <= max_steps <= the task's TimeLimit (else DNE_ERR_ARG).  Observation: float32 of
 * the task's observation vector; action: the first NaN logit if any, otherwise the first maximum; d_returns: the float64
 * rewards (+1 per CartPole step; -1 per Acrobot step, 0 on the terminating one; -1 per MountainCar step) summed in step
 * order and rounded to float32 once.  Supported nets: 1..4 dense layers of width <= 32, DNE_OB_VECTOR with the task's
 * ob_dim, n_out = its action count, ReLU hidden layers, linear head, no batch norm; anything else returns DNE_ERR_UNSUP
 * with the reason in dne_last_error(). */
int dne_discrete_episodes(dne_ctx* ctx, int env, const dne_net_desc* net, const float* d_theta,
                          const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                          int n_members, const double* d_init_state, int max_steps,
                          float* d_returns, int32_t* d_lengths, double* d_final_state, void* stream);

/* Pendulum-v1 (gymnasium classic_control pendulum.py, DESIGN.md 3.6) episodes run entirely on the device, one per member,
 * for MujocoPolicy 'continuous:' nets.  Weights as dne_cartpole_episodes; initial state d_init_state[m] = (th, thdot)
 * (float64); exactly max_steps (1..200) steps, there is no termination.  Per step: observation float32(cos th, sin th,
 * thdot); layer input clip((o - mean) / std, -5, 5) with d_ob_mean / d_ob_std (both or neither, as
 * dne_perturb_forward_mlp); fp32 dense forward (sequential fmaf per output, then + bias; tanh / ReLU hidden layers,
 * linear head); action = head + d_ac_noise[m][step] (nullable [n][max_steps][1], already scaled); the float64 step.
 * Outputs: d_returns / d_signreturns float[n] (float32 rewards summed in float64 in step order, rounded once),
 * d_lengths int32[n] (= max_steps), d_final_state double[n][2] (nullable: the 'final' behaviour characterisation),
 * d_ob_sum / d_ob_sumsq double[n][3] (both or neither: per-member float64 sums of the unnormalised observations fed to
 * the forward, dne_ob_stat_accumulate's formula, in step order).  Enqueued on `stream`, no host sync.
 * Supported nets: 1..DNE_MAX_LAYERS dense layers of any width, DNE_OB_VECTOR with ob_dim 3, n_out 1, tanh or ReLU hidden layers, a
 * linear head, no batch norm, and one member's weights plus two activation buffers in one CTA's shared memory (227 KB:
 * hidden [200, 200] runs, [256, 256] does not: dne_pendulum_cluster_episodes runs it); anything else returns
 * DNE_ERR_UNSUP with the reason in dne_last_error().
 * dne_pendulum_net_supported answers the same question without launching (0 or DNE_ERR_UNSUP). */
int dne_pendulum_net_supported(const dne_net_desc* net);
int dne_pendulum_episodes(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                          const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx, int n_members,
                          const double* d_init_state, int max_steps, const float* d_ob_mean, const float* d_ob_std,
                          const float* d_ac_noise, float* d_returns, float* d_signreturns, int32_t* d_lengths,
                          double* d_final_state, double* d_ob_sum, double* d_ob_sumsq, void* stream);

/* The hard maze of the reference's GPU path (gym_tensorflow/maze: maze.h stepped as tf_maze.cpp does; DESIGN.md 3.7):
 * the walls as segments (ax, ay, bx, by), at most DNE_MAZE_MAX_WALLS; the goal; the maze file's collision flag (nonzero:
 * a collision freezes the navigator for the rest of the episode; 0 in the hard maze). */
#define DNE_MAZE_MAX_WALLS 64
typedef struct {
    int32_t n_walls;
    int32_t collisions_stick;
    float goal[2];
    float walls[DNE_MAZE_MAX_WALLS][4];
} dne_maze_desc;

/* Hard-maze episodes run entirely on the device, one per member, for MujocoPolicy 'continuous:' nets.  Arguments as
 * dne_pendulum_episodes, with: d_init_state / d_final_state double[n][7] = (x, y, heading, speed, ang_vel, t, collided),
 * float32 values and t the steps already taken (the reset state is (start, 0, 0, 0, 0, 0)); 1 <= max_steps <= 400;
 * observation float32[11] = (1, the 6 rangefinders / 100, the 4 goal-radar sectors); action = head[2] +
 * d_ac_noise[m][step][0..1] (nullable [n][max_steps][2]), stepped as interpret_outputs(a0 + 0.5, a1 + 0.5) and Update();
 * the reward is 0, and -distance to the goal on the step on which t reaches 400 (a shorter episode pays 0);
 * d_ob_sum / d_ob_sumsq double[n][11].  The final (x, y) is the reference's MazeFinalState behaviour characterisation.
 * `maze` with n_walls outside 0..DNE_MAZE_MAX_WALLS returns DNE_ERR_ARG.  Supported nets: as dne_pendulum_episodes with
 * ob_dim 11 and n_out 2; anything else returns DNE_ERR_UNSUP with the reason in dne_last_error(), and
 * dne_maze_net_supported answers the same question without launching (0 or DNE_ERR_UNSUP). */
int dne_maze_net_supported(const dne_net_desc* net);
int dne_maze_episodes(dne_ctx* ctx, const dne_maze_desc* maze, const dne_net_desc* net, const float* d_theta,
                      const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx, int n_members,
                      const double* d_init_state, int max_steps, const float* d_ob_mean, const float* d_ob_std,
                      const float* d_ac_noise, float* d_returns, float* d_signreturns, int32_t* d_lengths,
                      double* d_final_state, double* d_ob_sum, double* d_ob_sumsq, void* stream);

/* Pendulum-v1 and hard-maze episodes for nets too wide for one CTA (MujocoPolicy's hidden [256, 256]; DESIGN.md 3.8):
 * one member per thread-block cluster of `cluster` CTAs, its hidden layers' outputs dealt to the CTAs in contiguous
 * slices and the activations exchanged through distributed shared memory.  Arguments, outputs and numerics as
 * dne_pendulum_episodes / dne_maze_episodes, plus `cluster`: 0 picks the size with the most members resident on the
 * device (the smaller on a tie), 2, 4 or 8 forces it; anything else returns DNE_ERR_ARG, and a forced size whose slices
 * do not fit a CTA returns DNE_ERR_UNSUP.  Every operation is the single-CTA kernel's, so for a net both run the
 * outputs are bit-identical at every cluster size.  Supported nets: as dne_pendulum_episodes / dne_maze_episodes, with
 * the size limit on one CTA's slice at cluster size 8 (hidden [256, 256] and [512, 512] run, [2048, 2048] does not);
 * anything else returns DNE_ERR_UNSUP with the reason in dne_last_error().  dne_*_cluster_net_supported answers the same
 * question without launching (0 or DNE_ERR_UNSUP).  The existing entry points above are unchanged: they still refuse a
 * net that does not fit one CTA. */
int dne_pendulum_cluster_net_supported(const dne_net_desc* net);
int dne_maze_cluster_net_supported(const dne_net_desc* net);
int dne_pendulum_cluster_episodes(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                                  const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                  int n_members, const double* d_init_state, int max_steps, const float* d_ob_mean,
                                  const float* d_ob_std, const float* d_ac_noise, float* d_returns, float* d_signreturns,
                                  int32_t* d_lengths, double* d_final_state, double* d_ob_sum, double* d_ob_sumsq,
                                  int cluster, void* stream);
int dne_maze_cluster_episodes(dne_ctx* ctx, const dne_maze_desc* maze, const dne_net_desc* net, const float* d_theta,
                              const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx, int n_members,
                              const double* d_init_state, int max_steps, const float* d_ob_mean, const float* d_ob_std,
                              const float* d_ac_noise, float* d_returns, float* d_signreturns, int32_t* d_lengths,
                              double* d_final_state, double* d_ob_sum, double* d_ob_sumsq, int cluster, void* stream);
/* The launch geometry those entries use for `net` and `cluster` on the current device: geometry[4] = (cluster size,
 * threads per CTA, dynamic shared memory bytes per CTA, members resident on the device at once by
 * cudaOccupancyMaxActiveClusters).  Errors as the episode entries. */
int dne_pendulum_cluster_geometry(const dne_net_desc* net, int cluster, int* geometry);
int dne_maze_cluster_geometry(const dne_net_desc* net, int cluster, int* geometry);

/* Pendulum-v1 and hard-maze episodes for MujocoPolicy's discretised heads ('uniform:N', 'custom:v0,..,vk'; DESIGN.md
 * 3.9), with adim = 1 (Pendulum) or 2 (maze) action dimensions of n_bins bins each.  Arguments, outputs and numerics as
 * dne_*_cluster_episodes, plus bin_values_host, the policy's float32 table [adim][n_bins] on the HOST (copied into the
 * launch), and n_bins.  Per step the net's n_out = adim * n_bins outputs are scores, each a sequential fmaf over its
 * inputs in index order, then + bias; score d * n_bins + b is bin b of action dimension d.  For each dimension the bin
 * taken is the first one whose score is NaN if any is, otherwise the first maximum (numpy's argmax); the action is
 * a[d] = bin_values_host[d][bin], then + d_ac_noise[m][step][d] (nullable [n][max_steps][adim]: the noise is added after
 * the discretisation, and has adim, not n_out, components).  The task's step (Pendulum's clip, the maze's rate limits),
 * the observation normalisation and sums, returns, sign-returns and final states are the continuous entries'.
 * cluster 0 runs one member per CTA group when it fits one CTA and otherwise picks the cluster size as
 * dne_*_cluster_episodes does; 2, 4 or 8 force a cluster of that size (the outputs are bit-identical either way);
 * anything else returns DNE_ERR_ARG.  A NULL bin_values_host returns DNE_ERR_ARG.  Supported: 2 <= n_bins <= 32,
 * n_out = adim * n_bins, and otherwise the nets dne_*_cluster_net_supported takes; anything else returns DNE_ERR_UNSUP
 * with the reason in dne_last_error().  dne_*_binned_net_supported answers the same question without launching (0 or
 * DNE_ERR_UNSUP).  The continuous entries above are unchanged and still refuse n_out != adim. */
int dne_pendulum_binned_net_supported(const dne_net_desc* net, int n_bins);
int dne_maze_binned_net_supported(const dne_net_desc* net, int n_bins);
int dne_pendulum_binned_episodes(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                                 const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                 int n_members, const double* d_init_state, int max_steps, const float* d_ob_mean,
                                 const float* d_ob_std, const float* d_ac_noise, float* d_returns, float* d_signreturns,
                                 int32_t* d_lengths, double* d_final_state, double* d_ob_sum, double* d_ob_sumsq,
                                 const float* bin_values_host, int n_bins, int cluster, void* stream);
int dne_maze_binned_episodes(dne_ctx* ctx, const dne_maze_desc* maze, const dne_net_desc* net, const float* d_theta,
                             const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx, int n_members,
                             const double* d_init_state, int max_steps, const float* d_ob_mean, const float* d_ob_std,
                             const float* d_ac_noise, float* d_returns, float* d_signreturns, int32_t* d_lengths,
                             double* d_final_state, double* d_ob_sum, double* d_ob_sumsq, const float* bin_values_host,
                             int n_bins, int cluster, void* stream);

/* The hard maze seen from above as an 84x84 uint8 image (DESIGN.md 3.10), stepped one tick at a time for the Atari conv
 * policies.  The dynamics are dne_maze_episodes' (the same device code); the image is this project's own rendering rule:
 * the walls' bounding box mapped uniformly onto 84x84 (aspect kept, anchored at the lower bounds, row = y), each pixel
 * tested at its centre; 255 where a wall lies within half a pixel, 0 elsewhere; the navigator a disc of radius 8 maze
 * units over that, 64 on its front half (towards the heading) and 128 on the back.  The goal is not drawn.
 * Every entry takes `maze` with 1..DNE_MAZE_MAX_WALLS walls spanning a nonzero area (else DNE_ERR_ARG).
 * dne_image_maze_background  the walls alone into d_plane uint8 [84][84]: once per maze.
 * dne_image_maze_reset       for e < k: d_state[d_slots[e]] = d_init[e] (double[7], dne_maze_episodes' state layout),
 *                            and all four planes of d_stacks[d_slots[e]] (uint8 [84][84][4], NHWC) set to its frame.
 * dne_image_maze_step        for e < k: slot d_slots[e] steps with action row d_actions[e] of actions_host (the HOST
 *                            table float32 [n_actions][2] = (turn, speed), copied into the launch; an index outside
 *                            0..n_actions-1 steps as row 0), exactly as dne_maze_episodes steps a head output;
 *                            d_reward[e] float32 (0, and -distance to the goal on the 400th step), d_done[e] = (t >= 400),
 *                            d_pos[e] double[2] = the new (x, y) (nullable); the new frame is appended to the slot's
 *                            stack as plane 3 after planes 1..3 move to 0..2.
 * d_background is dne_image_maze_background's plane for the same maze.  The listed slots must be distinct.  Enqueued on
 * `stream`, no host sync. */
#define DNE_IMAGE_MAZE_MAX_ACTIONS 32
int dne_image_maze_background(const dne_maze_desc* maze, uint8_t* d_plane, void* stream);
int dne_image_maze_reset(const dne_maze_desc* maze, const uint8_t* d_background, const double* d_init,
                         const int32_t* d_slots, int k, double* d_state, uint8_t* d_stacks, void* stream);
int dne_image_maze_step(const dne_maze_desc* maze, const uint8_t* d_background, const float* actions_host, int n_actions,
                        const int32_t* d_slots, const int32_t* d_actions, int k, double* d_state, uint8_t* d_stacks,
                        float* d_reward, uint8_t* d_done, double* d_pos, void* stream);

/* Observation statistics of the running normaliser (es.py:356-363 rollout_and_update_ob_stat; RunningStat es.py:26-48):
 * adds the observations d_obs[slot, :] (float32 [*, ob_dim], the unnormalised vectors fed to this tick's forward) of the m
 * listed slots -- the slots whose episode was sampled with probability calc_obstat_prob -- into float64 running sums
 * d_sum[ob_dim], d_sumsq[ob_dim].  The episode count stays with the caller (m per tick). */
int dne_ob_stat_accumulate(const float* d_obs, int ob_dim, const int32_t* d_slots, int m, double* d_sum, double* d_sumsq,
                           void* stream);

/* Virtual batch norm reference pass, per member before each episode (policies.py:322-328,399;
 * es.py:105-113): forwards the shared reference batch d_ref [n_ref,84,84,4] through every listed slot's
 * perturbed weights with batch statistics and stores (mean, biased var) per BN layer in d_vbn[slot]. */
int dne_vbn_ws_bytes(const dne_net_desc* net, int n_slots, int n_ref, size_t* out_bytes);
int dne_vbn_reference_pass(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                           const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                           const uint8_t* d_active, int n_slots,
                           const uint8_t* d_ref, int n_ref, float* d_vbn,
                           void* d_ws, size_t ws_bytes, void* stream);

/* Observation preprocess (atari_wrappers.py:105,167-180 mode 0; tf_atari.py:90 + stack_frames.py:33-43 mode 1):
 * max over two 84x84 uint8 frames, then frame-stack k=4 in place in d_stack [n_slots,84,84,4]. */
int dne_preprocess_atari(const uint8_t* d_prev, const uint8_t* d_cur, uint8_t* d_stack,
                         const uint8_t* d_reset_mask, int n_slots, int mode, void* stream);

/* The 210x160 -> 84x84 warp in front of the frame stack, both reference flavours (one 84x84 frame per raw frame pair):
 * dne_warp_atari_rgb      atari_wrappers.py:105,138-142: d_raw uint8 [n, 2, 210, 160, 3] (the last two RGB frames) ->
 *                         per-channel max -> gray float32 -> PIL BILINEAR (area-scaled triangle filter, two passes, double
 *                         accumulation) -> uint8 [n, 84, 84] (truncating cast).  Bit-exact with Pillow on the same gray.
 * dne_warp_atari_palette  tf_atari.py:88-92,149: d_raw uint8 [n, 2, 210, 160] NTSC palette indices, d_gray_lut float[256]
 *                         -> max of the two gray frames -> resize_bilinear(align_corners=True) -> float32 [n, 84, 84]
 *                         (d_out_f32, nullable) and / or its uint8 quantisation round(255*x) (d_out_u8, nullable) for
 *                         the uint8 frame-stack pipeline.
 * Feed the result to dne_preprocess_atari with d_prev = NULL (the max has already been taken on the raw frames). */
int dne_warp_atari_rgb(const uint8_t* d_raw, uint8_t* d_out, int n_frames, void* stream);
int dne_warp_atari_palette(const uint8_t* d_raw, const float* d_gray_lut, float* d_out_f32, uint8_t* d_out_u8,
                           int n_frames, void* stream);

/* ---- update side -------------------------------------------------------------------------------- */
/* compute_ranks / compute_centered_ranks (es.py:70-85) over the flattened returns; stable tie rule. */
int dne_centered_rank(const float* d_returns, int count, float* d_centered, int32_t* d_ranks, void* stream);

/* batched_weighted_sum + normalise (es.py:115-122,291-296):
 *   g[j] = (1/denom) * sum_i (d_proc[2i]-d_proc[2i+1]) * noise[d_noise_idx[i] + j],  j in [0,P)
 * d_proc: centred ranks (or any processed returns) [n,2]; denom = returns_n2.size of the WHOLE generation
 * (es.py:296); float64 accumulation, one float32 rounding.
 * accumulate != 0 adds into d_g instead of overwriting it. */
int dne_es_grad(dne_ctx* ctx, const float* d_proc_n2, const int64_t* d_noise_idx, int n, int64_t P,
                double denom, float* d_g, int accumulate, void* stream);

/* optimizer.update(-g + l2coeff*theta) (es.py:298; optimizers.py:10-17,35-50).  t is the 1-based step
 * count AFTER the increment at optimizers.py:11.  d_update_ratio: float32 scalar ||step||/||theta_old||. */
int dne_adam_step(dne_ctx* ctx, float* d_theta, float* d_m, float* d_v, const float* d_g, int64_t P,
                  double l2coeff, double stepsize, double beta1, double beta2, double epsilon, int t,
                  float* d_update_ratio, void* stream);
/* SGD with EMA momentum (optimizers.py:23-32). */
int dne_sgd_step(dne_ctx* ctx, float* d_theta, float* d_v, const float* d_g, int64_t P,
                 double l2coeff, double stepsize, double momentum, float* d_update_ratio, void* stream);

/* ---- GA / novelty -------------------------------------------------------------------------------- */
/* Seed chain -> weights.
 * mode 0 (gpu path, models/base.py:140-146,155-156; dqn.py:26-28): theta = noise[seed0]*scale_by; theta += power_k*noise[seed_k]
 * mode 1 (cpu path, ga.py:256-264; policies.py:42-44; tf_util.py:122-130): theta = column-normalise(noise[seed0]),
 *        biases 0; theta += power_k*noise[seed_k].
 * d_seeds int64[len], d_powers float[len] (powers[0] unused) on the device; h_std double[n_layers] on the HOST:
 * init std per layer (NULL = 1.0). */
int dne_ga_materialize(dne_ctx* ctx, const dne_net_desc* net, const int64_t* d_seeds, const float* d_powers,
                       int len, const double* h_std, int mode, float* d_theta_out, void* stream);
/* theta_out = theta_parent + power*noise[seed] (models/base.py:155-156) -- one mutation on a cached parent. */
int dne_ga_mutate(dne_ctx* ctx, const float* d_parent, int64_t seed, float power, int64_t P,
                  float* d_theta_out, void* stream);
/* Truncation selection (ga.py:145-149; gpu_implementation/ga.py:180): indices of the top-T fitness values,
 * descending, ties by arrival order. */
int dne_ga_truncate(const float* d_fitness, int pop, int T, int32_t* d_selected, void* stream);

/* k-NN novelty (nses.py:12-32): BC sequences are [*, t_max, D] uint8 padded with their LAST row, with
 * true lengths; distance over rows t < max(len_q, len_a); novelty = mean of the k smallest distances. */
int dne_knn_ws_bytes(int q, int A, size_t* out_bytes);
int dne_knn_novelty(const uint8_t* d_bc, const int32_t* d_bc_len, int q,
                    const uint8_t* d_archive, const int32_t* d_archive_len, int A,
                    int t_max, int D, int k, float* d_novelty, void* d_ws, size_t ws_bytes, void* stream);

/* Same for vector BCs (MujocoPolicy: final (x, y) position / trajectory, policies.py:292-299): float64 [*, D] of equal
 * length, plain L2 distance in float64 (nses.py:12-20 with equal lengths), mean of the k smallest.  Distances are ordered
 * like numpy's sort, NaN (from a NaN coordinate) after every number, so the novelty is NaN exactly when fewer than
 * min(k, A) of the query's distances are numbers. */
int dne_knn_novelty_vec(const double* d_bc, int q, const double* d_archive, int A, int D, int k, float* d_novelty,
                        void* d_ws, size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DNE_H_ */
