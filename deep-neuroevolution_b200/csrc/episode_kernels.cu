// episode_kernels.cu -- whole episodes of a device-resident environment in one launch.
//
// CartPole-v1 and Pendulum-v1 (gym classic_control): the policy has a few hundred to a few tens of thousands of
// parameters and the environment step is a few dozen flops, so the per-tick runner (one forward launch + a device -> host
// -> device round trip per step) would spend nearly all its time on overhead.  Here a group of threads runs one member's
// episode from reset to the end: it builds the member's weights once in shared memory, then loops observation -> dense
// forward -> action -> environment step on the device.
//
// Numerics contract (DESIGN.md 3.5, 3.6):
//   * weights w = fl(theta[row] + fl(scale * noise[idx + j])) -- the same rounding as every other forward of the engine;
//   * dense layers in fp32: each output a sequential fmaf over its inputs in index order, then + bias; the hidden layers'
//     activation is apply_act (common.cuh), the head is linear;
//   * the environment step in float64, in gym's operation order, every operation an explicit round-to-nearest intrinsic so
//     nvcc cannot contract it into FMAs; sin / cos are CUDA's double sin / cos.
// No workspace, no atomics, no device RNG: reruns are bit-identical.
#include "common.cuh"
#include "forward.cuh"
#include <math_constants.h>

constexpr int EP_WARPS = 8;                 // CartPole: members per CTA (one per warp)
constexpr int EP_MAX_WIDTH = 32;            // CartPole: every layer width fits one warp: lane j owns output j
constexpr int CARTPOLE_MAX_LAYERS = 4;
constexpr int CARTPOLE_OB_DIM = 4, CARTPOLE_ACTIONS = 2;
#define EP_STR2(x) #x
#define EP_STR(x) EP_STR2(x)

struct EpisodeNet {
    int n_layers;
    int cin[DNE_MAX_LAYERS], cout[DNE_MAX_LAYERS], act[DNE_MAX_LAYERS];
    int off_w[DNE_MAX_LAYERS], off_b[DNE_MAX_LAYERS];     // off_b < 0: no bias
    int P;
    int P_pad;                                            // per-member shared-memory stride of the weights (floats)
};

static EpisodeNet make_episode_net(const dne_net_desc* net) {
    EpisodeNet en;
    en.n_layers = net->n_layers;
    for (int l = 0; l < DNE_MAX_LAYERS; ++l) {
        const bool on = l < net->n_layers;
        en.cin[l] = on ? net->layers[l].cin : 0;
        en.cout[l] = on ? net->layers[l].cout : 0;
        en.act[l] = on ? net->layers[l].act : DNE_ACT_NONE;
        en.off_w[l] = on ? (int)net->layers[l].off_w : 0;
        en.off_b[l] = on ? (int)net->layers[l].off_b : -1;
    }
    en.P = (int)net->num_params;
    en.P_pad = (en.P + 31) / 32 * 32;
    return en;
}

// The member's weights, once per episode, by `nthr` threads starting at thread `t`.
__device__ __forceinline__ void build_member_weights(float* w, const EpisodeNet& net, const float* __restrict__ theta,
                                                     const float* __restrict__ noise, const int64_t* __restrict__ noise_idx,
                                                     const float* __restrict__ scale, const int32_t* __restrict__ theta_idx,
                                                     int m, int t, int nthr) {
    const float* th = theta + (theta_idx ? (int64_t)theta_idx[m] * net.P : 0);
    const float* nz = noise + noise_idx[m];
    const float s = scale[m];
    for (int j = t; j < net.P; j += nthr) w[j] = __fadd_rn(th[j], __fmul_rn(s, nz[j]));
}

// The checks both episode kernels share: dense layers only, chained widths, no batch norm, vector observations of
// dimension `ob_dim`, `n_out` outputs, a linear head, every parameter offset inside num_params.  The caller checks the
// widths and the hidden activations.
static bool episode_net_common(const dne_net_desc* net, int max_layers, int ob_dim, int n_out, const char* ob_why,
                               const char* out_why, const char** why) {
    if (net->n_layers < 1 || net->n_layers > max_layers) {
        *why = max_layers == CARTPOLE_MAX_LAYERS ? "needs 1..4 layers" : "needs 1.." EP_STR(DNE_MAX_LAYERS) " layers";
        return false;
    }
    if (net->ob_kind != DNE_OB_VECTOR) { *why = "needs vector observations (DNE_OB_VECTOR)"; return false; }
    if (net->ob_dim != ob_dim) { *why = ob_why; return false; }
    if (net->n_out != n_out) { *why = out_why; return false; }
    if (net->vbn_len != 0) { *why = "batch norm is not supported"; return false; }
    int prev = net->ob_dim;
    for (int l = 0; l < net->n_layers; ++l) {
        const dne_layer_desc& L = net->layers[l];
        if (L.kind != DNE_DENSE) { *why = "dense layers only"; return false; }
        if (L.bn != DNE_BN_NONE) { *why = "batch norm is not supported"; return false; }
        if (L.cin != prev) { *why = "layer input size mismatch"; return false; }
        if (L.cin < 1 || L.cout < 1) { *why = "empty layer"; return false; }
        if (L.off_w < 0 || L.off_w + (int64_t)L.cin * L.cout > net->num_params ||
            (L.off_b >= 0 && L.off_b + L.cout > net->num_params)) {
            *why = "layer offsets outside num_params";
            return false;
        }
        prev = L.cout;
    }
    return true;
}

// Which nets the fused CartPole kernel runs: dense layers only (<= 4, every width <= 32), vector observations of dimension
// 4, 2 outputs, ReLU hidden layers, no activation on the head, no batch norm.  On failure `why` names the reason.
bool dne_cartpole_net_supported(const dne_net_desc* net, const char** why) {
    if (!episode_net_common(net, CARTPOLE_MAX_LAYERS, CARTPOLE_OB_DIM, CARTPOLE_ACTIONS,
                            "CartPole observations have ob_dim 4", "CartPole has 2 actions (n_out 2)", why))
        return false;
    for (int l = 0; l < net->n_layers; ++l) {
        const dne_layer_desc& L = net->layers[l];
        const bool head = (l == net->n_layers - 1);
        if (L.cin > EP_MAX_WIDTH || L.cout > EP_MAX_WIDTH) { *why = "layer width above 32"; return false; }
        if (head ? L.act != DNE_ACT_NONE : L.act != DNE_ACT_RELU) {
            *why = "hidden layers must be ReLU and the head linear";
            return false;
        }
    }
    // the largest net the rules above allow (4 layers of width 32) has 3328 parameters
    if (net->num_params > 4096) { *why = "num_params too large for the shared-memory weights"; return false; }
    return true;
}

// one CartPole-v1 step (gym cartpole.py), left-to-right products, explicit rounding
struct CartPole {
    double x, x_dot, th, th_dot;
};
__device__ __forceinline__ bool cartpole_step(CartPole& s, int action, double total_mass, double polemass_length,
                                              double theta_threshold) {
    const double gravity = 9.8, masspole = 0.1, length = 0.5, force_mag = 10.0, tau = 0.02, x_threshold = 2.4;
    const double force = action == 1 ? force_mag : -force_mag;
    const double c = cos(s.th), sn = sin(s.th);
    // temp = (force + polemass_length * theta_dot**2 * sintheta) / total_mass
    const double temp = __ddiv_rn(__dadd_rn(force, __dmul_rn(__dmul_rn(polemass_length, __dmul_rn(s.th_dot, s.th_dot)), sn)),
                                  total_mass);
    // thetaacc = (gravity * sintheta - costheta * temp) / (length * (4.0 / 3.0 - masspole * costheta**2 / total_mass))
    const double den = __dmul_rn(length, __dsub_rn(__ddiv_rn(4.0, 3.0),
                                                   __ddiv_rn(__dmul_rn(masspole, __dmul_rn(c, c)), total_mass)));
    const double thetaacc = __ddiv_rn(__dsub_rn(__dmul_rn(gravity, sn), __dmul_rn(c, temp)), den);
    // xacc = temp - polemass_length * thetaacc * costheta / total_mass
    const double xacc = __dsub_rn(temp, __ddiv_rn(__dmul_rn(__dmul_rn(polemass_length, thetaacc), c), total_mass));
    s.x = __dadd_rn(s.x, __dmul_rn(tau, s.x_dot));                 // Euler, gym's order
    s.x_dot = __dadd_rn(s.x_dot, __dmul_rn(tau, xacc));
    s.th = __dadd_rn(s.th, __dmul_rn(tau, s.th_dot));
    s.th_dot = __dadd_rn(s.th_dot, __dmul_rn(tau, thetaacc));
    return s.x < -x_threshold || s.x > x_threshold || s.th < -theta_threshold || s.th > theta_threshold;
}

// 6 CTAs (48 member warps) per SM: 40 registers, no spills (the 40-byte stack frame is the local array of double
// sin / cos's slow-path argument reduction).  The loop is latency bound, so resident warps are what hides it; 8 CTAs per SM
// (32 registers) spills.
__global__ void __launch_bounds__(EP_WARPS * 32, 6)
cartpole_episode_kernel(EpisodeNet net, const float* __restrict__ theta, const float* __restrict__ noise,
                        const int64_t* __restrict__ noise_idx, const float* __restrict__ scale,
                        const int32_t* __restrict__ theta_idx, int n_members, const double* __restrict__ init_state,
                        int max_steps, float* __restrict__ returns, int32_t* __restrict__ lengths,
                        double* __restrict__ final_state) {
    extern __shared__ float ep_smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m = blockIdx.x * EP_WARPS + warp;
    if (m >= n_members) return;                                   // whole warps leave together
    float* w = ep_smem + (int64_t)warp * net.P_pad;

    build_member_weights(w, net, theta, noise, noise_idx, scale, theta_idx, m, lane, 32);
    __syncwarp();

    // gym derives these from its parameters: total_mass = masspole + masscart, polemass_length = masspole * length,
    // theta_threshold_radians = 12 * 2 * math.pi / 360
    const double total_mass = __dadd_rn(0.1, 1.0);
    const double polemass_length = __dmul_rn(0.1, 0.5);
    const double theta_threshold = __ddiv_rn(__dmul_rn(24.0, CUDART_PI), 360.0);

    CartPole st;
    st.x = init_state[4 * m + 0];
    st.x_dot = init_state[4 * m + 1];
    st.th = init_state[4 * m + 2];
    st.th_dot = init_state[4 * m + 3];
    int len = 0;
    bool done = false;
    while (!done && len < max_steps) {
        // lane k < 4 holds observation component k (every lane keeps the full state: the step is warp-uniform)
        const double sk = lane == 0 ? st.x : lane == 1 ? st.x_dot : lane == 2 ? st.th : st.th_dot;
        float x = lane < CARTPOLE_OB_DIM ? __double2float_rn(sk) : 0.0f;
        for (int l = 0; l < net.n_layers; ++l) {
            const int K = net.cin[l], N = net.cout[l];
            const float* wl = w + net.off_w[l];
            const int n = lane < N ? lane : 0;
            float acc = 0.0f;
            for (int k = 0; k < K; ++k) acc = fmaf(__shfl_sync(0xffffffffu, x, k), wl[k * N + n], acc);
            float y = net.off_b[l] >= 0 ? acc + w[net.off_b[l] + n] : acc;
            if (l + 1 < net.n_layers) y = fmaxf(y, 0.0f);                 // ReLU (hidden layers)
            x = lane < N ? y : 0.0f;
        }
        const float y0 = __shfl_sync(0xffffffffu, x, 0), y1 = __shfl_sync(0xffffffffu, x, 1);
        const int action = (y0 != y0) ? 0 : ((y1 > y0 || y1 != y1) ? 1 : 0);   // first max, NaN is the max
        done = cartpole_step(st, action, total_mass, polemass_length, theta_threshold);
        ++len;
    }
    if (lane == 0) {
        returns[m] = (float)len;                                  // reward 1.0 on every step, the terminating one included
        lengths[m] = len;
        if (final_state) {
            final_state[4 * m + 0] = st.x;
            final_state[4 * m + 1] = st.x_dot;
            final_state[4 * m + 2] = st.th;
            final_state[4 * m + 3] = st.th_dot;
        }
    }
}

int dne_launch_cartpole_episodes(const dne_net_desc* net, const float* theta, const float* noise, const int64_t* noise_idx,
                                 const float* scale, const int32_t* theta_idx, int n_members, const double* init_state,
                                 int max_steps, float* returns, int32_t* lengths, double* final_state, cudaStream_t st) {
    const EpisodeNet en = make_episode_net(net);
    const size_t smem = (size_t)EP_WARPS * en.P_pad * sizeof(float);
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(cartpole_episode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return DNE_ERR_CUDA;
    }
    const unsigned grid = (unsigned)((n_members + EP_WARPS - 1) / EP_WARPS);
    cartpole_episode_kernel<<<grid, EP_WARPS * 32, smem, st>>>(en, theta, noise, noise_idx, scale, theta_idx, n_members,
                                                               init_state, max_steps, returns, lengths, final_state);
    DNE_LAUNCHED(1);
    return DNE_OK;
}

// ---- Pendulum-v1 ------------------------------------------------------------------------------------------------------
// gymnasium classic_control pendulum.py: g = 10, m = l = 1, dt = 0.05, max_speed = 8, max_torque = 2, TimeLimit 200, no
// termination.  One member per group of min(max layer width, 256) threads, rounded up to a warp (thread t owns outputs
// t, t + threads, ... of every layer); as many groups per CTA as maximise the members resident per SM, each group
// synchronised by its own named barrier.  Thread 0 of a group keeps the float64 state, writes the normalised observation,
// computes the head (n_out 1) and steps the pendulum.
constexpr int PEND_OB_DIM = 3, PEND_ACTIONS = 1, PEND_MAX_STEPS = 200;
constexpr int PEND_CTA_THREADS = 256;
constexpr int PEND_MAX_GROUPS = 15;                   // named barriers 1..15 (0 is __syncthreads')
constexpr size_t PEND_SMEM_LIMIT = 227 * 1024;        // H100 opt-in shared memory per CTA

struct PendulumGeom {
    int threads;                                      // threads per member: min(max layer width, 256), a multiple of 32
    int act_pad;                                      // floats of one activation buffer: max layer width rounded up to 32
    size_t member_bytes;                              // weights + two activation buffers
};

static PendulumGeom pendulum_geom(const dne_net_desc* net) {
    int width = PEND_OB_DIM;
    for (int l = 0; l < net->n_layers; ++l) width = width > net->layers[l].cout ? width : net->layers[l].cout;
    PendulumGeom g;
    g.act_pad = (width + 31) / 32 * 32;
    g.threads = g.act_pad < PEND_CTA_THREADS ? g.act_pad : PEND_CTA_THREADS;
    g.member_bytes = ((size_t)(net->num_params + 31) / 32 * 32 + 2 * (size_t)g.act_pad) * sizeof(float);
    return g;
}

// Which nets the fused Pendulum kernel runs: 1..DNE_MAX_LAYERS dense layers, vector observations of dimension 3, 1
// output, tanh or ReLU hidden layers, a linear head, no batch norm, and one member's weights plus its two activation
// buffers within one CTA's shared memory (hidden [200, 200] fits, [256, 256] does not).  Any layer width runs: a group
// has at most 256 threads, each looping over its outputs.
bool dne_pendulum_net_supported(const dne_net_desc* net, const char** why) {
    if (!episode_net_common(net, DNE_MAX_LAYERS, PEND_OB_DIM, PEND_ACTIONS, "Pendulum observations have ob_dim 3",
                            "Pendulum has one continuous action (n_out 1)", why))
        return false;
    for (int l = 0; l < net->n_layers; ++l) {
        const int act = net->layers[l].act;
        if (l == net->n_layers - 1 ? act != DNE_ACT_NONE : (act != DNE_ACT_TANH && act != DNE_ACT_RELU)) {
            *why = "hidden layers must be tanh or ReLU and the head linear";
            return false;
        }
    }
    if (net->num_params > (1 << 24) || pendulum_geom(net).member_bytes > PEND_SMEM_LIMIT) {
        *why = "one member's weights and activations exceed a CTA's shared memory (227 KB)";
        return false;
    }
    return true;
}

__device__ __forceinline__ void group_sync(int id, int nthr) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthr) : "memory");
}

// numpy's float64 divmod remainder (npy_divmod): fmod, then moved to the divisor's sign
__device__ __forceinline__ double py_mod(double a, double b) {
    double r = fmod(a, b);
    if (r != 0.0) {
        if ((r < 0.0) != (b < 0.0)) r = __dadd_rn(r, b);
    } else {
        r = copysign(0.0, b);
    }
    return r;
}

// One Pendulum-v1 step with the float32 action a (already noised): updates (th, thdot), returns the float64 reward.
__device__ __forceinline__ double pendulum_step(double& th, double& thdot, float a) {
    const float u = a < -2.0f ? -2.0f : (a > 2.0f ? 2.0f : a);            // np.clip on the float32 action (NaN stays)
    const double two_pi = __dmul_rn(2.0, CUDART_PI);
    const double an = __dsub_rn(py_mod(__dadd_rn(th, CUDART_PI), two_pi), CUDART_PI);     // angle_normalize(th)
    // costs = angle_normalize(th)**2 + 0.1 * thdot**2 + 0.001 * (u**2)   (u**2 is a float32 product)
    const double costs = __dadd_rn(__dadd_rn(__dmul_rn(an, an), __dmul_rn(0.1, __dmul_rn(thdot, thdot))),
                                   __dmul_rn(0.001, (double)__fmul_rn(u, u)));
    // newthdot = thdot + (3 * g / (2 * l) * sin(th) + 3.0 / (m * l**2) * u) * dt, clipped to +-max_speed
    double nthdot = __dadd_rn(thdot, __dmul_rn(__dadd_rn(__dmul_rn(15.0, sin(th)), __dmul_rn(3.0, (double)u)), 0.05));
    nthdot = nthdot < -8.0 ? -8.0 : (nthdot > 8.0 ? 8.0 : nthdot);
    th = __dadd_rn(th, __dmul_rn(nthdot, 0.05));
    thdot = nthdot;
    return -costs;
}

// No spills (40-byte stack frame: double sin / cos's slow-path argument reduction; registers in DESIGN.md 3.6).  Shared
// memory bounds the residency: hidden [64, 64] keeps 12 members (24 warps) per SM, [128, 128] 3, [200, 200] 1.
__global__ void __launch_bounds__(PEND_CTA_THREADS)
pendulum_episode_kernel(EpisodeNet net, int threads, int act_pad, int groups, const float* __restrict__ theta,
                        const float* __restrict__ noise, const int64_t* __restrict__ noise_idx,
                        const float* __restrict__ scale, const int32_t* __restrict__ theta_idx, int n_members,
                        const double* __restrict__ init_state, int max_steps, const float* __restrict__ ob_mean,
                        const float* __restrict__ ob_std, const float* __restrict__ ac_noise, float* __restrict__ returns,
                        float* __restrict__ signreturns, int32_t* __restrict__ lengths, double* __restrict__ final_state,
                        double* __restrict__ ob_sum, double* __restrict__ ob_sumsq) {
    extern __shared__ float ep_smem[];
    const int grp = threadIdx.x / threads, t = threadIdx.x - grp * threads;
    if (grp >= groups) return;
    const int m = blockIdx.x * groups + grp;
    if (m >= n_members) return;                                   // whole groups leave together
    const int bar = 1 + grp;
    float* w = ep_smem + (int64_t)grp * (net.P_pad + 2 * act_pad);
    float* buf0 = w + net.P_pad;
    float* buf1 = buf0 + act_pad;

    build_member_weights(w, net, theta, noise, noise_idx, scale, theta_idx, m, t, threads);

    double th = 0.0, thdot = 0.0, ret = 0.0, sret = 0.0;
    double os0 = 0.0, os1 = 0.0, os2 = 0.0, oq0 = 0.0, oq1 = 0.0, oq2 = 0.0;
    if (t == 0) {
        th = init_state[2 * m + 0];
        thdot = init_state[2 * m + 1];
    }
    const int L = net.n_layers;
    for (int step = 0; step < max_steps; ++step) {
        if (t == 0) {                         // observation float32([cos th, sin th, thdot]), normalised as ob_norm_kernel
            const float o0 = __double2float_rn(cos(th)), o1 = __double2float_rn(sin(th)), o2 = __double2float_rn(thdot);
            if (ob_sum) {                     // ob_stat_accum_kernel's sums of the unnormalised observation
                os0 = __dadd_rn(os0, (double)o0);
                os1 = __dadd_rn(os1, (double)o1);
                os2 = __dadd_rn(os2, (double)o2);
                oq0 = __dadd_rn(oq0, __dmul_rn((double)o0, (double)o0));
                oq1 = __dadd_rn(oq1, __dmul_rn((double)o1, (double)o1));
                oq2 = __dadd_rn(oq2, __dmul_rn((double)o2, (double)o2));
            }
            float x0 = o0, x1 = o1, x2 = o2;
            if (ob_mean) {
                x0 = fminf(fmaxf(__fdiv_rn(__fsub_rn(x0, ob_mean[0]), ob_std[0]), -5.0f), 5.0f);
                x1 = fminf(fmaxf(__fdiv_rn(__fsub_rn(x1, ob_mean[1]), ob_std[1]), -5.0f), 5.0f);
                x2 = fminf(fmaxf(__fdiv_rn(__fsub_rn(x2, ob_mean[2]), ob_std[2]), -5.0f), 5.0f);
            }
            buf0[0] = x0;
            buf0[1] = x1;
            buf0[2] = x2;
        }
        group_sync(bar, threads);
        // hidden layers: all threads, ping-pong buffers, one barrier per layer (a layer's reads of its output buffer, by
        // the layer before, finished before that barrier)
        const float* x = buf0;
        float* y = buf1;
        for (int l = 0; l + 1 < L; ++l) {
            const int K = net.cin[l], N = net.cout[l];
            for (int j = t; j < N; j += threads) {
                const float* wl = w + net.off_w[l] + j;
                float acc = 0.0f;
#pragma unroll 4
                for (int k = 0; k < K; ++k) acc = fmaf(x[k], wl[k * N], acc);
                if (net.off_b[l] >= 0) acc = __fadd_rn(acc, w[net.off_b[l] + j]);
                y[j] = apply_act(acc, net.act[l]);
            }
            group_sync(bar, threads);
            const float* nx = y;
            y = (float*)x;
            x = nx;
        }
        if (t == 0) {                         // the linear head (n_out 1), the action noise, the environment step
            const int K = net.cin[L - 1];
            const float* wl = w + net.off_w[L - 1];
            float acc = 0.0f;
#pragma unroll 4
            for (int k = 0; k < K; ++k) acc = fmaf(x[k], wl[k], acc);
            if (net.off_b[L - 1] >= 0) acc = __fadd_rn(acc, w[net.off_b[L - 1]]);
            const float a = ac_noise ? __fadd_rn(acc, ac_noise[(int64_t)m * max_steps + step]) : acc;
            const float r = __double2float_rn(pendulum_step(th, thdot, a));       // BatchEnv.step returns float32
            ret = __dadd_rn(ret, (double)r);
            sret = __dadd_rn(sret, r > 0.0f ? 1.0 : r < 0.0f ? -1.0 : (double)r);    // np.sign (0 -> 0, NaN -> NaN)
        }
    }
    if (t == 0) {
        returns[m] = __double2float_rn(ret);
        signreturns[m] = __double2float_rn(sret);
        lengths[m] = max_steps;
        if (final_state) {
            final_state[2 * m + 0] = th;
            final_state[2 * m + 1] = thdot;
        }
        if (ob_sum) {
            ob_sum[3 * m + 0] = os0;
            ob_sum[3 * m + 1] = os1;
            ob_sum[3 * m + 2] = os2;
            ob_sumsq[3 * m + 0] = oq0;
            ob_sumsq[3 * m + 1] = oq1;
            ob_sumsq[3 * m + 2] = oq2;
        }
    }
}

int dne_launch_pendulum_episodes(const dne_net_desc* net, const float* theta, const float* noise, const int64_t* noise_idx,
                                 const float* scale, const int32_t* theta_idx, int n_members, const double* init_state,
                                 int max_steps, const float* ob_mean, const float* ob_std, const float* ac_noise,
                                 float* returns, float* signreturns, int32_t* lengths, double* final_state, double* ob_sum,
                                 double* ob_sumsq, cudaStream_t st) {
    const EpisodeNet en = make_episode_net(net);
    const PendulumGeom g = pendulum_geom(net);
    if (cudaFuncSetAttribute(pendulum_episode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PEND_SMEM_LIMIT) !=
        cudaSuccess)
        return DNE_ERR_CUDA;
    // members per CTA: the count that keeps the most members resident per SM (registers, shared memory, threads, as the
    // occupancy calculator counts them); on a tie the more (hidden [64, 64], 5000 members on an H100: 4 per CTA 2.74 and
    // 2.84 ms in two runs, 2 per CTA 3.05 ms, both with 12 members resident per SM)
    int groups = 1, best = 0;
    const int max_groups = PEND_CTA_THREADS / g.threads < PEND_MAX_GROUPS ? PEND_CTA_THREADS / g.threads : PEND_MAX_GROUPS;
    for (int gr = 1; gr <= max_groups && (size_t)gr * g.member_bytes <= PEND_SMEM_LIMIT; ++gr) {
        int blocks = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, pendulum_episode_kernel, gr * g.threads,
                                                          (size_t)gr * g.member_bytes) != cudaSuccess)
            return DNE_ERR_CUDA;
        if (blocks * gr >= best) {
            best = blocks * gr;
            groups = gr;
        }
    }
    const size_t smem = (size_t)groups * g.member_bytes;
    const unsigned grid = (unsigned)((n_members + groups - 1) / groups);
    pendulum_episode_kernel<<<grid, groups * g.threads, smem, st>>>(
        en, g.threads, g.act_pad, groups, theta, noise, noise_idx, scale, theta_idx, n_members, init_state, max_steps,
        ob_mean, ob_std, ac_noise, returns, signreturns, lengths, final_state, ob_sum, ob_sumsq);
    DNE_LAUNCHED(1);
    return DNE_OK;
}
