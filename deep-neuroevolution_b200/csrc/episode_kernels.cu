// episode_kernels.cu -- whole episodes of a device-resident environment in one launch.
//
// CartPole-v1 (gym classic_control, cartpole.py): the policy has a few hundred parameters and the environment step is a few
// dozen flops, so the per-tick runner (one forward launch + a device -> host -> device round trip per step) would spend
// nearly all its time on overhead.  Here one warp runs one member's episode from reset to termination: it builds the member's
// weights once in shared memory, then loops observation -> dense forward -> argmax -> environment step on the device.
//
// Numerics contract (DESIGN.md 3.5):
//   * weights w = fl(theta[row] + fl(scale * noise[idx + j])) -- the same rounding as every other forward of the engine;
//   * observation = (float)state, round to nearest (gym returns np.array(state, dtype=np.float32));
//   * dense layers in fp32: sequential fmaf over the inputs, then + bias, ReLU on hidden layers, no activation on the head;
//   * action = argmax of the 2 logits, first max on ties, NaN counts as the maximum (dense_small_kernel's rule);
//   * the environment step in float64, in gym's operation order, every operation an explicit round-to-nearest intrinsic so
//     nvcc cannot contract it into FMAs; sin / cos are CUDA's double sin / cos.
// No workspace, no atomics, no device RNG: reruns are bit-identical.
#include "common.cuh"
#include "forward.cuh"
#include <math_constants.h>

constexpr int EP_WARPS = 8;                 // members per CTA (one per warp)
constexpr int EP_MAX_LAYERS = 4;
constexpr int EP_MAX_WIDTH = 32;            // every layer width fits one warp: lane j owns output j
constexpr int CARTPOLE_OB_DIM = 4, CARTPOLE_ACTIONS = 2;

struct EpisodeNet {
    int n_layers;
    int cin[EP_MAX_LAYERS], cout[EP_MAX_LAYERS];
    int off_w[EP_MAX_LAYERS], off_b[EP_MAX_LAYERS];       // off_b < 0: no bias
    int P;
    int P_pad;                                            // per-warp shared-memory stride (floats)
};

// Which nets the fused episode kernel runs: dense layers only (<= 4, every width <= 32), vector observations of dimension
// 4, 2 outputs, ReLU hidden layers, no activation on the head, no batch norm.  On failure `why` names the reason.
bool dne_cartpole_net_supported(const dne_net_desc* net, const char** why) {
    if (net->n_layers < 1 || net->n_layers > EP_MAX_LAYERS) { *why = "needs 1..4 layers"; return false; }
    if (net->ob_kind != DNE_OB_VECTOR) { *why = "needs vector observations (DNE_OB_VECTOR)"; return false; }
    if (net->ob_dim != CARTPOLE_OB_DIM) { *why = "CartPole observations have ob_dim 4"; return false; }
    if (net->n_out != CARTPOLE_ACTIONS) { *why = "CartPole has 2 actions (n_out 2)"; return false; }
    if (net->vbn_len != 0) { *why = "batch norm is not supported"; return false; }
    int prev = net->ob_dim;
    for (int l = 0; l < net->n_layers; ++l) {
        const dne_layer_desc& L = net->layers[l];
        const bool head = (l == net->n_layers - 1);
        if (L.kind != DNE_DENSE) { *why = "dense layers only"; return false; }
        if (L.bn != DNE_BN_NONE) { *why = "batch norm is not supported"; return false; }
        if (L.cin != prev) { *why = "layer input size mismatch"; return false; }
        if (L.cin < 1 || L.cout < 1 || L.cin > EP_MAX_WIDTH || L.cout > EP_MAX_WIDTH) { *why = "layer width above 32"; return false; }
        if (head ? L.act != DNE_ACT_NONE : L.act != DNE_ACT_RELU) {
            *why = "hidden layers must be ReLU and the head linear";
            return false;
        }
        if (L.off_w < 0 || L.off_w + (int64_t)L.cin * L.cout > net->num_params ||
            (L.off_b >= 0 && L.off_b + L.cout > net->num_params)) {
            *why = "layer offsets outside num_params";
            return false;
        }
        prev = L.cout;
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

// 6 CTAs (48 member warps) per SM: 40 registers, no spills (the 120-byte stack frame is the local array of double
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

    // the member's weights, once per episode
    const float* th = theta + (theta_idx ? (int64_t)theta_idx[m] * net.P : 0);
    const float* nz = noise + noise_idx[m];
    const float s = scale[m];
    for (int j = lane; j < net.P; j += 32) w[j] = __fadd_rn(th[j], __fmul_rn(s, nz[j]));
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
    EpisodeNet en;
    en.n_layers = net->n_layers;
    for (int l = 0; l < EP_MAX_LAYERS; ++l) {
        const bool on = l < net->n_layers;
        en.cin[l] = on ? net->layers[l].cin : 0;
        en.cout[l] = on ? net->layers[l].cout : 0;
        en.off_w[l] = on ? (int)net->layers[l].off_w : 0;
        en.off_b[l] = on ? (int)net->layers[l].off_b : -1;
    }
    en.P = (int)net->num_params;
    en.P_pad = (en.P + 31) / 32 * 32;
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
