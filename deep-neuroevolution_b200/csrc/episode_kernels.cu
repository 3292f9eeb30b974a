// episode_kernels.cu -- whole episodes of a device-resident environment in one launch.
//
// CartPole-v1, Acrobot-v1, MountainCar-v0 and Pendulum-v1 (gym classic_control): the policy has a few hundred to a few
// tens of thousands of parameters and the environment step is a few dozen to a few hundred flops, so the per-tick runner
// (one forward launch + a device -> host -> device round trip per step) would spend nearly all its time on overhead.  Here a
// group of threads runs one member's episode from reset to the end: it builds the member's weights once in shared memory,
// then loops observation -> dense forward -> action -> environment step on the device.
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

constexpr int EP_WARPS = 8;                 // discrete tasks: members per CTA (one per warp)
constexpr int EP_MAX_WIDTH = 32;            // discrete tasks: every layer width fits one warp: lane j owns output j
constexpr int DISCRETE_MAX_LAYERS = 4;
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
        *why = max_layers == DISCRETE_MAX_LAYERS ? "needs 1..4 layers" : "needs 1.." EP_STR(DNE_MAX_LAYERS) " layers";
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

// ---- discrete-action tasks: CartPole-v1, Acrobot-v1, MountainCar-v0 ---------------------------------------------------
// One warp per member; every lane keeps the whole float64 state and steps it (the step is warp-uniform).  A task type
// supplies STATE_DIM, OB_DIM (<= 32), ACTIONS (<= 32), TIME_LIMIT and MIN_CTAS (the kernel's minimum CTAs per SM: as many
// as its step fits in without spilling), a constructor loading the float64 state, store(), ob(k) (observation component k
// as float32) and step(action, reward) (returns done).  Every reward of these tasks is -1.0, 0.0 or +1.0, so their float64
// sum in step order is an exact integer: step() reports the reward as that integer and the kernel sums integers.

// one CartPole-v1 step (gym cartpole.py), left-to-right products, explicit rounding
struct CartPoleTask {
    static constexpr int STATE_DIM = 4, OB_DIM = 4, ACTIONS = 2, TIME_LIMIT = 500;
    // 6 CTAs (48 member warps) per SM: 40 registers, no spills (the 40-byte stack frame is the local array of double
    // sin / cos's slow-path argument reduction).  The loop is latency bound, so resident warps are what hides it; 8 CTAs
    // per SM (32 registers) spills.
    static constexpr int MIN_CTAS = 6;
    static constexpr const char* OB_WHY = "CartPole observations have ob_dim 4";
    static constexpr const char* OUT_WHY = "CartPole has 2 actions (n_out 2)";
    double x, x_dot, th, th_dot;
    // gym derives these from its parameters: total_mass = masspole + masscart, polemass_length = masspole * length,
    // theta_threshold_radians = 12 * 2 * math.pi / 360
    double total_mass, polemass_length, theta_threshold;

    __device__ __forceinline__ explicit CartPoleTask(const double* s) : x(s[0]), x_dot(s[1]), th(s[2]), th_dot(s[3]) {
        total_mass = __dadd_rn(0.1, 1.0);
        polemass_length = __dmul_rn(0.1, 0.5);
        theta_threshold = __ddiv_rn(__dmul_rn(24.0, CUDART_PI), 360.0);
    }
    __device__ __forceinline__ void store(double* s) const {
        s[0] = x;
        s[1] = x_dot;
        s[2] = th;
        s[3] = th_dot;
    }
    __device__ __forceinline__ float ob(int k) const {       // float32(state)
        return __double2float_rn(k == 0 ? x : k == 1 ? x_dot : k == 2 ? th : th_dot);
    }
    __device__ __forceinline__ bool step(int action, int& reward) {
        const double gravity = 9.8, masspole = 0.1, length = 0.5, force_mag = 10.0, tau = 0.02, x_threshold = 2.4;
        const double force = action == 1 ? force_mag : -force_mag;
        const double c = cos(th), sn = sin(th);
        // temp = (force + polemass_length * theta_dot**2 * sintheta) / total_mass
        const double temp = __ddiv_rn(__dadd_rn(force, __dmul_rn(__dmul_rn(polemass_length, __dmul_rn(th_dot, th_dot)), sn)),
                                      total_mass);
        // thetaacc = (gravity * sintheta - costheta * temp) / (length * (4.0 / 3.0 - masspole * costheta**2 / total_mass))
        const double den = __dmul_rn(length, __dsub_rn(__ddiv_rn(4.0, 3.0),
                                                       __ddiv_rn(__dmul_rn(masspole, __dmul_rn(c, c)), total_mass)));
        const double thetaacc = __ddiv_rn(__dsub_rn(__dmul_rn(gravity, sn), __dmul_rn(c, temp)), den);
        // xacc = temp - polemass_length * thetaacc * costheta / total_mass
        const double xacc = __dsub_rn(temp, __ddiv_rn(__dmul_rn(__dmul_rn(polemass_length, thetaacc), c), total_mass));
        x = __dadd_rn(x, __dmul_rn(tau, x_dot));                     // Euler, gym's order
        x_dot = __dadd_rn(x_dot, __dmul_rn(tau, xacc));
        th = __dadd_rn(th, __dmul_rn(tau, th_dot));
        th_dot = __dadd_rn(th_dot, __dmul_rn(tau, thetaacc));
        reward = 1;                                                   // the terminating step included
        return x < -x_threshold || x > x_threshold || th < -theta_threshold || th > theta_threshold;
    }
};

// Acrobot-v1 (gymnasium acrobot.py, "book" dynamics, no torque noise): state (theta1, theta2, dtheta1, dtheta2), one RK4
// step of dt = 0.2 per action, torque [-1, 0, +1][action].  DESIGN.md 3.5 writes out the operation order.
constexpr double ACRO_M1 = 1.0, ACRO_M2 = 1.0, ACRO_L1 = 1.0, ACRO_LC1 = 0.5, ACRO_LC2 = 0.5, ACRO_I1 = 1.0,
                 ACRO_I2 = 1.0, ACRO_G = 9.8, ACRO_DT = 0.2;
// gym's wrap() loops for ever on an angle it cannot bring into [-pi, pi]; the kernel gives up after this many turns (a
// state the dynamics reach from any reset moves far less than one turn per step)
constexpr int ACRO_WRAP_MAX_TURNS = 4096;

// _dsdt: the time derivative (ddtheta1, ddtheta2) of the velocities under torque `a` (the angles' derivatives are the
// velocities themselves, the torque's is 0)
__device__ __forceinline__ void acrobot_accel(double th1, double th2, double dth1, double dth2, double a, double& ddth1,
                                              double& ddth2) {
    const double m1 = ACRO_M1, m2 = ACRO_M2, l1 = ACRO_L1, lc1 = ACRO_LC1, lc2 = ACRO_LC2, I1 = ACRO_I1, I2 = ACRO_I2,
                 g = ACRO_G, pi = CUDART_PI;
    const double ct2 = cos(th2), st2 = sin(th2);
    // d1 = m1 * lc1**2 + m2 * (l1**2 + lc2**2 + 2 * l1 * lc2 * cos(theta2)) + I1 + I2
    const double d1 = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(m1, __dmul_rn(lc1, lc1)),
                                                    __dmul_rn(m2, __dadd_rn(__dadd_rn(__dmul_rn(l1, l1), __dmul_rn(lc2, lc2)),
                                                                            __dmul_rn(__dmul_rn(__dmul_rn(2.0, l1), lc2), ct2)))),
                                          I1),
                                I2);
    // d2 = m2 * (lc2**2 + l1 * lc2 * cos(theta2)) + I2
    const double d2 = __dadd_rn(__dmul_rn(m2, __dadd_rn(__dmul_rn(lc2, lc2), __dmul_rn(__dmul_rn(l1, lc2), ct2))), I2);
    // phi2 = m2 * lc2 * g * cos(theta1 + theta2 - pi / 2.0)
    const double phi2 = __dmul_rn(__dmul_rn(__dmul_rn(m2, lc2), g), cos(__dsub_rn(__dadd_rn(th1, th2), __ddiv_rn(pi, 2.0))));
    // phi1 = -m2 * l1 * lc2 * dtheta2**2 * sin(theta2) - 2 * m2 * l1 * lc2 * dtheta2 * dtheta1 * sin(theta2)
    //        + (m1 * lc1 + m2 * l1) * g * cos(theta1 - pi / 2) + phi2
    const double p1 = __dmul_rn(__dmul_rn(__dmul_rn(__dmul_rn(-m2, l1), lc2), __dmul_rn(dth2, dth2)), st2);
    const double p2 = __dmul_rn(__dmul_rn(__dmul_rn(__dmul_rn(__dmul_rn(__dmul_rn(2.0, m2), l1), lc2), dth2), dth1), st2);
    const double p3 = __dmul_rn(__dmul_rn(__dadd_rn(__dmul_rn(m1, lc1), __dmul_rn(m2, l1)), g),
                                cos(__dsub_rn(th1, __ddiv_rn(pi, 2.0))));
    const double phi1 = __dadd_rn(__dadd_rn(__dsub_rn(p1, p2), p3), phi2);
    // ddtheta2 = (a + d2 / d1 * phi1 - m2 * l1 * lc2 * dtheta1**2 * sin(theta2) - phi2) / (m2 * lc2**2 + I2 - d2**2 / d1)
    const double num = __dsub_rn(__dsub_rn(__dadd_rn(a, __dmul_rn(__ddiv_rn(d2, d1), phi1)),
                                           __dmul_rn(__dmul_rn(__dmul_rn(__dmul_rn(m2, l1), lc2), __dmul_rn(dth1, dth1)), st2)),
                                 phi2);
    const double den = __dsub_rn(__dadd_rn(__dmul_rn(m2, __dmul_rn(lc2, lc2)), I2), __ddiv_rn(__dmul_rn(d2, d2), d1));
    ddth2 = __ddiv_rn(num, den);
    // ddtheta1 = -(d2 * ddtheta2 + phi1) / d1
    ddth1 = __ddiv_rn(-__dadd_rn(__dmul_rn(d2, ddth2), phi1), d1);
}

struct AcrobotTask {
    static constexpr int STATE_DIM = 4, OB_DIM = 6, ACTIONS = 3, TIME_LIMIT = 500;
    static constexpr int MIN_CTAS = 4;            // 64 registers, no spills; 5 CTAs per SM (48 registers) spills
    static constexpr const char* OB_WHY = "Acrobot observations have ob_dim 6";
    static constexpr const char* OUT_WHY = "Acrobot has 3 actions (n_out 3)";
    double th1, th2, dth1, dth2;

    __device__ __forceinline__ explicit AcrobotTask(const double* s) : th1(s[0]), th2(s[1]), dth1(s[2]), dth2(s[3]) {}
    __device__ __forceinline__ void store(double* s) const {
        s[0] = th1;
        s[1] = th2;
        s[2] = dth1;
        s[3] = dth2;
    }
    __device__ __forceinline__ float ob(int k) const {       // float32([cos th1, sin th1, cos th2, sin th2, dth1, dth2])
        const double a = k < 2 ? th1 : th2;
        return __double2float_rn(k == 4 ? dth1 : k == 5 ? dth2 : (k & 1) ? sin(a) : cos(a));
    }
    static __device__ __forceinline__ double wrap(double x) {                // gym's wrap(x, -pi, pi)
        const double m = -CUDART_PI, M = CUDART_PI, diff = __dsub_rn(M, m);
        for (int i = 0; i < ACRO_WRAP_MAX_TURNS && x > M; ++i) x = __dsub_rn(x, diff);
        for (int i = 0; i < ACRO_WRAP_MAX_TURNS && x < m; ++i) x = __dadd_rn(x, diff);
        return x;
    }
    static __device__ __forceinline__ double bound(double x, double B) {      // gym's bound(x, -B, B) = min(max(x, -B), B)
        x = -B > x ? -B : x;
        return B < x ? B : x;
    }
    __device__ __forceinline__ bool step(int action, int& reward) {
        const double a = (double)(action - 1);                        // AVAIL_TORQUE = [-1.0, 0.0, +1]
        const double dt = ACRO_DT, dt2 = __ddiv_rn(dt, 2.0);
        // rk4: k1 = f(y0), k2 = f(y0 + dt2 * k1), k3 = f(y0 + dt2 * k2), k4 = f(y0 + dt * k3);
        // y0 + dt / 6.0 * (k1 + 2 * k2 + 2 * k3 + k4), the sum accumulated left to right as it is built
        double k0, k1, k2, k3;                                        // one stage's derivative
        double s0, s1, s2, s3;                                        // k1 + 2 * k2 + ..., so far
        acrobot_accel(th1, th2, dth1, dth2, a, k2, k3);
        k0 = dth1;
        k1 = dth2;
        s0 = k0, s1 = k1, s2 = k2, s3 = k3;
#pragma unroll 1
        for (int stage = 1; stage < 4; ++stage) {
            const double h = stage < 3 ? dt2 : dt;
            const double y0 = __dadd_rn(th1, __dmul_rn(h, k0)), y1 = __dadd_rn(th2, __dmul_rn(h, k1));
            const double y2 = __dadd_rn(dth1, __dmul_rn(h, k2)), y3 = __dadd_rn(dth2, __dmul_rn(h, k3));
            acrobot_accel(y0, y1, y2, y3, a, k2, k3);
            k0 = y2;
            k1 = y3;
            const double c = stage < 3 ? 2.0 : 1.0;
            s0 = __dadd_rn(s0, __dmul_rn(c, k0));
            s1 = __dadd_rn(s1, __dmul_rn(c, k1));
            s2 = __dadd_rn(s2, __dmul_rn(c, k2));
            s3 = __dadd_rn(s3, __dmul_rn(c, k3));
        }
        const double d6 = __ddiv_rn(dt, 6.0);
        th1 = wrap(__dadd_rn(th1, __dmul_rn(d6, s0)));
        th2 = wrap(__dadd_rn(th2, __dmul_rn(d6, s1)));
        dth1 = bound(__dadd_rn(dth1, __dmul_rn(d6, s2)), __dmul_rn(4.0, CUDART_PI));     // MAX_VEL_1 = 4 * pi
        dth2 = bound(__dadd_rn(dth2, __dmul_rn(d6, s3)), __dmul_rn(9.0, CUDART_PI));     // MAX_VEL_2 = 9 * pi
        // _terminal: -cos(s[0]) - cos(s[1] + s[0]) > 1.0; reward -1, 0 on the terminating step
        const bool done = __dsub_rn(-cos(th1), cos(__dadd_rn(th2, th1))) > 1.0;
        reward = done ? 0 : -1;
        return done;
    }
};

// MountainCar-v0 (gymnasium mountain_car.py): state (position, velocity), reward -1 on every step.
struct MountainCarTask {
    static constexpr int STATE_DIM = 2, OB_DIM = 2, ACTIONS = 3, TIME_LIMIT = 200;
    static constexpr int MIN_CTAS = 6;            // 40 registers, no spills; 8 CTAs per SM (32 registers) spills
    static constexpr const char* OB_WHY = "MountainCar observations have ob_dim 2";
    static constexpr const char* OUT_WHY = "MountainCar has 3 actions (n_out 3)";
    double x, v;

    __device__ __forceinline__ explicit MountainCarTask(const double* s) : x(s[0]), v(s[1]) {}
    __device__ __forceinline__ void store(double* s) const {
        s[0] = x;
        s[1] = v;
    }
    __device__ __forceinline__ float ob(int k) const { return __double2float_rn(k == 0 ? x : v); }
    __device__ __forceinline__ bool step(int action, int& reward) {
        const double force = 0.001, gravity = 0.0025, max_speed = 0.07, min_position = -1.2, max_position = 0.6;
        // velocity += (action - 1) * force + math.cos(3 * position) * (-gravity); np.clip(velocity, -max_speed, max_speed)
        v = __dadd_rn(v, __dadd_rn(__dmul_rn((double)(action - 1), force), __dmul_rn(cos(__dmul_rn(3.0, x)), -gravity)));
        v = v < -max_speed ? -max_speed : (v > max_speed ? max_speed : v);
        // position += velocity; np.clip(position, min_position, max_position)
        x = __dadd_rn(x, v);
        x = x < min_position ? min_position : (x > max_position ? max_position : x);
        if (x == min_position && v < 0.0) v = 0.0;
        reward = -1;                                                  // the terminating step included
        return x >= 0.5 && v >= 0.0;                                  // goal_position 0.5, goal_velocity 0
    }
};

// argmax over the logits held by lanes 0..A-1: the first NaN if any logit is NaN, otherwise the first maximum
// (dense_small_kernel's rule).  For A = 2 this is (y0 != y0) ? 0 : ((y1 > y0 || y1 != y1) ? 1 : 0).
template <int A>
__device__ __forceinline__ int warp_argmax(float x) {
    int best = 0;
    float bv = __shfl_sync(0xffffffffu, x, 0);
#pragma unroll
    for (int j = 1; j < A; ++j) {
        const float y = __shfl_sync(0xffffffffu, x, j);
        if (bv == bv && (y > bv || y != y)) {
            best = j;
            bv = y;
        }
    }
    return best;
}

// Which nets the discrete episode kernel runs for task T: dense layers only (<= 4, every width <= 32), vector observations
// of dimension T::OB_DIM, T::ACTIONS outputs, ReLU hidden layers, no activation on the head, no batch norm.  On failure
// `why` names the reason.
template <class T>
static bool discrete_net_supported(const dne_net_desc* net, const char** why) {
    static_assert(T::OB_DIM <= EP_MAX_WIDTH && T::ACTIONS <= EP_MAX_WIDTH, "one lane per observation and per action");
    if (!episode_net_common(net, DISCRETE_MAX_LAYERS, T::OB_DIM, T::ACTIONS, T::OB_WHY, T::OUT_WHY, why)) return false;
    for (int l = 0; l < net->n_layers; ++l) {
        const dne_layer_desc& L = net->layers[l];
        const bool head = (l == net->n_layers - 1);
        if (L.cin > EP_MAX_WIDTH || L.cout > EP_MAX_WIDTH) { *why = "layer width above 32"; return false; }
        if (head ? L.act != DNE_ACT_NONE : L.act != DNE_ACT_RELU) {
            *why = "hidden layers must be ReLU and the head linear";
            return false;
        }
    }
    // the largest net the rules above allow (4 layers of width 32) has at most 3328 parameters
    if (net->num_params > 4096) { *why = "num_params too large for the shared-memory weights"; return false; }
    return true;
}

template <class T>
__global__ void __launch_bounds__(EP_WARPS * 32, T::MIN_CTAS)
discrete_episode_kernel(EpisodeNet net, const float* __restrict__ theta, const float* __restrict__ noise,
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

    T env(init_state + (int64_t)T::STATE_DIM * m);
    int ret = 0;                                                  // the sum of the rewards, exact
    int len = 0;
    bool done = false;
    while (!done && len < max_steps) {
        // lane k < OB_DIM holds observation component k (the others compute the last one and drop it: no branch)
        const float o = env.ob(lane < T::OB_DIM ? lane : T::OB_DIM - 1);
        float x = lane < T::OB_DIM ? o : 0.0f;
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
        int r;
        done = env.step(warp_argmax<T::ACTIONS>(x), r);
        ret += r;
        ++len;
    }
    if (lane == 0) {
        returns[m] = (float)ret;                                  // |ret| <= 500: exact
        lengths[m] = len;
        if (final_state) env.store(final_state + (int64_t)T::STATE_DIM * m);
    }
}

template <class T>
static int launch_discrete(const dne_net_desc* net, const float* theta, const float* noise, const int64_t* noise_idx,
                           const float* scale, const int32_t* theta_idx, int n_members, const double* init_state,
                           int max_steps, float* returns, int32_t* lengths, double* final_state, cudaStream_t st) {
    const EpisodeNet en = make_episode_net(net);
    const size_t smem = (size_t)EP_WARPS * en.P_pad * sizeof(float);
    if (smem > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(discrete_episode_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   (int)smem);
        if (e != cudaSuccess) return DNE_ERR_CUDA;
    }
    const unsigned grid = (unsigned)((n_members + EP_WARPS - 1) / EP_WARPS);
    discrete_episode_kernel<T><<<grid, EP_WARPS * 32, smem, st>>>(en, theta, noise, noise_idx, scale, theta_idx, n_members,
                                                                  init_state, max_steps, returns, lengths, final_state);
    DNE_LAUNCHED(1);
    return DNE_OK;
}

int dne_discrete_time_limit(int env) {
    switch (env) {
        case DNE_EPISODE_CARTPOLE: return CartPoleTask::TIME_LIMIT;
        case DNE_EPISODE_ACROBOT: return AcrobotTask::TIME_LIMIT;
        case DNE_EPISODE_MOUNTAINCAR: return MountainCarTask::TIME_LIMIT;
        default: return 0;
    }
}

bool dne_discrete_net_supported(int env, const dne_net_desc* net, const char** why) {
    switch (env) {
        case DNE_EPISODE_CARTPOLE: return discrete_net_supported<CartPoleTask>(net, why);
        case DNE_EPISODE_ACROBOT: return discrete_net_supported<AcrobotTask>(net, why);
        case DNE_EPISODE_MOUNTAINCAR: return discrete_net_supported<MountainCarTask>(net, why);
        default: *why = "unknown environment"; return false;
    }
}

int dne_launch_discrete_episodes(int env, const dne_net_desc* net, const float* theta, const float* noise,
                                 const int64_t* noise_idx, const float* scale, const int32_t* theta_idx, int n_members,
                                 const double* init_state, int max_steps, float* returns, int32_t* lengths,
                                 double* final_state, cudaStream_t st) {
    switch (env) {
        case DNE_EPISODE_CARTPOLE:
            return launch_discrete<CartPoleTask>(net, theta, noise, noise_idx, scale, theta_idx, n_members, init_state,
                                                 max_steps, returns, lengths, final_state, st);
        case DNE_EPISODE_ACROBOT:
            return launch_discrete<AcrobotTask>(net, theta, noise, noise_idx, scale, theta_idx, n_members, init_state,
                                                max_steps, returns, lengths, final_state, st);
        case DNE_EPISODE_MOUNTAINCAR:
            return launch_discrete<MountainCarTask>(net, theta, noise, noise_idx, scale, theta_idx, n_members, init_state,
                                                    max_steps, returns, lengths, final_state, st);
        default: return DNE_ERR_ARG;
    }
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
