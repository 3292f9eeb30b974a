// episode_kernels.cu -- whole episodes of a device-resident environment in one launch.
//
// CartPole-v1, Acrobot-v1, MountainCar-v0, Pendulum-v1 (gym classic_control) and the hard maze: the policy has a few
// hundred to a few tens of thousands of parameters and the environment step is a few dozen to a few hundred flops, so the
// per-tick runner (one forward launch + a device -> host -> device round trip per step) would spend nearly all its time on
// overhead.  Here a group of threads runs one member's episode from reset to the end: it builds the member's weights once
// in shared memory, then loops observation -> dense forward -> action -> environment step on the device.
//
// Numerics contract (DESIGN.md 3.5, 3.6, 3.7):
//   * weights w = fl(theta[row] + fl(scale * noise[idx + j])) -- the same rounding as every other forward of the engine;
//   * dense layers in fp32: each output a sequential fmaf over its inputs in index order, then + bias; the hidden layers'
//     activation is apply_act (common.cuh), the head is linear;
//   * the environment step in float64, in gym's operation order, every operation an explicit round-to-nearest intrinsic so
//     nvcc cannot contract it into FMAs; sin / cos are CUDA's double sin / cos.  The maze steps in the reference's float32
//     and double operations, explicit intrinsics too.
// No workspace, no atomics, no device RNG: reruns are bit-identical.
#include "common.cuh"
#include "forward.cuh"
#include "maze_task.cuh"
#include <math_constants.h>
#include <type_traits>

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

// Parameter j of a member: fl(theta[row][j] + fl(scale * noise[idx + j])), the rounding of every forward of the engine.
__device__ __forceinline__ float member_weight(const float* th, const float* nz, float s, int j) {
    return __fadd_rn(th[j], __fmul_rn(s, nz[j]));
}

// The member's weights, once per episode, by `nthr` threads starting at thread `t`.
__device__ __forceinline__ void build_member_weights(float* w, const EpisodeNet& net, const float* __restrict__ theta,
                                                     const float* __restrict__ noise, const int64_t* __restrict__ noise_idx,
                                                     const float* __restrict__ scale, const int32_t* __restrict__ theta_idx,
                                                     int m, int t, int nthr) {
    const float* th = theta + (theta_idx ? (int64_t)theta_idx[m] * net.P : 0);
    const float* nz = noise + noise_idx[m];
    const float s = scale[m];
    for (int j = t; j < net.P; j += nthr) w[j] = member_weight(th, nz, s, j);
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

// ---- continuous-action tasks: Pendulum-v1, the hard maze ---------------------------------------------------------------
// MujocoPolicy 'continuous:' nets.  One member per group of min(max layer width, 256) threads, rounded up to a warp
// (thread t owns outputs t, t + threads, ... of every layer); as many groups per CTA as maximise the members resident per
// SM, each group synchronised by its own named barrier.  The first Task::STEP_THREADS threads of a group (1, or the
// group's first warp) keep the task's state and compute its observation; thread 0 writes the normalised observation,
// keeps the observation sums, computes the linear head and adds the action noise; the same threads then step the task.
// A task type supplies OB_DIM, N_OUT, STATE_DIM, TIME_LIMIT, STEP_THREADS, its Params (passed by value to the kernel),
// load / store of the float64 state, ob(o, params, lane) (the full float32 observation in every stepping thread) and
// step(a, params, lane) (returns the float32 reward).
constexpr int CONT_CTA_THREADS = 256;
constexpr int CONT_MAX_GROUPS = 15;                   // named barriers 1..15 (0 is __syncthreads')
constexpr size_t CONT_SMEM_LIMIT = 227 * 1024;        // H100 opt-in shared memory per CTA

struct NoParams {};

// Pendulum-v1: gymnasium classic_control pendulum.py, g = 10, m = l = 1, dt = 0.05, max_speed = 8, max_torque = 2,
// TimeLimit 200, no termination.
struct PendulumTask {
    static constexpr int OB_DIM = 3, N_OUT = 1, STATE_DIM = 2, TIME_LIMIT = 200, STEP_THREADS = 1;
    static constexpr const char* OB_WHY = "Pendulum observations have ob_dim 3";
    static constexpr const char* OUT_WHY = "Pendulum has one continuous action (n_out 1)";
    static constexpr const char* BIN_OUT_WHY = "Pendulum's binned head scores n_bins bins of its one action (n_out n_bins)";
    using Params = NoParams;
    double th = 0.0, thdot = 0.0;

    __device__ __forceinline__ void load(const double* s) {
        th = s[0];
        thdot = s[1];
    }
    __device__ __forceinline__ void store(double* s) const {
        s[0] = th;
        s[1] = thdot;
    }
    __device__ __forceinline__ void ob(float* o, const Params&, int) const {      // float32([cos th, sin th, thdot])
        o[0] = __double2float_rn(cos(th));
        o[1] = __double2float_rn(sin(th));
        o[2] = __double2float_rn(thdot);
    }
    // one step with the float32 action a[0] (already noised); the float64 reward rounded to float32, as BatchEnv.step
    // returns it
    __device__ __forceinline__ float step(const float* a, const Params&, int) {
        return __double2float_rn(pendulum_step(th, thdot, a[0]));
    }

    // numpy's float64 divmod remainder (npy_divmod): fmod, then moved to the divisor's sign
    static __device__ __forceinline__ double py_mod(double a, double b) {
        double r = fmod(a, b);
        if (r != 0.0) {
            if ((r < 0.0) != (b < 0.0)) r = __dadd_rn(r, b);
        } else {
            r = copysign(0.0, b);
        }
        return r;
    }
    static __device__ __forceinline__ double pendulum_step(double& th, double& thdot, float a) {
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
};

// ---- discretised heads (MujocoPolicy 'uniform:N' / 'custom:v0,..,vk'; DESIGN.md 3.9) ----------------------------------
// The net scores N_OUT * nb bins, score d * nb + b being bin b of action dimension d; per dimension the action is the
// value of the bin with the highest score (the first NaN if any score is NaN, otherwise the first maximum: numpy's
// argmax), then the action noise is added.  The kernels take the head mode at compile time: BINNED = false is the linear
// head, whose parameters stay the task's own, so those instantiations are unchanged.
constexpr int BIN_MAX = 32;                           // bins per action dimension: one dimension's bins fit one warp

template <class Task>
struct BinnedParams {
    typename Task::Params task;
    float values[Task::N_OUT][BIN_MAX];               // the policy's bin table: values[d][b], b < nb
    int nb;
};

template <class Task, bool BINNED>
using EpisodeParams = typename std::conditional<BINNED, BinnedParams<Task>, typename Task::Params>::type;

template <class Task>
__device__ __forceinline__ const typename Task::Params& task_params(const typename Task::Params& p) { return p; }
template <class Task>
__device__ __forceinline__ const typename Task::Params& task_params(const BinnedParams<Task>& p) { return p.task; }

// The chosen bin of one action dimension, in every lane of the warp; lane b < nb holds bin b's score s.  "The first NaN,
// otherwise the first maximum" is the maximum under a total order (NaN above every number, then the larger value, then
// the smaller index), so a shuffle butterfly finds it in 5 rounds whatever the pairing.  Lanes past nb hold -inf with a
// larger index: they never win.
__device__ __forceinline__ int warp_bin_argmax(float s, int lane, int nb) {
    float v = lane < nb ? s : -CUDART_INF_F;
    int i = lane;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, v, off);
        const int oi = __shfl_xor_sync(0xffffffffu, i, off);
        const bool vn = v != v, on = ov != ov;
        if (vn != on ? on : (vn || ov == v ? oi < i : ov > v)) {
            v = ov;
            i = oi;
        }
    }
    return i;
}

// The binned head's scores: score j = sequential fmaf over the K inputs x in index order, then + bias (the linear head's
// operations), thread t of `threads` computing scores t, t + threads, ...; the weights are [K][NS] at wl, the bias at bl
// (nullptr: none).
__device__ __forceinline__ void bin_scores(const float* x, const float* wl, const float* bl, int K, int NS, float* y,
                                           int t, int threads) {
    for (int j = t; j < NS; j += threads) {
        float acc = 0.0f;
#pragma unroll 4
        for (int k = 0; k < K; ++k) acc = fmaf(x[k], wl[k * NS + j], acc);
        if (bl) acc = __fadd_rn(acc, bl[j]);
        y[j] = acc;
    }
}

// Warp 0 of the member, after the scores are in y: every lane takes each dimension's bin, its value and member m's action
// noise of this step (ac_noise nullable, [n][max_steps][N_OUT]); the lanes below Task::STEP_THREADS then step the task.
template <class Task>
__device__ __forceinline__ void binned_act_and_step(Task& env, const BinnedParams<Task>& prm, const float* y, int t,
                                                    const float* __restrict__ ac_noise, int m, int max_steps, int step,
                                                    double& ret, double& sret) {
    constexpr int NO = Task::N_OUT;
    const int nb = prm.nb;
    float a[NO];
#pragma unroll
    for (int d = 0; d < NO; ++d) {
        const int b = warp_bin_argmax(t < nb ? y[d * nb + t] : 0.0f, t, nb);
        a[d] = prm.values[d][b];
        if (ac_noise) a[d] = __fadd_rn(a[d], ac_noise[((int64_t)m * max_steps + step) * NO + d]);
    }
    __syncwarp();                                     // every lane's reads of y before any later write into it
    if (t < Task::STEP_THREADS) {
        const float r = env.step(a, prm.task, t);
        if (t == 0) {
            ret = __dadd_rn(ret, (double)r);
            sret = __dadd_rn(sret, r > 0.0f ? 1.0 : r < 0.0f ? -1.0 : (double)r);
        }
    }
}

struct ContinuousGeom {
    int threads;                                      // threads per member: min(max layer width, 256), a multiple of 32
    int act_pad;                                      // floats of one activation buffer: max layer width rounded up to 32
    size_t member_bytes;                              // weights + two activation buffers
};

template <class Task>
static ContinuousGeom continuous_geom(const dne_net_desc* net) {
    int width = Task::OB_DIM;
    for (int l = 0; l < net->n_layers; ++l) width = width > net->layers[l].cout ? width : net->layers[l].cout;
    ContinuousGeom g;
    g.act_pad = (width + 31) / 32 * 32;
    g.threads = g.act_pad < CONT_CTA_THREADS ? g.act_pad : CONT_CTA_THREADS;
    g.member_bytes = ((size_t)(net->num_params + 31) / 32 * 32 + 2 * (size_t)g.act_pad) * sizeof(float);
    return g;
}

// Which nets the continuous episode kernel runs for Task: 1..DNE_MAX_LAYERS dense layers, vector observations of
// dimension Task::OB_DIM, Task::N_OUT outputs, tanh or ReLU hidden layers, a linear head, no batch norm, and one member's
// weights plus its two activation buffers within one CTA's shared memory (for Pendulum hidden [200, 200] fits,
// [256, 256] does not).  Any layer width runs: a group has at most 256 threads, each looping over its outputs.
// A binned head checks the same with n_out = Task::N_OUT * nb.
template <class Task>
static bool continuous_net_layers(const dne_net_desc* net, const char** why, int n_out = Task::N_OUT,
                                  const char* out_why = Task::OUT_WHY) {     // every check but the size
    if (!episode_net_common(net, DNE_MAX_LAYERS, Task::OB_DIM, n_out, Task::OB_WHY, out_why, why)) return false;
    for (int l = 0; l < net->n_layers; ++l) {
        const int act = net->layers[l].act;
        if (l == net->n_layers - 1 ? act != DNE_ACT_NONE : (act != DNE_ACT_TANH && act != DNE_ACT_RELU)) {
            *why = "hidden layers must be tanh or ReLU and the head linear";
            return false;
        }
    }
    return true;
}

template <class Task>
static bool continuous_net_supported(const dne_net_desc* net, const char** why) {
    if (!continuous_net_layers<Task>(net, why)) return false;
    if (net->num_params > (1 << 24) || continuous_geom<Task>(net).member_bytes > CONT_SMEM_LIMIT) {
        *why = "one member's weights and activations exceed a CTA's shared memory (227 KB)";
        return false;
    }
    return true;
}

bool dne_pendulum_net_supported(const dne_net_desc* net, const char** why) {
    return continuous_net_supported<PendulumTask>(net, why);
}

bool dne_maze_net_supported(const dne_net_desc* net, const char** why) {
    return continuous_net_supported<MazeTask>(net, why);
}

__device__ __forceinline__ void group_sync(int id, int nthr) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthr) : "memory");
}

// ---- the cluster kernel's per-step pieces (thread 0 of the member runs them): continuous_episode_kernel's code, which
// keeps its own inline copy (routed through these helpers its maze instantiation compiles to other SASS, 0.3 % slower) ----
// Observation component k as the first layer takes it, normalised as ob_norm_kernel; with `sums`, the unnormalised value
// first goes into the member's float64 sums (ob_stat_accum_kernel's formula).
__device__ __forceinline__ float ob_input(const float* o, int k, bool sums, double* os, double* oq,
                                          const float* __restrict__ ob_mean, const float* __restrict__ ob_std) {
    if (sums) {
        os[k] = __dadd_rn(os[k], (double)o[k]);
        oq[k] = __dadd_rn(oq[k], __dmul_rn((double)o[k], (double)o[k]));
    }
    return ob_mean ? fminf(fmaxf(__fdiv_rn(__fsub_rn(o[k], ob_mean[k]), ob_std[k]), -5.0f), 5.0f) : o[k];
}

// The linear head over the K inputs x (weights w[off_w + k * NO + j], bias w[off_b + j] unless off_b < 0), plus member
// m's action noise of this step (ac_noise nullable, [n][max_steps][NO])
template <int NO>
__device__ __forceinline__ void linear_head(const float* x, const float* w, int off_w, int off_b, int K,
                                            const float* __restrict__ ac_noise, int m, int max_steps, int step, float* a) {
    const float* wl = w + off_w;
#pragma unroll
    for (int j = 0; j < NO; ++j) {
        float acc = 0.0f;
#pragma unroll 4
        for (int k = 0; k < K; ++k) acc = fmaf(x[k], wl[k * NO + j], acc);
        if (off_b >= 0) acc = __fadd_rn(acc, w[off_b + j]);
        a[j] = ac_noise ? __fadd_rn(acc, ac_noise[((int64_t)m * max_steps + step) * NO + j]) : acc;
    }
}

// The float32 reward into the float64 return and sign-return
__device__ __forceinline__ void add_reward(float r, double& ret, double& sret) {
    ret = __dadd_rn(ret, (double)r);
    sret = __dadd_rn(sret, r > 0.0f ? 1.0 : r < 0.0f ? -1.0 : (double)r);    // np.sign (0 -> 0, NaN -> NaN)
}

// Member m's outputs
template <class Task>
__device__ __forceinline__ void store_member(const Task& env, int m, int max_steps, double ret, double sret,
                                             const double* os, const double* oq, float* __restrict__ returns,
                                             float* __restrict__ signreturns, int32_t* __restrict__ lengths,
                                             double* __restrict__ final_state, double* __restrict__ ob_sum,
                                             double* __restrict__ ob_sumsq) {
    constexpr int OB = Task::OB_DIM;
    returns[m] = __double2float_rn(ret);
    signreturns[m] = __double2float_rn(sret);
    lengths[m] = max_steps;
    if (final_state) env.store(final_state + (int64_t)Task::STATE_DIM * m);
    if (ob_sum) {
#pragma unroll
        for (int k = 0; k < OB; ++k) {
            ob_sum[(int64_t)OB * m + k] = os[k];
            ob_sumsq[(int64_t)OB * m + k] = oq[k];
        }
    }
}

// No spills (registers in DESIGN.md 3.6, 3.7).  Shared memory bounds the residency: for Pendulum hidden [64, 64] keeps
// 12 members (24 warps) per SM, [128, 128] 3, [200, 200] 1.
// BINNED: the head is discretised (BinnedParams): every thread of the group computes its scores into the free activation
// buffer, one more group barrier, then warp 0 picks the bins (binned_act_and_step).
template <class Task, bool BINNED>
__global__ void __launch_bounds__(CONT_CTA_THREADS)
continuous_episode_kernel(EpisodeNet net, int threads, int act_pad, int groups, const __grid_constant__ EpisodeParams<Task, BINNED> prm,
                          const float* __restrict__ theta, const float* __restrict__ noise,
                          const int64_t* __restrict__ noise_idx, const float* __restrict__ scale,
                          const int32_t* __restrict__ theta_idx, int n_members, const double* __restrict__ init_state,
                          int max_steps, const float* __restrict__ ob_mean, const float* __restrict__ ob_std,
                          const float* __restrict__ ac_noise, float* __restrict__ returns, float* __restrict__ signreturns,
                          int32_t* __restrict__ lengths, double* __restrict__ final_state, double* __restrict__ ob_sum,
                          double* __restrict__ ob_sumsq) {
    constexpr int OB = Task::OB_DIM, NO = Task::N_OUT;
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

    Task env;
    double ret = 0.0, sret = 0.0;
    double os[OB], oq[OB];
#pragma unroll
    for (int k = 0; k < OB; ++k) os[k] = oq[k] = 0.0;
    if (t < Task::STEP_THREADS) env.load(init_state + (int64_t)Task::STATE_DIM * m);
    const int L = net.n_layers;
    for (int step = 0; step < max_steps; ++step) {
        if (t < Task::STEP_THREADS) {         // the observation, normalised as ob_norm_kernel
            float o[OB];
            env.ob(o, task_params<Task>(prm), t);
            if (t == 0) {
#pragma unroll
                for (int k = 0; k < OB; ++k) {
                    if (ob_sum) {             // ob_stat_accum_kernel's sums of the unnormalised observation
                        os[k] = __dadd_rn(os[k], (double)o[k]);
                        oq[k] = __dadd_rn(oq[k], __dmul_rn((double)o[k], (double)o[k]));
                    }
                    buf0[k] = ob_mean ? fminf(fmaxf(__fdiv_rn(__fsub_rn(o[k], ob_mean[k]), ob_std[k]), -5.0f), 5.0f)
                                      : o[k];
                }
            }
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
        if constexpr (BINNED) {               // the scores into y, which no thread reads again this step
            const int NS = net.cout[L - 1];
            bin_scores(x, w + net.off_w[L - 1], net.off_b[L - 1] >= 0 ? w + net.off_b[L - 1] : nullptr,
                       net.cin[L - 1], NS, y, t, threads);
            group_sync(bar, threads);
            if (t < 32) binned_act_and_step(env, prm, y, t, ac_noise, m, max_steps, step, ret, sret);
        } else if (t < Task::STEP_THREADS) {  // the linear head, the action noise, the environment step
            float a[NO];
            if (t == 0) {
                const int K = net.cin[L - 1];
                const float* wl = w + net.off_w[L - 1];
#pragma unroll
                for (int j = 0; j < NO; ++j) {
                    float acc = 0.0f;
#pragma unroll 4
                    for (int k = 0; k < K; ++k) acc = fmaf(x[k], wl[k * NO + j], acc);
                    if (net.off_b[L - 1] >= 0) acc = __fadd_rn(acc, w[net.off_b[L - 1] + j]);
                    a[j] = ac_noise ? __fadd_rn(acc, ac_noise[((int64_t)m * max_steps + step) * NO + j]) : acc;
                }
            }
            if (Task::STEP_THREADS > 1) {
#pragma unroll
                for (int j = 0; j < NO; ++j) a[j] = __shfl_sync(0xffffffffu, a[j], 0);
            }
            const float r = env.step(a, prm, t);
            if (t == 0) {
                ret = __dadd_rn(ret, (double)r);
                sret = __dadd_rn(sret, r > 0.0f ? 1.0 : r < 0.0f ? -1.0 : (double)r);    // np.sign (0 -> 0, NaN -> NaN)
            }
        }
    }
    if (t == 0) {
        returns[m] = __double2float_rn(ret);
        signreturns[m] = __double2float_rn(sret);
        lengths[m] = max_steps;
        if (final_state) env.store(final_state + (int64_t)Task::STATE_DIM * m);
        if (ob_sum) {
#pragma unroll
            for (int k = 0; k < OB; ++k) {
                ob_sum[(int64_t)OB * m + k] = os[k];
                ob_sumsq[(int64_t)OB * m + k] = oq[k];
            }
        }
    }
}

template <class Task, bool BINNED = false>
static int launch_continuous(const dne_net_desc* net, const EpisodeParams<Task, BINNED>& prm, const float* theta,
                             const float* noise, const int64_t* noise_idx, const float* scale, const int32_t* theta_idx,
                             int n_members, const double* init_state, int max_steps, const float* ob_mean,
                             const float* ob_std, const float* ac_noise, float* returns, float* signreturns,
                             int32_t* lengths, double* final_state, double* ob_sum, double* ob_sumsq, cudaStream_t st) {
    const EpisodeNet en = make_episode_net(net);
    const ContinuousGeom g = continuous_geom<Task>(net);
    auto kern = continuous_episode_kernel<Task, BINNED>;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CONT_SMEM_LIMIT) != cudaSuccess)
        return DNE_ERR_CUDA;
    // members per CTA: the count that keeps the most members resident per SM (registers, shared memory, threads, as the
    // occupancy calculator counts them); on a tie the more (Pendulum hidden [64, 64], 5000 members on an H100: 4 per CTA
    // 2.74 and 2.84 ms in two runs, 2 per CTA 3.05 ms, both with 12 members resident per SM)
    int groups = 1, best = 0;
    const int max_groups = CONT_CTA_THREADS / g.threads < CONT_MAX_GROUPS ? CONT_CTA_THREADS / g.threads : CONT_MAX_GROUPS;
    for (int gr = 1; gr <= max_groups && (size_t)gr * g.member_bytes <= CONT_SMEM_LIMIT; ++gr) {
        int blocks = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, kern, gr * g.threads, (size_t)gr * g.member_bytes) !=
            cudaSuccess)
            return DNE_ERR_CUDA;
        if (blocks * gr >= best) {
            best = blocks * gr;
            groups = gr;
        }
    }
    const size_t smem = (size_t)groups * g.member_bytes;
    const unsigned grid = (unsigned)((n_members + groups - 1) / groups);
    kern<<<grid, groups * g.threads, smem, st>>>(en, g.threads, g.act_pad, groups, prm, theta, noise, noise_idx, scale,
                                                 theta_idx, n_members, init_state, max_steps, ob_mean, ob_std, ac_noise,
                                                 returns, signreturns, lengths, final_state, ob_sum, ob_sumsq);
    DNE_LAUNCHED(1);
    return DNE_OK;
}

int dne_launch_pendulum_episodes(const dne_net_desc* net, const float* theta, const float* noise, const int64_t* noise_idx,
                                 const float* scale, const int32_t* theta_idx, int n_members, const double* init_state,
                                 int max_steps, const float* ob_mean, const float* ob_std, const float* ac_noise,
                                 float* returns, float* signreturns, int32_t* lengths, double* final_state, double* ob_sum,
                                 double* ob_sumsq, cudaStream_t st) {
    return launch_continuous<PendulumTask>(net, NoParams{}, theta, noise, noise_idx, scale, theta_idx, n_members,
                                           init_state, max_steps, ob_mean, ob_std, ac_noise, returns, signreturns, lengths,
                                           final_state, ob_sum, ob_sumsq, st);
}

int dne_launch_maze_episodes(const dne_maze_desc* maze, const dne_net_desc* net, const float* theta, const float* noise,
                             const int64_t* noise_idx, const float* scale, const int32_t* theta_idx, int n_members,
                             const double* init_state, int max_steps, const float* ob_mean, const float* ob_std,
                             const float* ac_noise, float* returns, float* signreturns, int32_t* lengths,
                             double* final_state, double* ob_sum, double* ob_sumsq, cudaStream_t st) {
    return launch_continuous<MazeTask>(net, make_maze_params(maze), theta, noise, noise_idx, scale, theta_idx, n_members,
                                       init_state, max_steps, ob_mean, ob_std, ac_noise, returns, signreturns, lengths,
                                       final_state, ob_sum, ob_sumsq, st);
}

// ---- continuous-action members too wide for one CTA: one member per thread-block cluster --------------------------------
// MujocoPolicy's [256, 256] net (humanoid*.json) is 264-273 KiB of weights and activations, above a CTA's 227 KB.  Here
// one member runs on a cluster of c in {2, 4, 8} CTAs (portable sizes), one group per CTA, and its weights are spread over
// the cluster's shared memory (DSMEM, Hopper's distributed shared memory).  Layer l's N outputs are dealt to the ranks in
// contiguous slices of S = ceil(N / c) (the last slices shorter or empty): rank r keeps its columns of W_l compacted to
// [K][S] (columns past its slice unused) and its slice of the bias; the linear head lives on rank 0.  Every output is
// still one thread's sequential fmaf over all K inputs in index order, then + bias, then apply_act, from weights built
// with the same fl(theta + fl(scale * noise)), so every operation, and every result, equals continuous_episode_kernel's.
// The K reduction is never split: that would change the fmaf order.
// Per step: rank 0's stepping threads form the observation and thread 0 pushes it, normalised, into every rank's input
// buffer; each hidden layer's slice is pushed into every rank's output buffer (ping-pong); rank 0 runs the head, adds the
// action noise and steps the task.  Remote stores are st.shared::cluster to mapa-translated addresses; the cluster
// barrier is barrier.cluster.arrive.release / wait.acquire, so the stores before it are visible to every rank after it.
constexpr int CLUSTER_MAX = 8;                        // the largest portable cluster size
constexpr int CLUSTER_SIZES[3] = {2, 4, 8};

struct ClusterNet {
    EpisodeNet net;                                   // the layers as theta lays them out
    int slice[DNE_MAX_LAYERS];                        // hidden layer l: outputs per rank, ceil(cout / c)
    int woff[DNE_MAX_LAYERS];                         // hidden layer l: this rank's weights [cin][slice], then bias [slice]
    int head_off;                                     // rank 0: the head's weights [cin][n_out], then bias [n_out]
    int buf_off;                                      // the two activation buffers, act_pad floats each
    int act_pad;                                      // the widest layer (or observation) rounded up to 32 floats
};

struct ClusterGeom {
    ClusterNet cn;
    int c;                                            // CTAs per member
    int threads;                                      // threads per CTA: the widest slice rounded up to 32, at most 256
    size_t smem;                                      // dynamic shared memory per CTA (every rank gets rank 0's size)
};

// The split of a net that passed continuous_net_layers over c ranks
template <class Task>
static ClusterGeom cluster_geom(const dne_net_desc* net, int c) {
    ClusterGeom g;
    g.c = c;
    g.cn.net = make_episode_net(net);
    int width = Task::OB_DIM, max_slice = 0, off = 0;
    const int L = net->n_layers;
    for (int l = 0; l < DNE_MAX_LAYERS; ++l) g.cn.slice[l] = g.cn.woff[l] = 0;
    for (int l = 0; l < L; ++l) {
        const int K = net->layers[l].cin, N = net->layers[l].cout;
        width = width > N ? width : N;
        if (l + 1 < L) {
            const int S = (N + c - 1) / c;
            g.cn.slice[l] = S;
            g.cn.woff[l] = off;
            off += (K + 1) * S;
            max_slice = max_slice > S ? max_slice : S;
        } else {
            g.cn.head_off = off;
            off += (K + 1) * N;
        }
    }
    g.cn.buf_off = (off + 31) / 32 * 32;
    g.cn.act_pad = (width + 31) / 32 * 32;
    const int thr = (max_slice + 31) / 32 * 32;
    g.threads = thr < 32 ? 32 : (thr > CONT_CTA_THREADS ? CONT_CTA_THREADS : thr);
    g.smem = ((size_t)g.cn.buf_off + 2 * (size_t)g.cn.act_pad) * sizeof(float);
    return g;
}

// Which nets the cluster kernel runs for Task: continuous_net_supported's, except that the size limit is on one rank's
// slices at c = 8 (the smallest) instead of on the whole member.  Hidden [256, 256] runs (maze: 142 KB per CTA at c = 2),
// [2048, 2048] does not (2.1 MB per CTA even at c = 8).
template <class Task>
static bool continuous_cluster_net_supported(const dne_net_desc* net, const char** why) {
    if (!continuous_net_layers<Task>(net, why)) return false;
    if (net->num_params > (1 << 24) || cluster_geom<Task>(net, CLUSTER_MAX).smem > CONT_SMEM_LIMIT) {
        *why = "one rank's slice of the weights and the activations exceed a CTA's shared memory (227 KB) even split "
               "over a cluster of 8";
        return false;
    }
    return true;
}

bool dne_pendulum_cluster_net_supported(const dne_net_desc* net, const char** why) {
    return continuous_cluster_net_supported<PendulumTask>(net, why);
}

bool dne_maze_cluster_net_supported(const dne_net_desc* net, const char** why) {
    return continuous_cluster_net_supported<MazeTask>(net, why);
}

__device__ __forceinline__ uint32_t cluster_addr(const float* p, int rank) {   // p in rank `rank`'s shared memory
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"((uint32_t)__cvta_generic_to_shared(p)), "r"(rank));
    return r;
}

__device__ __forceinline__ void cluster_store(const float* p, int rank, float v) {
    asm volatile("st.shared::cluster.f32 [%0], %1;" ::"r"(cluster_addr(p, rank)), "f"(v) : "memory");
}

// Every thread of every CTA of the cluster; the stores (local or remote) before it are visible to all of them after it
__device__ __forceinline__ void cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// BINNED: rank 0 keeps the discretised head's [cin][n_out] weights; its threads compute the scores into its free buffer,
// one CTA barrier, then its warp 0 picks the bins (binned_act_and_step).  The other ranks go on to the next observation's
// cluster barrier, which rank 0 reaches after its step, so nothing is stored into rank 0's buffers meanwhile.
template <class Task, bool BINNED>
__global__ void __launch_bounds__(CONT_CTA_THREADS)
continuous_cluster_episode_kernel(ClusterNet cn, const __grid_constant__ EpisodeParams<Task, BINNED> prm,
                                  const float* __restrict__ theta, const float* __restrict__ noise,
                                  const int64_t* __restrict__ noise_idx, const float* __restrict__ scale,
                                  const int32_t* __restrict__ theta_idx, int n_members,
                                  const double* __restrict__ init_state, int max_steps, const float* __restrict__ ob_mean,
                                  const float* __restrict__ ob_std, const float* __restrict__ ac_noise,
                                  float* __restrict__ returns, float* __restrict__ signreturns,
                                  int32_t* __restrict__ lengths, double* __restrict__ final_state,
                                  double* __restrict__ ob_sum, double* __restrict__ ob_sumsq) {
    constexpr int OB = Task::OB_DIM, NO = Task::N_OUT;
    extern __shared__ float ep_smem[];
    uint32_t c, rank;
    asm("mov.u32 %0, %%cluster_nctarank;" : "=r"(c));
    asm("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    const int m = blockIdx.x / c;                     // cluster index = member: the exit below is uniform over the cluster
    if (m >= n_members) return;                       // (before any access to a peer's shared memory)
    const int t = threadIdx.x, threads = blockDim.x;
    const EpisodeNet& net = cn.net;
    const int L = net.n_layers;
    float* w = ep_smem;
    float* buf0 = ep_smem + cn.buf_off;
    float* buf1 = buf0 + cn.act_pad;

    {   // this rank's slices of the member's weights (rank 0: and the head), element for element build_member_weights'
        const float* th = theta + (theta_idx ? (int64_t)theta_idx[m] * net.P : 0);
        const float* nz = noise + noise_idx[m];
        const float s = scale[m];
        for (int l = 0; l + 1 < L; ++l) {
            const int K = net.cin[l], N = net.cout[l], S = cn.slice[l], n0 = (int)rank * S;
            const int ns = N - n0 < S ? N - n0 : S;   // <= 0: an empty slice
            float* wl = w + cn.woff[l];
            for (int i = t; i < K * ns; i += threads) {
                const int k = i / ns, j = i - k * ns;
                wl[k * S + j] = member_weight(th, nz, s, net.off_w[l] + k * N + n0 + j);
            }
            if (net.off_b[l] >= 0)
                for (int j = t; j < ns; j += threads) wl[K * S + j] = member_weight(th, nz, s, net.off_b[l] + n0 + j);
        }
        if (rank == 0) {
            const int K = net.cin[L - 1], NH = BINNED ? net.cout[L - 1] : NO;
            float* wh = w + cn.head_off;
            for (int i = t; i < K * NH; i += threads) wh[i] = member_weight(th, nz, s, net.off_w[L - 1] + i);
            if (net.off_b[L - 1] >= 0)
                for (int j = t; j < NH; j += threads) wh[K * NH + j] = member_weight(th, nz, s, net.off_b[L - 1] + j);
        }
    }

    const bool stepper = rank == 0 && t < Task::STEP_THREADS;
    Task env;
    double ret = 0.0, sret = 0.0;
    double os[OB], oq[OB];
#pragma unroll
    for (int k = 0; k < OB; ++k) os[k] = oq[k] = 0.0;
    if (stepper) env.load(init_state + (int64_t)Task::STATE_DIM * m);
    // Every rank has started (its shared memory exists) and built its weights before the first remote store.
    cluster_sync();
    // Races: buffer b is read by the layer that takes it as input (every rank) and, when the last hidden layer wrote it,
    // by rank 0's head.  Every write into b, local or remote, comes after a cluster barrier that follows every read of b:
    // layer l writes the buffer layer l - 1 read, after layer l - 1's barrier; layer 0 writes buf1, which the previous
    // step's last hidden layer or head read, before the observation barrier; the observation goes into buf0, whose last
    // readers (a layer of the previous step, before that layer's barrier, or the head, by the thread that writes the
    // observation) are done.
    for (int step = 0; step < max_steps; ++step) {
        if (stepper) {                                // the observation, normalised as ob_norm_kernel, to every rank
            float o[OB];
            env.ob(o, task_params<Task>(prm), t);
            if (t == 0) {
#pragma unroll
                for (int k = 0; k < OB; ++k) {
                    const float v = ob_input(o, k, ob_sum != nullptr, os, oq, ob_mean, ob_std);
                    for (int q = 0; q < (int)c; ++q) cluster_store(buf0 + k, q, v);
                }
            }
        }
        cluster_sync();
        const float* x = buf0;
        float* y = buf1;
        for (int l = 0; l + 1 < L; ++l) {             // hidden layers: this rank's slice, pushed to every rank
            const int K = net.cin[l], S = cn.slice[l], n0 = (int)rank * S;
            const int ns = net.cout[l] - n0 < S ? net.cout[l] - n0 : S;
            const float* wl = w + cn.woff[l];
            for (int j = t; j < ns; j += threads) {
                float acc = 0.0f;
#pragma unroll 4
                for (int k = 0; k < K; ++k) acc = fmaf(x[k], wl[k * S + j], acc);
                if (net.off_b[l] >= 0) acc = __fadd_rn(acc, wl[K * S + j]);
                const float v = apply_act(acc, net.act[l]);
                for (int q = 0; q < (int)c; ++q) cluster_store(y + n0 + j, q, v);
            }
            cluster_sync();
            const float* nx = y;
            y = (float*)x;
            x = nx;
        }
        if constexpr (BINNED) {
            if (rank == 0) {
                const int K = net.cin[L - 1], NS = net.cout[L - 1];
                bin_scores(x, w + cn.head_off, net.off_b[L - 1] >= 0 ? w + cn.head_off + K * NS : nullptr, K, NS, y, t,
                           threads);
                __syncthreads();                      // rank 0's CTA only
                if (t < 32) binned_act_and_step(env, prm, y, t, ac_noise, m, max_steps, step, ret, sret);
            }
        } else if (stepper) {                         // rank 0: the linear head, the action noise, the environment step
            float a[NO];
            if (t == 0)
                linear_head<NO>(x, w, cn.head_off, net.off_b[L - 1] >= 0 ? cn.head_off + net.cin[L - 1] * NO : -1,
                                net.cin[L - 1], ac_noise, m, max_steps, step, a);
            if (Task::STEP_THREADS > 1) {
#pragma unroll
                for (int j = 0; j < NO; ++j) a[j] = __shfl_sync(0xffffffffu, a[j], 0);
            }
            const float r = env.step(a, prm, t);
            if (t == 0) add_reward(r, ret, sret);
        }
    }
    // No CTA leaves while a peer may still store into its shared memory.
    cluster_sync();
    if (rank == 0 && t == 0)
        store_member(env, m, max_steps, ret, sret, os, oq, returns, signreturns, lengths, final_state, ob_sum, ob_sumsq);
}

// Clusters of g resident on the device at once (the members one launch keeps in flight)
template <class Task, bool BINNED>
static cudaError_t cluster_residency(const ClusterGeom& g, int* clusters) {
    auto kern = continuous_cluster_episode_kernel<Task, BINNED>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)CONT_SMEM_LIMIT);
    if (e != cudaSuccess) return e;
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)g.c;
    attr[0].val.clusterDim.y = attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)g.c);
    cfg.blockDim = dim3((unsigned)g.threads);
    cfg.dynamicSmemBytes = g.smem;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaOccupancyMaxActiveClusters(clusters, (void*)kern, &cfg);
}

// The cluster size for `want` (0: automatic, else 2, 4 or 8; the caller checked the value and the net).  Automatic: among
// the sizes whose slices fit a CTA, the one with the most members resident on the device; on a tie the smaller.
template <class Task, bool BINNED = false>
static int choose_cluster(const dne_net_desc* net, int want, ClusterGeom* out, int* resident, const char** why) {
    int best = 0;
    for (int c : CLUSTER_SIZES) {
        if (want && c != want) continue;
        const ClusterGeom g = cluster_geom<Task>(net, c);
        if (g.smem > CONT_SMEM_LIMIT) continue;
        int k = 0;
        if (cluster_residency<Task, BINNED>(g, &k) != cudaSuccess) return DNE_ERR_CUDA;
        if (k > best) {
            best = k;
            *out = g;
        }
    }
    if (best == 0) {
        *why = want ? "one rank's slice of the weights and the activations exceed a CTA's shared memory (227 KB) at this "
                      "cluster size, or no such cluster fits the device"
                    : "no cluster size fits the device";
        return DNE_ERR_UNSUP;
    }
    *resident = best;
    return DNE_OK;
}

template <class Task>
static int cluster_geometry(const dne_net_desc* net, int cluster, int* out, const char** why) {
    ClusterGeom g;
    int resident = 0;
    const int rc = choose_cluster<Task>(net, cluster, &g, &resident, why);
    if (rc) return rc;
    out[0] = g.c;
    out[1] = g.threads;
    out[2] = (int)g.smem;
    out[3] = resident;
    return DNE_OK;
}

int dne_pendulum_cluster_geometry(const dne_net_desc* net, int cluster, int* out, const char** why) {
    return cluster_geometry<PendulumTask>(net, cluster, out, why);
}

int dne_maze_cluster_geometry(const dne_net_desc* net, int cluster, int* out, const char** why) {
    return cluster_geometry<MazeTask>(net, cluster, out, why);
}

template <class Task, bool BINNED = false>
static int launch_continuous_cluster(const dne_net_desc* net, const EpisodeParams<Task, BINNED>& prm, const float* theta,
                                     const float* noise, const int64_t* noise_idx, const float* scale,
                                     const int32_t* theta_idx, int n_members, const double* init_state, int max_steps,
                                     const float* ob_mean, const float* ob_std, const float* ac_noise, float* returns,
                                     float* signreturns, int32_t* lengths, double* final_state, double* ob_sum,
                                     double* ob_sumsq, int cluster, const char** why, cudaStream_t st) {
    ClusterGeom g;
    int resident = 0;
    const int rc = choose_cluster<Task, BINNED>(net, cluster, &g, &resident, why);
    if (rc) return rc;
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)g.c;
    attr[0].val.clusterDim.y = attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)((int64_t)n_members * g.c));
    cfg.blockDim = dim3((unsigned)g.threads);
    cfg.dynamicSmemBytes = g.smem;
    cfg.stream = st;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, continuous_cluster_episode_kernel<Task, BINNED>, g.cn, prm, theta,
                                             noise, noise_idx, scale, theta_idx, n_members, init_state, max_steps,
                                             ob_mean, ob_std, ac_noise, returns, signreturns, lengths, final_state, ob_sum,
                                             ob_sumsq);
    DNE_LAUNCHED(1);
    if (e != cudaSuccess) {
        *why = cudaGetErrorString(e);
        return DNE_ERR_CUDA;
    }
    return DNE_OK;
}

int dne_launch_pendulum_cluster_episodes(const dne_net_desc* net, const float* theta, const float* noise,
                                         const int64_t* noise_idx, const float* scale, const int32_t* theta_idx,
                                         int n_members, const double* init_state, int max_steps, const float* ob_mean,
                                         const float* ob_std, const float* ac_noise, float* returns, float* signreturns,
                                         int32_t* lengths, double* final_state, double* ob_sum, double* ob_sumsq,
                                         int cluster, const char** why, cudaStream_t st) {
    return launch_continuous_cluster<PendulumTask>(net, NoParams{}, theta, noise, noise_idx, scale, theta_idx, n_members,
                                                   init_state, max_steps, ob_mean, ob_std, ac_noise, returns, signreturns,
                                                   lengths, final_state, ob_sum, ob_sumsq, cluster, why, st);
}

int dne_launch_maze_cluster_episodes(const dne_maze_desc* maze, const dne_net_desc* net, const float* theta,
                                     const float* noise, const int64_t* noise_idx, const float* scale,
                                     const int32_t* theta_idx, int n_members, const double* init_state, int max_steps,
                                     const float* ob_mean, const float* ob_std, const float* ac_noise, float* returns,
                                     float* signreturns, int32_t* lengths, double* final_state, double* ob_sum,
                                     double* ob_sumsq, int cluster, const char** why, cudaStream_t st) {
    return launch_continuous_cluster<MazeTask>(net, make_maze_params(maze), theta, noise, noise_idx, scale, theta_idx,
                                               n_members, init_state, max_steps, ob_mean, ob_std, ac_noise, returns,
                                               signreturns, lengths, final_state, ob_sum, ob_sumsq, cluster, why, st);
}

// ---- discretised heads: one entry per task, the single-CTA kernel or a cluster ------------------------------------------
// Which nets the binned entry runs for Task with nb bins per action dimension: continuous_net_layers' checks with n_out =
// Task::N_OUT * nb, and the member within one CTA or, split, within a cluster of 8.
template <class Task>
static bool binned_net_supported(const dne_net_desc* net, int nb, const char** why) {
    if (nb < 2 || nb > BIN_MAX) {
        *why = "a binned head needs 2..32 bins per action dimension";
        return false;
    }
    if (!continuous_net_layers<Task>(net, why, Task::N_OUT * nb, Task::BIN_OUT_WHY)) return false;
    if (net->num_params > (1 << 24) || (continuous_geom<Task>(net).member_bytes > CONT_SMEM_LIMIT &&
                                        cluster_geom<Task>(net, CLUSTER_MAX).smem > CONT_SMEM_LIMIT)) {
        *why = "one rank's slice of the weights and the activations exceed a CTA's shared memory (227 KB) even split "
               "over a cluster of 8";
        return false;
    }
    return true;
}

bool dne_pendulum_binned_net_supported(const dne_net_desc* net, int nb, const char** why) {
    return binned_net_supported<PendulumTask>(net, nb, why);
}

bool dne_maze_binned_net_supported(const dne_net_desc* net, int nb, const char** why) {
    return binned_net_supported<MazeTask>(net, nb, why);
}

// cluster 0 with a member that fits one CTA: the single-CTA kernel; otherwise the cluster kernel at `cluster` (0:
// automatic).  `bins` is the host table [N_OUT][nb], copied into the kernel's parameters.
template <class Task>
static int launch_binned(const dne_net_desc* net, const typename Task::Params& tp, const float* bins, int nb,
                         const float* theta, const float* noise, const int64_t* noise_idx, const float* scale,
                         const int32_t* theta_idx, int n_members, const double* init_state, int max_steps,
                         const float* ob_mean, const float* ob_std, const float* ac_noise, float* returns,
                         float* signreturns, int32_t* lengths, double* final_state, double* ob_sum, double* ob_sumsq,
                         int cluster, const char** why, cudaStream_t st) {
    BinnedParams<Task> prm = {};
    prm.task = tp;
    prm.nb = nb;
    for (int d = 0; d < Task::N_OUT; ++d)
        for (int b = 0; b < nb; ++b) prm.values[d][b] = bins[d * nb + b];
    if (cluster == 0 && continuous_geom<Task>(net).member_bytes <= CONT_SMEM_LIMIT) {
        const int rc = launch_continuous<Task, true>(net, prm, theta, noise, noise_idx, scale, theta_idx, n_members,
                                                     init_state, max_steps, ob_mean, ob_std, ac_noise, returns,
                                                     signreturns, lengths, final_state, ob_sum, ob_sumsq, st);
        if (rc) *why = "the single-CTA kernel's attributes or occupancy could not be set";
        return rc;
    }
    return launch_continuous_cluster<Task, true>(net, prm, theta, noise, noise_idx, scale, theta_idx, n_members,
                                                 init_state, max_steps, ob_mean, ob_std, ac_noise, returns, signreturns,
                                                 lengths, final_state, ob_sum, ob_sumsq, cluster, why, st);
}

int dne_launch_pendulum_binned_episodes(const dne_net_desc* net, const float* theta, const float* noise,
                                        const int64_t* noise_idx, const float* scale, const int32_t* theta_idx,
                                        int n_members, const double* init_state, int max_steps, const float* ob_mean,
                                        const float* ob_std, const float* ac_noise, float* returns, float* signreturns,
                                        int32_t* lengths, double* final_state, double* ob_sum, double* ob_sumsq,
                                        const float* bins, int nb, int cluster, const char** why, cudaStream_t st) {
    return launch_binned<PendulumTask>(net, NoParams{}, bins, nb, theta, noise, noise_idx, scale, theta_idx, n_members,
                                       init_state, max_steps, ob_mean, ob_std, ac_noise, returns, signreturns, lengths,
                                       final_state, ob_sum, ob_sumsq, cluster, why, st);
}

int dne_launch_maze_binned_episodes(const dne_maze_desc* maze, const dne_net_desc* net, const float* theta,
                                    const float* noise, const int64_t* noise_idx, const float* scale,
                                    const int32_t* theta_idx, int n_members, const double* init_state, int max_steps,
                                    const float* ob_mean, const float* ob_std, const float* ac_noise, float* returns,
                                    float* signreturns, int32_t* lengths, double* final_state, double* ob_sum,
                                    double* ob_sumsq, const float* bins, int nb, int cluster, const char** why,
                                    cudaStream_t st) {
    return launch_binned<MazeTask>(net, make_maze_params(maze), bins, nb, theta, noise, noise_idx, scale, theta_idx,
                                   n_members, init_state, max_steps, ob_mean, ob_std, ac_noise, returns, signreturns,
                                   lengths, final_state, ob_sum, ob_sumsq, cluster, why, st);
}
