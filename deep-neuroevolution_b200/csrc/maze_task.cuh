// maze_task.cuh -- the hard maze's state and step (MazeTask), shared by the whole-episode kernels (episode_kernels.cu)
// and the per-tick image maze (image_maze_kernels.cu).
#pragma once
#include "common.cuh"

// The hard maze of the reference's GPU path (gym_tensorflow/maze/maze.h stepped as tf_maze.cpp's MazeEnvironment;
// DESIGN.md 3.7).  A navigator of radius 8 with 6 rangefinders (range 100) and a 4-sector goal radar; observation
// [1, range_i / 100, radar_j]; actions (turn, speed) + 0.5 through interpret_outputs' rate limits and clamps; Update()
// moves it unless the new position is within the radius of a wall; the only reward is -distance to the goal on the
// 400th step.  Single-precision C++ restated operation by operation: every float operation an explicit __f*_rn
// intrinsic (nvcc would contract products into FMAs), double where the C++ promotes, cosf / sinf / atanf where it calls
// the float overloads, double cos / sin where it calls those.  The state is float32 values kept in float64.
struct MazeParams {
    float4 walls[DNE_MAZE_MAX_WALLS];                 // (ax, ay, bx, by)
    int n_walls;
    int sticky;                                       // the file's collision flag: a hit freezes the navigator
    float gx, gy;                                     // goal
    float ray_dx[6], ray_dy[6];                       // fl(cosf(rad_i) * 100), fl(sinf(rad_i) * 100), host libm
};

__device__ __forceinline__ float maze_deg2rad(float deg) {   // angle/180.0*3.1415926 in double, stored to float
    return __double2float_rn(__dmul_rn(__ddiv_rn((double)deg, 180.0), 3.1415926));
}

__device__ __forceinline__ float maze_dist(float ax, float ay, float bx, float by) {   // Point(a).distance(b)
    const float dx = __fsub_rn(bx, ax), dy = __fsub_rn(by, ay);
    return __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
}

struct MazeTask {
    static constexpr int OB_DIM = 11, N_OUT = 2, STATE_DIM = 7, TIME_LIMIT = 400, STEP_THREADS = 32;
    static constexpr const char* OB_WHY = "maze observations have ob_dim 11";
    static constexpr const char* OUT_WHY = "the maze has two continuous actions (n_out 2)";
    static constexpr const char* BIN_OUT_WHY = "the maze's binned head scores n_bins bins of each of its two actions "
                                               "(n_out 2 * n_bins)";
    using Params = MazeParams;
    float x = 0.f, y = 0.f, heading = 0.f, speed = 0.f, ang_vel = 0.f;
    int t = 0;
    bool collide = false;

    __device__ __forceinline__ void load(const double* s) {
        x = (float)s[0];
        y = (float)s[1];
        heading = (float)s[2];
        speed = (float)s[3];
        ang_vel = (float)s[4];
        t = (int)s[5];
        collide = s[6] != 0.0;
    }
    __device__ __forceinline__ void store(double* s) const {
        s[0] = x;
        s[1] = y;
        s[2] = heading;
        s[3] = speed;
        s[4] = ang_vel;
        s[5] = t;
        s[6] = collide ? 1.0 : 0.0;
    }

    // Rangefinders: the 6 x n_walls ray-wall tests are dealt over the warp; each lane keeps a running minimum per ray
    // starting from the range 100, and the lanes' minima are combined with the same comparison.  The reference's
    // sequential `if (found < range) range = found` keeps the minimum of the numbers found (a NaN never compares less),
    // and a minimum under `<` is the same in any order, so the result is exact.
    __device__ __forceinline__ void ob(float* o, const Params& p, int lane) const {
        const float rh = maze_deg2rad(heading);
        const float c = cosf(rh), sn = sinf(rh);
        float rng[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) rng[i] = 100.0f;
        for (int k = lane; k < 6 * p.n_walls; k += 32) {
            const int ray = k / p.n_walls;
            const float4 w = p.walls[k - ray * p.n_walls];
            // the projected point (x + cos(rad)*100, y + sin(rad)*100) rotated by the heading about (x, y)
            const float ox = __fsub_rn(__fadd_rn(x, p.ray_dx[ray]), x), oy = __fsub_rn(__fadd_rn(y, p.ray_dy[ray]), y);
            const float px = __fadd_rn(__fsub_rn(__fmul_rn(c, ox), __fmul_rn(sn, oy)), x);
            const float py = __fadd_rn(__fadd_rn(__fmul_rn(sn, ox), __fmul_rn(c, oy)), y);
            // Line::intersection of the wall (A, B) with (x, y) -> (px, py); rBot and sBot are the same expression
            const float ay_c = __fsub_rn(w.y, y), ax_c = __fsub_rn(w.x, x), bax = __fsub_rn(w.z, w.x),
                        bay = __fsub_rn(w.w, w.y), dxc = __fsub_rn(px, x), dyc = __fsub_rn(py, y);
            const float rtop = __fsub_rn(__fmul_rn(ay_c, dxc), __fmul_rn(ax_c, dyc));
            const float rbot = __fsub_rn(__fmul_rn(bax, dyc), __fmul_rn(bay, dxc));
            const float stop = __fsub_rn(__fmul_rn(ay_c, bax), __fmul_rn(ax_c, bay));
            if (rbot == 0.0f) continue;
            const float r = __fdiv_rn(rtop, rbot), s = __fdiv_rn(stop, rbot);
            if (!(r > 0.0f && r < 1.0f && s > 0.0f && s < 1.0f)) continue;
            const float d = maze_dist(__fadd_rn(w.x, __fmul_rn(r, bax)), __fadd_rn(w.y, __fmul_rn(r, bay)), x, y);
#pragma unroll
            for (int i = 0; i < 6; ++i)
                if (ray == i && d < rng[i]) rng[i] = d;
        }
#pragma unroll
        for (int i = 0; i < 6; ++i) {
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                const float v = __shfl_xor_sync(0xffffffffu, rng[i], off);
                if (v < rng[i]) rng[i] = v;
            }
        }
        o[0] = 1.0f;
#pragma unroll
        for (int i = 0; i < 6; ++i) o[1 + i] = __fdiv_rn(rng[i], 100.0f);
        // the goal radar: the goal rotated by -heading about (x, y), moved to the navigator's frame, Point::angle()
        const float rg = maze_deg2rad(-heading);
        const float cg = cosf(rg), sg = sinf(rg);
        const float gx = __fsub_rn(p.gx, x), gy = __fsub_rn(p.gy, y);
        const float tx = __fsub_rn(__fadd_rn(__fsub_rn(__fmul_rn(cg, gx), __fmul_rn(sg, gy)), x), x);
        const float ty = __fsub_rn(__fadd_rn(__fadd_rn(__fmul_rn(sg, gx), __fmul_rn(cg, gy)), y), y);
        float ang;
        if (tx == 0.0f) {
            ang = ty > 0.0f ? 90.0f : 270.0f;
        } else {
            ang = __double2float_rn(__dmul_rn(__ddiv_rn((double)atanf(__fdiv_rn(ty, tx)), 3.1415926), 180.0));
            if (!(tx > 0.0f)) ang = __double2float_rn(__dadd_rn((double)ang, 180.0));
        }
        const double ang360 = __dadd_rn((double)ang, 360.0);
        const float lo[4] = {315.0f, 45.0f, 135.0f, 225.0f}, hi[4] = {405.0f, 135.0f, 225.0f, 315.0f};
#pragma unroll
        for (int j = 0; j < 4; ++j)      // half-open sectors, tested on the angle and on the angle + 360 (in double)
            o[7 + j] = ((ang >= lo[j] && ang < hi[j]) || (ang360 >= (double)lo[j] && ang360 < (double)hi[j])) ? 1.0f
                                                                                                             : 0.0f;
    }

    // Line::distance(n): the distance from (nx, ny) to the wall segment
    static __device__ __forceinline__ float line_distance(const float4 w, float nx, float ny) {
        const float bax = __fsub_rn(w.z, w.x), bay = __fsub_rn(w.w, w.y);
        const float utop = __fadd_rn(__fmul_rn(__fsub_rn(nx, w.x), bax), __fmul_rn(__fsub_rn(ny, w.y), bay));
        float ubot = maze_dist(w.x, w.y, w.z, w.w);
        ubot = __fmul_rn(ubot, ubot);
        float d;
        if (ubot == 0.0f) {
            d = 0.0f;
        } else {
            const float u = __fdiv_rn(utop, ubot);
            if (u < 0.0f || u > 1.0f) {
                const float d1 = maze_dist(w.x, w.y, nx, ny), d2 = maze_dist(w.z, w.w, nx, ny);
                d = d1 < d2 ? d1 : d2;
            } else {
                d = maze_dist(__fadd_rn(w.x, __fmul_rn(u, bax)), __fadd_rn(w.y, __fmul_rn(u, bay)), nx, ny);
            }
        }
        return d;
    }

    // Line::distance(n) < radius for one wall
    static __device__ __forceinline__ bool hits(const float4 w, float nx, float ny) { return line_distance(w, nx, ny) < 8.0f; }

    // interpret_outputs(float(a0) + 0.5, 0.5 + float(a1)), Update(), one more step taken; every lane of the warp steps
    // the same state, the collision tests (any wall within the radius, an order-free OR) dealt over the lanes
    __device__ __forceinline__ float step(const float* a, const Params& p, int lane) {
        float o1 = __double2float_rn(__dadd_rn((double)a[0], 0.5)), o2 = __double2float_rn(__dadd_rn(0.5, (double)a[1]));
        if (o1 > 1.0f) o1 = 1.0f;
        if (o1 < 0.0f) o1 = 0.0f;
        if (o2 > 1.0f) o2 = 1.0f;
        if (o2 < 0.0f) o2 = 0.0f;
        float d_ang = __fsub_rn(__double2float_rn(__dmul_rn(__dsub_rn((double)o1, 0.5), 6.0)), ang_vel);
        float d_speed = __fsub_rn(__double2float_rn(__dmul_rn(__dsub_rn((double)o2, 0.5), 6.0)), speed);
        if ((double)d_ang >= 0.2) d_ang = 0.2f;                   // float against double 0.2, assigned as float
        if ((double)d_ang <= -0.2) d_ang = -0.2f;
        if ((double)d_speed >= 0.2) d_speed = 0.2f;
        if ((double)d_speed <= -0.2) d_speed = -0.2f;
        ang_vel = __fadd_rn(ang_vel, d_ang);
        speed = __fadd_rn(speed, d_speed);
        if (speed > 3.0f) speed = 3.0f;
        if (speed < -3.0f) speed = -3.0f;
        if (ang_vel > 3.0f) ang_vel = 3.0f;
        if (ang_vel < -3.0f) ang_vel = -3.0f;
        // Update(): the velocity from the heading before the turn, in double
        const double h = __dmul_rn(__ddiv_rn((double)heading, 180.0), 3.1415926);
        const float vx = __double2float_rn(__dmul_rn(cos(h), (double)speed));
        const float vy = __double2float_rn(__dmul_rn(sin(h), (double)speed));
        heading = __fadd_rn(heading, ang_vel);
        if (heading > 360.0f) heading = __fsub_rn(heading, 360.0f);
        if (heading < 0.0f) heading = __fadd_rn(heading, 360.0f);
        const float nx = __fadd_rn(vx, x), ny = __fadd_rn(vy, y);
        bool hit = false;
        if (!collide) {
            for (int j = lane; j < p.n_walls; j += 32) hit = hit || hits(p.walls[j], nx, ny);
            hit = __any_sync(0xffffffffu, hit);
        }
        if (!collide && !hit) {
            x = nx;
            y = ny;
        } else if (p.sticky) {
            collide = true;
        }
        t += 1;
        if (t < TIME_LIMIT) return 0.0f;
        float d = maze_dist(x, y, p.gx, p.gy);                    // distance_to_target(): a NaN distance counts 500
        if (d != d) d = 500.0f;
        return -d;
    }
};

static inline MazeParams make_maze_params(const dne_maze_desc* maze) {
    MazeParams p = {};
    p.n_walls = maze->n_walls;
    p.sticky = maze->collisions_stick != 0;
    p.gx = maze->goal[0];
    p.gy = maze->goal[1];
    for (int j = 0; j < maze->n_walls; ++j)
        p.walls[j] = make_float4(maze->walls[j][0], maze->walls[j][1], maze->walls[j][2], maze->walls[j][3]);
    // the rangefinders' own directions: constant arguments, so computed here with the host C library's cosf / sinf,
    // which the reference calls too (float rad = angle/180.0*3.1415926; cos(rad)*range in float)
    const float angles[6] = {-90.0f, -45.0f, 0.0f, 45.0f, 90.0f, -180.0f};
    for (int i = 0; i < 6; ++i) {
        volatile float rad = (float)((double)angles[i] / 180.0 * 3.1415926);   // volatile: no compile-time folding
        p.ray_dx[i] = cosf(rad) * 100.0f;
        p.ray_dy[i] = sinf(rad) * 100.0f;
    }
    return p;
}
