// image_maze_kernels.cu -- the hard maze seen as an 84x84 overhead image (DESIGN.md 3.10), stepped and rendered on the
// device for the per-tick runner and the Atari conv policies.
//
// The dynamics are MazeTask's (maze_task.cuh), the same code the whole-episode kernels run; the discrete action index
// goes through a float32 table to MazeTask's two continuous actions.  The frame is a pure function of the walls and the
// navigator's (x, y, heading), in float32 with every operation an explicit round-to-nearest intrinsic and no
// transcendental, so a numpy referee (tests/image_maze_oracle.py) reproduces it bit for bit:
//   * pixel (i, j) (row i, column j) is tested at its centre (x0 + (j + 0.5) * upp, y0 + (i + 0.5) * upp), where
//     (x0, y0) are the walls' lower bounds and upp = ext / 84 the maze units per pixel, ext the larger of the walls'
//     extents in x and y (the aspect is kept; the shorter axis leaves the last rows or columns empty);
//   * background: 255 where a wall (Line::distance, MazeTask::line_distance) is at most half a pixel (upp / 2) from the
//     centre, else 0; rendered once per maze;
//   * navigator: a disc of radius 8 (dx^2 + dy^2 <= 64 from (x, y)) over the background, 64 on its front half (the
//     heading direction (hx, hy) dotted with (dx, dy) > 0) and 128 on the rest.  (hx, hy) is heading_dir()'s
//     polynomial, not cosf / sinf, whose last bits differ between CUDA and the host C library.
// The 84x84x4 stack of a slot (NHWC, newest plane last) is preprocess_kernel's mode-0 frame stack restated for a
// gathered slot list: a step shifts the planes left and appends the new frame, a reset fills all four with the first.
#include "common.cuh"
#include "maze_task.cuh"

namespace {
constexpr int RES = 84, NPIX = RES * RES;
constexpr int IM_THREADS = 256;                   // one CTA per slot: warp 0 steps, every thread renders

struct ImageMazeParams {
    MazeParams maze;
    float x0, y0, upp, half;                      // frame origin, maze units per pixel, half a pixel
    float actions[DNE_IMAGE_MAZE_MAX_ACTIONS][2]; // action index -> (turn, speed), MazeTask's a[0], a[1]
    int n_actions;
};

// (cos, sin) of the heading in degrees, to about 1e-3: the quadrant k = floor(h / 90), the remainder f in degrees,
// Taylor polynomials of x = f * pi / 180 in Horner form, then the quadrant's rotation.  Rendering only needs a direction.
__device__ __forceinline__ void heading_dir(float h, float& hx, float& hy) {
    const float q = floorf(__fdiv_rn(h, 90.0f));
    const float f = __fsub_rn(h, __fmul_rn(90.0f, q));
    const float x = __fmul_rn(f, 0.0174532925f), x2 = __fmul_rn(x, x);
    const float s = __fmul_rn(x, __fadd_rn(1.0f, __fmul_rn(x2, __fadd_rn(-0.166666667f, __fmul_rn(x2,
                              __fadd_rn(0.00833333333f, __fmul_rn(x2, -0.000198412698f)))))));
    const float c = __fadd_rn(1.0f, __fmul_rn(x2, __fadd_rn(-0.5f, __fmul_rn(x2,
                              __fadd_rn(0.0416666667f, __fmul_rn(x2, -0.00138888889f))))));
    const int k = (q == q && fabsf(q) < 1e6f) ? ((int)q & 3) : 0;
    hx = k == 0 ? c : k == 1 ? -s : k == 2 ? -c : s;
    hy = k == 0 ? s : k == 1 ? c : k == 2 ? -s : -c;
}

__device__ __forceinline__ void pixel_centre(const ImageMazeParams& p, int pix, float& cx, float& cy) {
    const int i = pix / RES, j = pix - i * RES;
    cx = __fadd_rn(p.x0, __fmul_rn(__fadd_rn((float)j, 0.5f), p.upp));
    cy = __fadd_rn(p.y0, __fmul_rn(__fadd_rn((float)i, 0.5f), p.upp));
}

// Every thread of the CTA: the frame of a navigator at (x, y, heading) pushed onto (fill: written four times into) the
// slot's stack
__device__ __forceinline__ void render_push(const ImageMazeParams& p, const uint8_t* __restrict__ bg, float x, float y,
                                            float heading, uint32_t* __restrict__ stack, bool fill) {
    float hx, hy;
    heading_dir(heading, hx, hy);
    for (int pix = threadIdx.x; pix < NPIX; pix += blockDim.x) {
        float cx, cy;
        pixel_centre(p, pix, cx, cy);
        const float dx = __fsub_rn(cx, x), dy = __fsub_rn(cy, y);
        uint32_t v = bg[pix];
        if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) <= 64.0f)
            v = __fadd_rn(__fmul_rn(dx, hx), __fmul_rn(dy, hy)) > 0.0f ? 64u : 128u;
        stack[pix] = fill ? v * 0x01010101u : (stack[pix] >> 8) | (v << 24);     // little endian: plane 3 is the top byte
    }
}

__global__ void __launch_bounds__(256) image_maze_background_kernel(const __grid_constant__ ImageMazeParams p,
                                                                    uint8_t* __restrict__ plane) {
    const int pix = blockIdx.x * blockDim.x + threadIdx.x;
    if (pix >= NPIX) return;
    float cx, cy;
    pixel_centre(p, pix, cx, cy);
    bool wall = false;                            // an order-free OR over the walls
    for (int w = 0; w < p.maze.n_walls; ++w) wall = wall || MazeTask::line_distance(p.maze.walls[w], cx, cy) <= p.half;
    plane[pix] = wall ? 255 : 0;
}

__global__ void __launch_bounds__(IM_THREADS) image_maze_reset_kernel(const __grid_constant__ ImageMazeParams p,
                                                                       const uint8_t* __restrict__ bg,
                                                                       const double* __restrict__ init,
                                                                       const int32_t* __restrict__ slots,
                                                                       double* __restrict__ state,
                                                                       uint8_t* __restrict__ stacks) {
    const int e = blockIdx.x, slot = slots[e];
    const double* s = init + (int64_t)MazeTask::STATE_DIM * e;
    if (threadIdx.x < MazeTask::STATE_DIM) state[(int64_t)MazeTask::STATE_DIM * slot + threadIdx.x] = s[threadIdx.x];
    render_push(p, bg, (float)s[0], (float)s[1], (float)s[2], reinterpret_cast<uint32_t*>(stacks) + (int64_t)slot * NPIX,
                true);
}

__global__ void __launch_bounds__(IM_THREADS) image_maze_step_kernel(const __grid_constant__ ImageMazeParams p,
                                                                      const uint8_t* __restrict__ bg,
                                                                      const int32_t* __restrict__ slots,
                                                                      const int32_t* __restrict__ actions,
                                                                      double* __restrict__ state,
                                                                      uint8_t* __restrict__ stacks,
                                                                      float* __restrict__ reward,
                                                                      uint8_t* __restrict__ done,
                                                                      double* __restrict__ pos) {
    __shared__ float nav[3];                      // the stepped (x, y, heading)
    const int e = blockIdx.x, slot = slots[e];
    if (threadIdx.x < 32) {                       // MazeTask's 32 stepping lanes
        const int lane = threadIdx.x;
        double* s = state + (int64_t)MazeTask::STATE_DIM * slot;
        MazeTask env;
        env.load(s);
        const int act = (unsigned)actions[e] < (unsigned)p.n_actions ? actions[e] : 0;
        const float r = env.step(p.actions[act], p.maze, lane);
        if (lane == 0) {
            env.store(s);
            reward[e] = r;
            done[e] = env.t >= MazeTask::TIME_LIMIT;
            if (pos) {
                pos[2 * e] = env.x;
                pos[2 * e + 1] = env.y;
            }
            nav[0] = env.x;
            nav[1] = env.y;
            nav[2] = env.heading;
        }
    }
    __syncthreads();
    render_push(p, bg, nav[0], nav[1], nav[2], reinterpret_cast<uint32_t*>(stacks) + (int64_t)slot * NPIX, false);
}

// The kernels' parameters for `maze` (n_walls checked by the caller); false when the walls span no area
bool make_params(const dne_maze_desc* maze, ImageMazeParams* p) {
    *p = {};
    p->maze = make_maze_params(maze);
    float x0 = maze->walls[0][0], y0 = maze->walls[0][1], x1 = x0, y1 = y0;
    for (int j = 0; j < maze->n_walls; ++j)
        for (int c = 0; c < 4; c += 2) {
            const float x = maze->walls[j][c], y = maze->walls[j][c + 1];
            x0 = x < x0 ? x : x0;
            x1 = x > x1 ? x : x1;
            y0 = y < y0 ? y : y0;
            y1 = y > y1 ? y : y1;
        }
    const float ex = x1 - x0, ey = y1 - y0;
    const float ext = ex > ey ? ex : ey;
    if (!(ext > 0.0f) || !(ext < 1e30f)) return false;
    p->x0 = x0;
    p->y0 = y0;
    p->upp = ext / (float)RES;
    p->half = p->upp * 0.5f;
    return true;
}
}  // namespace

#define IMAGE_MAZE_CHECK(maze, p)                                                                                      \
    DNE_CHECK_ARG(maze, "null maze");                                                                                  \
    DNE_CHECK_ARG(maze->n_walls >= 1 && maze->n_walls <= DNE_MAZE_MAX_WALLS, "the image maze needs 1..64 walls");      \
    DNE_CHECK_ARG(make_params(maze, &p), "the walls span no area (or not a finite one)")

extern "C" int dne_image_maze_background(const dne_maze_desc* maze, uint8_t* d_plane, void* stream) {
    ImageMazeParams p;
    IMAGE_MAZE_CHECK(maze, p);
    DNE_CHECK_ARG(d_plane, "null pointer");
    image_maze_background_kernel<<<(NPIX + 255) / 256, 256, 0, (cudaStream_t)stream>>>(p, d_plane);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}

extern "C" int dne_image_maze_reset(const dne_maze_desc* maze, const uint8_t* d_background, const double* d_init,
                                    const int32_t* d_slots, int k, double* d_state, uint8_t* d_stacks, void* stream) {
    ImageMazeParams p;
    IMAGE_MAZE_CHECK(maze, p);
    DNE_CHECK_ARG(k >= 0, "k < 0");
    if (k == 0) return DNE_OK;
    DNE_CHECK_ARG(d_background && d_init && d_slots && d_state && d_stacks, "null pointer");
    image_maze_reset_kernel<<<k, IM_THREADS, 0, (cudaStream_t)stream>>>(p, d_background, d_init, d_slots, d_state,
                                                                        d_stacks);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}

extern "C" int dne_image_maze_step(const dne_maze_desc* maze, const uint8_t* d_background, const float* actions_host,
                                   int n_actions, const int32_t* d_slots, const int32_t* d_actions, int k,
                                   double* d_state, uint8_t* d_stacks, float* d_reward, uint8_t* d_done, double* d_pos,
                                   void* stream) {
    ImageMazeParams p;
    IMAGE_MAZE_CHECK(maze, p);
    DNE_CHECK_ARG(actions_host && n_actions >= 1 && n_actions <= DNE_IMAGE_MAZE_MAX_ACTIONS,
                  "the action table needs 1..32 rows");
    DNE_CHECK_ARG(k >= 0, "k < 0");
    if (k == 0) return DNE_OK;
    DNE_CHECK_ARG(d_background && d_slots && d_actions && d_state && d_stacks && d_reward && d_done, "null pointer");
    p.n_actions = n_actions;
    for (int a = 0; a < n_actions; ++a) {
        p.actions[a][0] = actions_host[2 * a];
        p.actions[a][1] = actions_host[2 * a + 1];
    }
    image_maze_step_kernel<<<k, IM_THREADS, 0, (cudaStream_t)stream>>>(p, d_background, d_slots, d_actions, d_state,
                                                                       d_stacks, d_reward, d_done, d_pos);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}
