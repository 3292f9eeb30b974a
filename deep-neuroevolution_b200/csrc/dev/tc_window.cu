// tc_window.cu -- DEV self-test of the "shifted window" A operand the convolution kernels rely on (conv_s2d.cu).
//
// An activation image is kept in shared memory as channel-quad planes  img[plane = c/4][pixel][4 channels]  (16 B per
// pixel, PIXP pixels per plane).  That IS the wgmma K-major no-swizzle canonical layout of a matrix whose rows are the
// pixels: 8 consecutive pixels = one 128-byte core matrix (SBO = 128), the next channel quad LBO = PIXP*16 bytes away.
// A stride-1 convolution tap (dy, dx) over a W-wide pixel grid reads, for output position m, pixel m + dy*W + dx: the
// SAME image at a start address shifted by (dy*W + dx)*16 bytes.  So one descriptor per (tap, channel octet) addresses the
// implicit-GEMM A tile with no im2col copy -- provided wgmma accepts a start address that is only 16-byte
// aligned and an LBO that is not a multiple of 128 bytes.  This test proves exactly that on the hardware, with the
// image brought in either by threads (generic proxy + fence.proxy.async) or by ONE cp.async.bulk (TMA, async proxy).
//
//   D[m][n] = sum_{tap} sum_{c} img[c/4][row0 + m + off[tap]][c%4] * Bw[n][tap*C + c]        m in [0,128), n in [0,N)
// Inputs are TF32-exact (the caller passes small integers), so the result must be exact.
#include "dev.cuh"
#include "../wgmma.cuh"
using namespace wg;

struct WindowArgs {
    int C, n_taps, PIXP, N, row0, use_tma, rows_total;   // rows_total: pixels per plane actually present in global memory
    int off[16];
};

template <int N>
__global__ void __launch_bounds__(128) tc_window_test_kernel(const float* __restrict__ img, const float* __restrict__ Bw,
                                                             float* __restrict__ D, WindowArgs a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 127) & ~(uintptr_t)127);
    const int n_planes = a.C / 4;
    const int LBO_A = a.PIXP * 16;
    const int img_bytes = n_planes * LBO_A;
    const int K = a.n_taps * a.C;
    constexpr int LBO_B = N * 16;
    uint8_t* sImg = smem;
    uint8_t* sB = smem + ((img_bytes + 4096 + 127) & ~127);          // slack: tile over-reach past the last plane
    __shared__ uint64_t tma_bar;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) { mbar_init(&tma_bar, 1); fence_mbar_init(); }
    // zero the slack (garbage rows must at least be finite)
    for (int i = tid; i < 4096 / 16; i += 128) *reinterpret_cast<float4*>(sImg + img_bytes + i * 16) = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    if (a.use_tma) {
        if (tid == 0) {
            mbar_arrive_expect_tx(&tma_bar, (uint32_t)img_bytes);
            bulk_g2s(sImg, img, (uint32_t)img_bytes, &tma_bar);
        }
    } else {
        for (int i = tid; i < img_bytes / 16; i += 128)
            *reinterpret_cast<float4*>(sImg + i * 16) = reinterpret_cast<const float4*>(img)[i];
    }
    for (int u = tid; u < N * (K / 4); u += 128) {                    // B[n][k] -> planes [k/4][n][4]
        const int n = u % N, q = u / N;
        *reinterpret_cast<float4*>(sB + q * LBO_B + n * 16) = *reinterpret_cast<const float4*>(Bw + (int64_t)n * K + 4 * q);
    }
    fence_proxy_async_smem();
    __syncthreads();
    if (a.use_tma) mbar_wait(&tma_bar, 0);
    float acc[2][N / 2];
    const uint32_t a0 = smem_u32(sImg), b0 = smem_u32(sB);
    wgmma_fence();
    for (int tap = 0; tap < a.n_taps; ++tap)
        for (int c8 = 0; c8 < a.C / 8; ++c8) {
            const uint64_t dB = smem_desc(b0 + ((tap * a.C + 8 * c8) / 4) * LBO_B, LBO_B, 128);
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const uint64_t dA = smem_desc(a0 + 2 * c8 * LBO_A + (a.row0 + t * 64 + a.off[tap]) * 16, LBO_A, 128);
                wgmma_tf32<N>(acc[t], dA, dB, (tap | c8) != 0);
            }
        }
    wgmma_commit();
    wgmma_wait<0>();
    fence_regs<N / 2>(acc[0]);
    fence_regs<N / 2>(acc[1]);
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = t * 64 + warp * 16 + (lane >> 2) + 8 * h, n = 8 * j + 2 * (lane & 3);
                D[m * N + n] = acc[t][4 * j + 2 * h];
                D[m * N + n + 1] = acc[t][4 * j + 2 * h + 1];
            }
}

template <int N>
static int launch_window(const float* d_img, const float* d_Bw, float* d_D, const WindowArgs& a, int smem, cudaStream_t st) {
    DNE_CUDA(cudaFuncSetAttribute(tc_window_test_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    tc_window_test_kernel<N><<<1, 128, smem, st>>>(d_img, d_Bw, d_D, a);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}

// img: float [C/4][PIXP][4] (TF32-exact values); Bw: float [N][n_taps*C]; D: float [128][N]; off: int[n_taps] pixel offsets.
extern "C" int dne_dev_tc_window(const float* d_img, const float* d_Bw, float* d_D, int C, int n_taps, const int* h_off,
                                 int PIXP, int N, int row0, int use_tma, void* stream) {
    DNE_CHECK_ARG(d_img && d_Bw && d_D && h_off && C % 8 == 0 && n_taps >= 1 && n_taps <= 16 &&
                  (N == 16 || N == 32 || N == 64 || N == 128),
                  "bad arguments");
    WindowArgs a;
    a.C = C; a.n_taps = n_taps; a.PIXP = PIXP; a.N = N; a.row0 = row0; a.use_tma = use_tma; a.rows_total = PIXP;
    for (int i = 0; i < 16; ++i) a.off[i] = i < n_taps ? h_off[i] : 0;
    const int smem = (C / 4) * PIXP * 16 + 4096 + 128 + N * n_taps * C * 4 + 256;
    DNE_CHECK_ARG(smem <= 227 * 1024, "does not fit shared memory");
    cudaStream_t st = (cudaStream_t)stream;
    if (N == 16) return launch_window<16>(d_img, d_Bw, d_D, a, smem, st);
    if (N == 32) return launch_window<32>(d_img, d_Bw, d_D, a, smem, st);
    if (N == 64) return launch_window<64>(d_img, d_Bw, d_D, a, smem, st);
    return launch_window<128>(d_img, d_Bw, d_D, a, smem, st);
}
