// tc_selftest.cu -- self-test of the wgmma plumbing (descriptors, register accumulators, wgmma fence / commit / wait,
// 3xTF32 split) used by tests/test_gpu_tc.py.  Part of the DEV library libdne_dev.so, not of the product ABI (include/dne.h).
#include "dev.cuh"
#include "../wgmma.cuh"
using namespace wg;

// =====================================================================================================
// Self-test of the wgmma plumbing: C[128,N] = A[128,K] * B[N,K]^T with the same staging / descriptor / 3xTF32 code
// path (single CTA = one warpgroup, two m64 tiles).  Exposed by libdne_dev.so for tests/test_gpu_tc.py.
// =====================================================================================================
template <int N>
__global__ void __launch_bounds__(128) tc_gemm_test_kernel(const float* __restrict__ A, const float* __restrict__ B,
                                                           float* __restrict__ C, int K) {
    constexpr int KC = 32;
    constexpr int A_PLANE = 128 * 16, B_PLANE = N * 16;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 127) & ~(uintptr_t)127);
    uint8_t* sA_hi = smem;
    uint8_t* sA_lo = sA_hi + (KC / 4) * A_PLANE;
    uint8_t* sB_hi = sA_lo + (KC / 4) * A_PLANE;
    uint8_t* sB_lo = sB_hi + (KC / 4) * B_PLANE;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    float acc[2][N / 2];
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[t][i] = 0.0f;
    for (int k0 = 0; k0 < K; k0 += KC) {
        for (int u = tid; u < 128 * (KC / 4); u += 128) {
            const int r = u % 128, q = u / 128;
            const float4 v = *reinterpret_cast<const float4*>(A + (int64_t)r * K + k0 + 4 * q);
            float4 hi, lo;
            split_tf32(v.x, hi.x, lo.x); split_tf32(v.y, hi.y, lo.y); split_tf32(v.z, hi.z, lo.z); split_tf32(v.w, hi.w, lo.w);
            *reinterpret_cast<float4*>(sA_hi + q * A_PLANE + r * 16) = hi;
            *reinterpret_cast<float4*>(sA_lo + q * A_PLANE + r * 16) = lo;
        }
        for (int u = tid; u < N * (KC / 4); u += 128) {
            const int n = u % N, q = u / N;
            const float4 v = *reinterpret_cast<const float4*>(B + (int64_t)n * K + k0 + 4 * q);
            float4 hi, lo;
            split_tf32(v.x, hi.x, lo.x); split_tf32(v.y, hi.y, lo.y); split_tf32(v.z, hi.z, lo.z); split_tf32(v.w, hi.w, lo.w);
            *reinterpret_cast<float4*>(sB_hi + q * B_PLANE + n * 16) = hi;
            *reinterpret_cast<float4*>(sB_lo + q * B_PLANE + n * 16) = lo;
        }
        fence_proxy_async_smem();
        __syncthreads();
        wgmma_fence();
#pragma unroll
        for (int k8 = 0; k8 < KC / 8; ++k8) {
            const uint64_t dBh = smem_desc(smem_u32(sB_hi) + 2 * k8 * B_PLANE, B_PLANE, 128);
            const uint64_t dBl = smem_desc(smem_u32(sB_lo) + 2 * k8 * B_PLANE, B_PLANE, 128);
#pragma unroll
            for (int t = 0; t < 2; ++t) {
                const uint64_t dAh = smem_desc(smem_u32(sA_hi) + 2 * k8 * A_PLANE + t * 1024, A_PLANE, 128);
                const uint64_t dAl = smem_desc(smem_u32(sA_lo) + 2 * k8 * A_PLANE + t * 1024, A_PLANE, 128);
                wgmma_tf32<N>(acc[t], dAh, dBh, 1);
                wgmma_tf32<N>(acc[t], dAl, dBh, 1);
                wgmma_tf32<N>(acc[t], dAh, dBl, 1);
            }
        }
        wgmma_commit();
        wgmma_wait<0>();                   // synchronous version: wait before re-staging
        fence_regs<N / 2>(acc[0]);
        fence_regs<N / 2>(acc[1]);
        __syncthreads();
    }
#pragma unroll
    for (int t = 0; t < 2; ++t)
#pragma unroll
        for (int j = 0; j < N / 8; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = t * 64 + warp * 16 + (lane >> 2) + 8 * h, n = 8 * j + 2 * (lane & 3);
                *reinterpret_cast<float2*>(C + (int64_t)m * N + n) = make_float2(acc[t][4 * j + 2 * h], acc[t][4 * j + 2 * h + 1]);
            }
}

extern "C" int dne_test_tc_gemm(const float* d_A, const float* d_B, float* d_C, int K, int N, void* stream) {
    DNE_CHECK_ARG(d_A && d_B && d_C && K > 0 && K % 32 == 0 && (N == 16 || N == 32 || N == 64), "bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const int smem = 2 * 8 * 128 * 16 + 2 * 8 * N * 16 + 128;
    if (N == 16) {
        DNE_CUDA(cudaFuncSetAttribute(tc_gemm_test_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        tc_gemm_test_kernel<16><<<1, 128, smem, st>>>(d_A, d_B, d_C, K);
    } else if (N == 32) {
        DNE_CUDA(cudaFuncSetAttribute(tc_gemm_test_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        tc_gemm_test_kernel<32><<<1, 128, smem, st>>>(d_A, d_B, d_C, K);
    } else {
        DNE_CUDA(cudaFuncSetAttribute(tc_gemm_test_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        tc_gemm_test_kernel<64><<<1, 128, smem, st>>>(d_A, d_B, d_C, K);
    }
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}
