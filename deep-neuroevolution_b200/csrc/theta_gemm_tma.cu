// theta_gemm_tma.cu -- the shared-theta part of a dense layer, X[slots,K] . theta_w[K,N], as a pure TMA + wgmma kernel.
//
//   part[split][m][n] = sum_{k in split} X[m][k] * W[k][n]          (same contract as theta_gemm_tc_kernel / dense_theta_gemm_kernel)
//
// theta_gemm_tc_kernel (tc_conv.cu) stages both operands through the threads (global -> registers -> TF32 split ->
// st.shared) with a block barrier per 16-wide chunk.  Here both operands already exist in global memory in the wgmma
// K-major canonical layout, as 2 x fp16 splits (wgmma.cuh: x = h0 + h1*2^-11; f16 wgmma runs at twice the MAC rate of
// tf32 and the operands are half the bytes):
//   * W changes once per generation: dne_theta_prepare() relays it out (theta_prep_kernel) into
//       Wc[n tile of 128][k octet][h0 | h1][128 n][8 k]     one k-octet plane = [B_h0 ; B_h1] stacked along N = 4 KB
//   * X is the output of the last convolution: its epilogue (conv_s2d.cu) writes, besides the NHWC vector the noise GEMV
//     streams, the same values as
//       Xc[m tile of 128][k octet][h0 | h1][128 slots][8 k] one k-octet plane = [A_h0 ; A_h1] = 4 KB
// so a K chunk of 32 of either operand is one contiguous 16 KB run and the whole main loop is: one producer thread issuing
// cp.async.bulk into a 4-stage ring and two MMA warpgroups, each issuing A_h0*[B_h0;B_h1] as one N = 256 wgmma into its
// [main | correction] accumulator registers plus A_h1*B_h0 into the correction half (result = main + 2^-11 * correction)
// for one m64 half of the CTA's 128 x 128 tile; no staging threads at all.  A CTA owns one M tile, one N tile and one K
// split; partials are deterministic.
// Optionally (dne_set_option("theta_mc", 1)) the N tiles of one K split form a thread-block cluster: every CTA fetches
// 1/CL of the shared A chunk and MULTICASTS it into all CL CTAs' stages (cp.async.bulk ... .multicast::cluster), so X
// crosses the L2 -> SM fabric once per split instead of once per N tile; a stage is recycled when the MMA warps of ALL CL
// CTAs have read it (remote mbarrier arrivals on every peer's empty barrier).
#include "common.cuh"
#include "forward.cuh"
#include "wgmma.cuh"

using namespace wg;

int g_dne_theta_mc = 0;
namespace {
constexpr int TGM_KC = 32, TGM_STAGES = 4;                 // 32 k = four k-octet planes per chunk
constexpr int TGM_PLANE = 256 * 16;                         // bytes of one k-quad plane: 128 hi rows + 128 lo rows
constexpr int TGM_CHUNK = (TGM_KC / 8) * TGM_PLANE;         // 16 KB per operand tile and chunk
constexpr int TGM_THREADS = 32 * 9;                         // two MMA warpgroups + one TMA producer warp

__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// multicast variant of bulk_g2s: the bytes land at the same shared-memory offset in every CTA of cta_mask, each CTA's
// mbarrier (same offset) receives the complete_tx for its own copy
__device__ __forceinline__ void bulk_g2s_mc(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar, uint16_t cta_mask) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar)), "h"(cta_mask)
                 : "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}

template <int CL>
__global__ void __launch_bounds__(TGM_THREADS, 1)
theta_gemm_tma_kernel(const float* __restrict__ Xc, const float* __restrict__ Wc, int M, int N, int KQ, int chunks_per_split,
                      int n_chunks, float* __restrict__ part) {
    constexpr int STAGE = 2 * TGM_CHUNK;                    // [A chunk of the M tile | B chunk of the N tile]
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 127) & ~(uintptr_t)127);
    __shared__ uint64_t full_bar[TGM_STAGES], empty_bar[TGM_STAGES];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ntile = blockIdx.x, split = blockIdx.y, mtile = blockIdx.z;
    const int c0 = split * chunks_per_split, c1 = min(n_chunks, c0 + chunks_per_split);
    const int nc = max(0, c1 - c0);

    pdl_trigger();                                          // common.cuh: PDL chain of the tick
    if (tid == 0) {
        for (int i = 0; i < TGM_STAGES; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8 * CL); }
        fence_mbar_init();
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();                         // every peer's barriers exist before anyone multicasts into it
    constexpr uint16_t CL_MASK = (uint16_t)((1u << CL) - 1);
    pdl_wait();                                             // Xc is written by the previous kernel (conv3 epilogue); part is read by the next

    if (warp == 8) {
        // ===== TMA producer =====
        if (lane == 0) {
            const uint8_t* xa = (const uint8_t*)Xc + (size_t)mtile * KQ * TGM_PLANE;
            const uint8_t* wb = (const uint8_t*)Wc + (size_t)ntile * KQ * TGM_PLANE;
            for (int i = 0; i < nc; ++i) {
                const int st = i % TGM_STAGES;
                mbar_wait(&empty_bar[st], ((i / TGM_STAGES) & 1) ^ 1);
                mbar_arrive_expect_tx(&full_bar[st], STAGE);
                const size_t koff = (size_t)(c0 + i) * TGM_CHUNK;
                uint8_t* dst = smem + st * STAGE;
                if (CL == 1) {
                    bulk_g2s(dst, xa + koff, TGM_CHUNK, &full_bar[st]);
                } else {
                    // this CTA's 1/CL slice of the A chunk, delivered to every CTA of the cluster
                    constexpr int SLICE = TGM_CHUNK / CL;
                    const int off = (int)cluster_ctarank() * SLICE;
                    bulk_g2s_mc(dst + off, xa + koff + off, SLICE, &full_bar[st], CL_MASK);
                }
                bulk_g2s(dst + TGM_CHUNK, wb + koff, TGM_CHUNK, &full_bar[st]);
            }
        }
    } else {
        // ===== MMA warpgroups: warpgroup w owns rows 64*w .. 64*w+63 of the M tile =====
        const int w = warp >> 2, wq = warp & 3;
        // main and correction accumulators in separate register blocks (a wgmma into a sub-block of another wgmma's
        // accumulators leaves ptxas without registers for the pipeline and serialises every wgmma)
        float acc[64], cor[64];
#pragma unroll
        for (int x = 0; x < 64; ++x) acc[x] = cor[x] = 0.0f;
        const uint32_t s0 = smem_u32(smem);
        for (int i = 0; i < nc; ++i) {
            const int st = i % TGM_STAGES;
            mbar_wait(&full_bar[st], (i / TGM_STAGES) & 1);
            wgmma_fence();
#pragma unroll
            for (int k16 = 0; k16 < TGM_KC / 16; ++k16) {
                const uint32_t sa = s0 + st * STAGE + w * 1024 + 2 * k16 * TGM_PLANE;
                const uint64_t dA = smem_desc(sa, TGM_PLANE, 128);
                const uint64_t dB = smem_desc(s0 + st * STAGE + TGM_CHUNK + 2 * k16 * TGM_PLANE, TGM_PLANE, 128);
                wgmma_f16<128>(acc, dA, dB, 1);                                        // A_h0 * B_h0 -> main
                wgmma_f16<128>(cor, dA, dB + (uint64_t)(2048 >> 4), 1);                // A_h0 * B_h1 -> correction
                wgmma_f16<128>(cor, dA + (uint64_t)(2048 >> 4), dB, 1);                // A_h1 * B_h0 -> correction
            }
            wgmma_commit();
            wgmma_wait<1>();                                // the previous chunk's wgmmas have read their stage
            __syncwarp();
            if (i > 0 && lane == 0) {
                const int ps = (i - 1) % TGM_STAGES;
                if (CL == 1) mbar_arrive(&empty_bar[ps]);
                else
                    for (int r = 0; r < CL; ++r) mbar_arrive_cluster(&empty_bar[ps], r);   // every peer's stage holds data this CTA multicast
            }
        }
        wgmma_wait<0>();
        fence_regs<64>(acc);
        fence_regs<64>(cor);
        // ===== epilogue: part[split][m][n] = main + 2^-11 * correction =====
        float* P = part + (int64_t)split * M * N;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = mtile * 128 + w * 64 + wq * 16 + (lane >> 2) + 8 * h;
            if (m >= M) continue;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int n = ntile * 128 + 8 * j + 2 * (lane & 3);        // N % 4 == 0: n < N implies n + 1 < N
                if (n < N)
                    *reinterpret_cast<float2*>(P + (int64_t)m * N + n) =
                        make_float2(fmaf(cor[4 * j + 2 * h], F16_LO_INV, acc[4 * j + 2 * h]),
                                    fmaf(cor[4 * j + 2 * h + 1], F16_LO_INV, acc[4 * j + 2 * h + 1]));
            }
        }
    }
    if (CL > 1) cluster_sync_all();                         // no CTA leaves while a peer may still arrive on its barriers
}

// W[K][N] (row-major, arbitrary element alignment) -> Wc[n tile][k octet][h0 | h1][128][8 x fp16]; columns >= N are zero
__global__ void theta_prep_kernel(const float* __restrict__ W, int K, int N, int KO, float* __restrict__ Wc) {
    const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;      // (ntile, ko, n)
    const int n_tiles = (N + 127) / 128;
    if (u >= (int64_t)n_tiles * KO * 128) return;
    const int nl = (int)(u % 128);
    const int ko = (int)((u / 128) % KO), nt = (int)(u / ((int64_t)128 * KO));
    const int n = nt * 128 + nl;
    float w[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) w[j] = (n < N && 8 * ko + j < K) ? W[(int64_t)(8 * ko + j) * N + n] : 0.0f;
    uint4 hi, lo;
    split_f16x8(w, hi, lo);
    uint4* dst = reinterpret_cast<uint4*>(Wc) + ((int64_t)nt * KO + ko) * 256 + nl;
    dst[0] = hi;
    dst[128] = lo;
}
}  // namespace

// ---- host interface (forward.cuh) ---------------------------------------------------------------------------------
size_t dne_tgm_xc_bytes(int n_slots, int K) { return (size_t)((n_slots + 127) / 128) * (K / 8) * TGM_PLANE; }
size_t dne_tgm_wc_bytes(int K, int N) { return (size_t)((N + 127) / 128) * (K / 8) * TGM_PLANE; }
bool dne_tgm_supported(int K, int N, int k_per_split) { return K % TGM_KC == 0 && N % 4 == 0 && k_per_split % TGM_KC == 0; }

int dne_launch_theta_prep(const float* W, int K, int N, float* Wc, cudaStream_t st) {
    const int KO = K / 8;
    const int64_t units = (int64_t)((N + 127) / 128) * KO * 128;
    theta_prep_kernel<<<(unsigned)((units + 255) / 256), 256, 0, st>>>(W, K, N, KO, Wc);
    DNE_LAUNCHED(1);
    return 0;
}

template <int CL>
static int launch_tgm(const float* Xc, const float* Wc, int M, int N, int KQ, int cps, int n_chunks, int n_split, int m_tiles,
                      int n_tiles, float* part, cudaStream_t st) {
    constexpr int SMEM = TGM_STAGES * 2 * TGM_CHUNK + 256;
    auto kern = theta_gemm_tma_kernel<CL>;
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_done[64] = {};
    if (dev < 64 && !attr_done[dev]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM) != cudaSuccess) return DNE_ERR_CUDA;
        attr_done[dev] = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(n_tiles, n_split, m_tiles);           // blockIdx.x = N tile (= rank in the cluster when CL > 1)
    cfg.blockDim = dim3(TGM_THREADS);
    cfg.dynamicSmemBytes = SMEM;
    cfg.stream = st;
    cudaLaunchAttribute at[2];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = CL;
    at[0].val.clusterDim.y = 1;
    at[0].val.clusterDim.z = 1;
    at[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[1].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = g_dne_pdl ? 2 : 1;
    if (cudaLaunchKernelEx(&cfg, kern, Xc, Wc, M, N, KQ, cps, n_chunks, part) != cudaSuccess) return DNE_ERR_CUDA;
    DNE_LAUNCHED(1);
    return 0;
}

int dne_launch_theta_gemm_tma(const float* Xc, const float* Wc, int M, int K, int N, int k_per_split, int n_split, float* part,
                              cudaStream_t st) {
    if (!dne_tgm_supported(K, N, k_per_split)) return DNE_ERR_UNSUP;
    const int KQ = K / 8, n_chunks = K / TGM_KC, cps = k_per_split / TGM_KC;      // KQ: k-octet planes
    const int m_tiles = (M + 127) / 128, n_tiles = (N + 127) / 128;
#define TGM_ARGS Xc, Wc, M, N, KQ, cps, n_chunks, n_split, m_tiles, n_tiles, part, st
    // cluster multicast of the A chunk (g_dne_theta_mc, dne_set_option("theta_mc", 1)): off by default (not measured faster)
    if (g_dne_theta_mc && n_tiles == 4) return launch_tgm<4>(TGM_ARGS);
    if (g_dne_theta_mc && n_tiles == 2) return launch_tgm<2>(TGM_ARGS);
    return launch_tgm<1>(TGM_ARGS);
#undef TGM_ARGS
}
