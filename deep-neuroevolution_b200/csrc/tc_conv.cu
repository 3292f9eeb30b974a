// tc_conv.cu -- the member convolutions on the Hopper tensor cores (wgmma kind tf32, accumulators in registers).
//
// Same contraction as conv_kernel in forward_kernels.cu (implicit GEMM, one member per CTA):
//   A[m][k] = im2col(input)            m = output position, k = (ky,kx,ci)      (TF SAME, NHWC)
//   B[n][k] = theta_w[k][n] + s*noise[idx+off_w+k*COUT+n]   (member weights, built by the perturb stage)
//   D[m][n] = sum_k A*B  -> +bias (+virtual BN) -> relu -> NHWC store
// fp32 parity on tensor cores: 3xTF32 -- operands are split into hi + lo TF32 parts by the staging threads (hi rounded to
// nearest, so the hardware's fp32->tf32 truncation of hi is exact; lo = x - hi is truncated by the hardware) and
// D = Ahi*Bhi + Alo*Bhi + Ahi*Blo.  B_hi and B_lo are stacked along N in one tile, so Ahi*[Bhi;Blo] is ONE MMA (N = 2*COUT)
// and Alo*Bhi a second one; uint8 inputs are staged as exact integers (no lo plane, /255 in the epilogue).
// Operands are PRODUCED into shared memory by the perturb / im2col stage (they do not exist in global memory, so
// there is nothing for TMA to fetch); the layout is the wgmma K-major no-swizzle canonical layout (wgmma.cuh).
// Warp-specialised mbarrier pipeline, no block barriers in the loop: TC_GROUPS staging groups of 128 threads (group g
// owns shared-memory stage g and the k-chunks c = g mod TC_GROUPS) + two MMA warpgroups, each owning half of the M tile's
// rows in its registers; stage hand-off full[g] (staging warps arrive) / empty[g] (MMA warps arrive once their wgmmas
// of the stage have completed).  The MMA warpgroups then run the fused epilogue from their accumulator registers.
#include "common.cuh"
#include "forward.cuh"
#include "epilogue.cuh"
#include "wgmma.cuh"

using namespace wg;

#ifndef DNE_TC_GROUPS
#define DNE_TC_GROUPS 3      // staging groups of 128 threads (one shared-memory stage each)
#endif
constexpr int TC_GROUPS = DNE_TC_GROUPS;        // staging groups of 128 threads; group g owns smem stage g and stages chunks c = g (mod TC_GROUPS)
constexpr int TC_THREADS = TC_GROUPS * 128;     // conv kernels: the staging warps ...
constexpr int TC_BLOCK = TC_THREADS + 256;      // ... + two MMA warpgroups (warp-specialised, mbarrier pipeline, no block barriers)
constexpr int TG_THREADS = 256;                 // theta GEMM / self-test

template <int CIN, int COUT, int KS, int STRIDE, int HIN, int HOUT, int PAD, bool IN_U8, int MTC, int KC>
struct TcConvCfg {
    static constexpr int M = HOUT * HOUT;
    static constexpr int K = KS * KS * CIN;
    static constexpr int ROWS = MTC * 128;                       // A rows staged per CTA
    static constexpr int NCHUNK = K / KC;
    static constexpr int A_PLANE = ROWS * 16;                    // bytes per k-quad plane of A (= LBO of A)
    // B tile = [B_hi ; B_lo] stacked along N (2*COUT rows per k-quad plane): ONE MMA with N = 2*COUT computes
    // A_hi*B_hi (accumulator columns 0..COUT-1) and A_hi*B_lo (columns COUT..2*COUT-1) while reading A_hi once; the
    // A_lo*B_hi term is a second MMA over the first COUT rows of the same tile.  2 MMAs / 14 KB of operand reads per
    // k-step instead of 3 / 18 KB (the kernel is shared-memory-bandwidth bound); the two halves are summed in the epilogue.
    static constexpr int B_PLANE = 2 * COUT * 16;                // bytes per k-quad plane of B (= LBO of B)
    static constexpr int A_BYTES = (KC / 4) * A_PLANE;           // one of {hi, lo}
    static constexpr int B_BYTES = (KC / 4) * B_PLANE;           // hi and lo together
    // uint8 frames are staged as their integer value 0..255 -- exact in TF32, so A needs no lo plane (and one MMA less per
    // k-step); the /255 of atari_wrappers.py:186 is applied to the accumulator in the epilogue
    static constexpr int A_PLANES = IN_U8 ? 1 : 2;
    static constexpr int STAGE_BYTES = A_PLANES * A_BYTES + B_BYTES;
    static constexpr int NST = TC_GROUPS;                        // one shared-memory stage per staging group
    static constexpr int SMEM_BYTES = NST * STAGE_BYTES + 128;   // + alignment slack
    static constexpr int ACC = COUT / 2;                          // accumulator floats per thread and m64 tile, per accumulator
    static constexpr int PASSES = ROWS / 32;                     // A rows per staging thread and chunk
    static constexpr int B_UNITS = COUT * (KC / 4);
    static constexpr int B_PER_THREAD = (B_UNITS + 127) / 128;
    static_assert(KC == 16, "the lane -> (row, k-quad) staging map assumes 4 k-quads per chunk");
    static_assert(K % KC == 0 && CIN % 4 == 0 && COUT % 16 == 0 && KS <= 8, "tile constraints");
    static_assert(CIN == 4 || CIN % KC == 0, "a chunk is either 4 taps of 4 channels or part of one tap");
};

// Round-to-nearest TF32 hi part + fp32 remainder (the tensor core reads only the TF32 bits of lo): 3 instructions.
__device__ __forceinline__ void split_tf32_rn(float x, float& hi, float& lo) {
    hi = __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
    lo = x - hi;
}

template <int CIN, int COUT, int KS, int STRIDE, int HIN, int HOUT, int PAD, bool IN_U8, int MTC, int KC>
__global__ void __launch_bounds__(TC_BLOCK, 1)
conv_tc_kernel(SlotArgs sa, int64_t off_w, LayerEpi epi, const void* __restrict__ in_base, int64_t in_slot_stride,
               int64_t in_img_stride, float* __restrict__ out_base, int64_t out_slot_stride, int64_t out_img_stride) {
    using Cfg = TcConvCfg<CIN, COUT, KS, STRIDE, HIN, HOUT, PAD, IN_U8, MTC, KC>;
    const int slot = blockIdx.y;
    if (!slot_active(sa, slot)) return;
    const int img = blockIdx.z;
    const int row0 = blockIdx.x * Cfg::ROWS;                     // first output position of this CTA
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    constexpr int NST = Cfg::NST;
    constexpr int STAGE_WARPS = TC_THREADS / 32;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 127) & ~(uintptr_t)127);
    __shared__ uint64_t full_bar[NST], empty_bar[NST];
    __shared__ ChanEpi epi_s[COUT];                              // per-channel epilogue parameters, built once per CTA

    const float* th = slot_theta(sa, slot);
    const int64_t idx = sa.noise_idx[slot];
    const float s = sa.scale[slot];

    if (tid == 0) {
        for (int i = 0; i < NST; ++i) {
            mbar_init(&full_bar[i], 4);                          // one arrival per warp of the owning staging group
            mbar_init(&empty_bar[i], 8);                         // one arrival per MMA warp
        }
        fence_mbar_init();
    }
    if (tid < COUT) epi_s[tid] = make_chan_epi(sa, epi, slot, COUT, tid, th, idx, s);
    __syncthreads();

    if (warp >= STAGE_WARPS) {
        // ============ MMA warpgroups: warpgroup w owns the m64 tiles w*MTC .. w*MTC+MTC-1 of the CTA's rows ============
        const int w = (warp - STAGE_WARPS) >> 2, wq = warp & 3;
        const uint32_t s0 = smem_u32(smem);
        // A_hi*B_hi and the two cross terms in separate register blocks (a wgmma into a sub-block of another wgmma's
        // accumulators leaves ptxas without registers for the pipeline and serialises every wgmma)
        float acc[MTC][Cfg::ACC], cor[MTC][Cfg::ACC];
#pragma unroll
        for (int j = 0; j < MTC; ++j)
#pragma unroll
            for (int x = 0; x < Cfg::ACC; ++x) acc[j][x] = cor[j][x] = 0.0f;
        for (int c = 0; c < Cfg::NCHUNK; ++c) {
            const int st = c % NST;
            mbar_wait(&full_bar[st], (c / NST) & 1);             // the staging group has filled (and fenced) this stage
            const uint32_t sa0 = s0 + st * Cfg::STAGE_BYTES, sb0 = sa0 + Cfg::A_PLANES * Cfg::A_BYTES;
            wgmma_fence();
#pragma unroll
            for (int k8 = 0; k8 < KC / 8; ++k8) {
                const uint64_t dB = smem_desc(sb0 + 2 * k8 * Cfg::B_PLANE, Cfg::B_PLANE, 128);
#pragma unroll
                for (int j = 0; j < MTC; ++j) {
                    const uint64_t dAh = smem_desc(sa0 + 2 * k8 * Cfg::A_PLANE + (w * MTC + j) * 1024, Cfg::A_PLANE, 128);
                    wgmma_tf32<COUT>(acc[j], dAh, dB, 1);                                                      // A_hi * B_hi
                    wgmma_tf32<COUT>(cor[j], dAh, dB + (uint64_t)((COUT * 16) >> 4), 1);                       // A_hi * B_lo
                    if (!IN_U8) wgmma_tf32<COUT>(cor[j], dAh + (uint64_t)(Cfg::A_BYTES >> 4), dB, 1);          // A_lo * B_hi
                }
            }
            wgmma_commit();
            wgmma_wait<1>();                                     // the previous chunk's MMAs have read their stage
            __syncwarp();
            if (c > 0 && lane == 0) mbar_arrive(&empty_bar[(c - 1) % NST]);
        }
        wgmma_wait<0>();
#pragma unroll
        for (int j = 0; j < MTC; ++j) {
            fence_regs<Cfg::ACC>(acc[j]);
            fence_regs<Cfg::ACC>(cor[j]);
        }
        // ---- epilogue: registers -> (/255) + bias (+BN) + activation -> NHWC global ----
        float* out = out_base + slot * out_slot_stride + img * out_img_stride;
        constexpr float IN_SCALE = IN_U8 ? (1.0f / 255.0f) : 1.0f;
#pragma unroll
        for (int j = 0; j < MTC; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int m = row0 + (w * MTC + j) * 64 + wq * 16 + (lane >> 2) + 8 * h;
                if (m < Cfg::M) {
#pragma unroll
                    for (int i = 0; i < COUT / 8; ++i) {
                        const int n = 8 * i + 2 * (lane & 3);
                        float v0 = acc[j][4 * i + 2 * h] + cor[j][4 * i + 2 * h];
                        float v1 = acc[j][4 * i + 2 * h + 1] + cor[j][4 * i + 2 * h + 1];
                        if (IN_U8) { v0 *= IN_SCALE; v1 *= IN_SCALE; }
                        *reinterpret_cast<float2*>(out + (int64_t)m * COUT + n) = make_float2(epi_s[n].apply(v0), epi_s[n + 1].apply(v1));
                    }
                }
            }
    } else {
        // ============== staging groups: perturb + im2col -> shared memory (group g <-> stage g) ==============
        const int g = warp >> 2, wg = warp & 3, tg = tid & 127;
        const float* nz = sa.noise + idx + off_w;
        const float* tw = th + off_w;
        const uint8_t* in_u8 = nullptr;
        const float* in_f = nullptr;
        if (IN_U8) in_u8 = (const uint8_t*)in_base + slot * in_slot_stride + img * in_img_stride;
        else in_f = (const float*)in_base + slot * in_slot_stride + img * in_img_stride;

        // A: in every chunk this thread stages k-quad q of the rows i*32 + wg*8 + (lane & 7); a quarter warp covers 8
        // consecutive rows of one quad plane (128 contiguous shared-memory bytes: conflict-free 16-byte stores) and the
        // 4 quads of one row are 4 lanes reading 64 contiguous bytes (float) / 16 bytes (uint8) of the input
        constexpr int PASSES = Cfg::PASSES;
        const int q = lane >> 3;
        int a_off[PASSES];               // input element offset of the row's (ky = 0, kx = 0, ci = 0) corner
        uint32_t a_vm[PASSES];           // validity: bit ky -> row iy0+ky inside the image, bit 8+kx -> column ix0+kx inside
#pragma unroll
        for (int i = 0; i < PASSES; ++i) {
            const int m = row0 + i * 32 + wg * 8 + (lane & 7);
            const int mc = min(m, Cfg::M - 1);
            const int oy = mc / HOUT, ox = mc - oy * HOUT;
            const int iy0 = oy * STRIDE - PAD, ix0 = ox * STRIDE - PAD;
            a_off[i] = (iy0 * HIN + ix0) * CIN;
            const int ylo = max(0, -iy0), yhi = min(KS, HIN - iy0), xlo = max(0, -ix0), xhi = min(KS, HIN - ix0);
            const uint32_t my = (1u << yhi) - (1u << ylo), mx = (1u << xhi) - (1u << xlo);
            a_vm[i] = (m < Cfg::M) ? (my | (mx << 8)) : 0u;
        }
        // B: unit u = tg + i*128 -> (column n = u % COUT, k-quad u / COUT); element offset of its first k row
        constexpr int BPT = Cfg::B_PER_THREAD;
        // (128 % COUT == 0: unit i of a thread is the same column n, k-quad q0 + i*(128/COUT))
        static_assert(128 % COUT == 0, "B unit map");
        const int b_off0 = 4 * (tg / COUT) * COUT + (tg % COUT);             // global element offset of unit 0's first k row
        const int b_st0 = (tg / COUT) * Cfg::B_PLANE + (tg % COUT) * 16;     // byte offset of unit 0's hi quad in the B tile
        constexpr int B_OFF_STEP = 4 * 128, B_ST_STEP = (128 / COUT) * Cfg::B_PLANE;
        const uint32_t sA_hi = smem_u32(smem) + g * Cfg::STAGE_BYTES + q * Cfg::A_PLANE + (wg * 8 + (lane & 7)) * 16;   // + i*512 per pass
        const uint32_t sA_lo = sA_hi + Cfg::A_BYTES;
        const uint32_t sB = smem_u32(smem) + g * Cfg::STAGE_BYTES + Cfg::A_PLANES * Cfg::A_BYTES;

        for (int c = g, it = 0; c < Cfg::NCHUNK; c += TC_GROUPS, ++it) {
            // ---- raw global loads of the chunk (issued before the stage wait so that their latency overlaps it) ----
            const int k = c * KC + 4 * q;
            const int ci = k % CIN, t = k / CIN;
            const int ky = t / KS, kx = t - ky * KS;
            const int tap = (ky * HIN + kx) * CIN + ci;
            const uint32_t vbit = (1u << ky) | (1u << (8 + kx));
            uint32_t rawA_u8[IN_U8 ? PASSES : 1];
            float4 rawA_f[IN_U8 ? 1 : PASSES];
#pragma unroll
            for (int i = 0; i < PASSES; ++i) {
                const bool ok = (a_vm[i] & vbit) == vbit;
                if (IN_U8) rawA_u8[IN_U8 ? i : 0] = ok ? *reinterpret_cast<const uint32_t*>(in_u8 + a_off[i] + tap) : 0u;
                else rawA_f[IN_U8 ? 0 : i] = ok ? *reinterpret_cast<const float4*>(in_f + a_off[i] + tap) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
            float rawB_t[BPT][4], rawB_n[BPT][4];
            const int64_t fb = (int64_t)c * KC * COUT;
#pragma unroll
            for (int i = 0; i < BPT; ++i) {
                if (tg + i * 128 < Cfg::B_UNITS) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        rawB_t[i][j] = tw[fb + b_off0 + i * B_OFF_STEP + j * COUT];
                        rawB_n[i][j] = nz[fb + b_off0 + i * B_OFF_STEP + j * COUT];
                    }
                }
            }
            mbar_wait(&empty_bar[g], (it & 1) ^ 1);              // the MMAs of this group's previous chunk have drained the stage
            // ---- convert + store: A ----
#pragma unroll
            for (int i = 0; i < PASSES; ++i) {
                if (IN_U8) {
                    const uint32_t px = rawA_u8[IN_U8 ? i : 0];
                    sts128(sA_hi + i * 512, make_float4((float)(px & 255u), (float)((px >> 8) & 255u), (float)((px >> 16) & 255u),
                                                        (float)(px >> 24)));
                } else {
                    const float4 v = rawA_f[IN_U8 ? 0 : i];
                    float4 hi, lo;
                    split_tf32_rn(v.x, hi.x, lo.x);
                    split_tf32_rn(v.y, hi.y, lo.y);
                    split_tf32_rn(v.z, hi.z, lo.z);
                    split_tf32_rn(v.w, hi.w, lo.w);
                    sts128(sA_hi + i * 512, hi);
                    sts128(sA_lo + i * 512, lo);
                }
            }
            // ---- perturb + convert + store: B ----
#pragma unroll
            for (int i = 0; i < BPT; ++i) {
                const int u = tg + i * 128;
                if (u < Cfg::B_UNITS) {
                    float4 hi, lo;
                    split_tf32_rn(perturbed(rawB_t[i][0], s, rawB_n[i][0]), hi.x, lo.x);
                    split_tf32_rn(perturbed(rawB_t[i][1], s, rawB_n[i][1]), hi.y, lo.y);
                    split_tf32_rn(perturbed(rawB_t[i][2], s, rawB_n[i][2]), hi.z, lo.z);
                    split_tf32_rn(perturbed(rawB_t[i][3], s, rawB_n[i][3]), hi.w, lo.w);
                    sts128(sB + b_st0 + i * B_ST_STEP, hi);
                    sts128(sB + b_st0 + i * B_ST_STEP + COUT * 16, lo);
                }
            }
            fence_proxy_async_smem();                            // generic-proxy writes -> async proxy
            __syncwarp();
            if (lane == 0) mbar_arrive(&full_bar[g]);
        }
    }
}

// =====================================================================================================
template <int CIN, int COUT, int KS, int STRIDE, int HIN, int HOUT, int PAD, bool IN_U8, int MTC, int KC>
static int launch_conv_tc(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, const void* in,
                          int64_t in_slot_stride, int64_t in_img_stride, float* out, int64_t out_slot_stride,
                          int64_t out_img_stride, int n_slots, int n_img, cudaStream_t st) {
    using Cfg = TcConvCfg<CIN, COUT, KS, STRIDE, HIN, HOUT, PAD, IN_U8, MTC, KC>;
    auto kern = conv_tc_kernel<CIN, COUT, KS, STRIDE, HIN, HOUT, PAD, IN_U8, MTC, KC>;
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_done_dev[64] = {};                           // per device
    bool& attr_done = attr_done_dev[dev < 64 ? dev : 63];
    if (!attr_done) {
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES) != cudaSuccess)
            return DNE_ERR_CUDA;
        attr_done = true;
    }
    dim3 grid((Cfg::M + Cfg::ROWS - 1) / Cfg::ROWS, n_slots, n_img);
    kern<<<grid, TC_BLOCK, Cfg::SMEM_BYTES, st>>>(sa, L.off_w, epi, in, in_slot_stride, in_img_stride, out,
                                                   out_slot_stride, out_img_stride);
    DNE_LAUNCHED(1);
    return 0;
}

static bool tconv_is(const dne_layer_desc& L, int cin, int cout, int ks, int stride, int hin, int hout, int pad) {
    return L.cin == cin && L.cout == cout && L.ksize == ks && L.stride == stride && L.hin == hin &&
           L.hout == hout && L.pad == pad;
}

int dne_launch_conv_layer_tc(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, bool in_u8,
                             const void* in, int64_t in_slot_stride, int64_t in_img_stride, float* out,
                             int64_t out_slot_stride, int64_t out_img_stride, int n_slots, int n_img,
                             cudaStream_t st) {
#define ARGS sa, L, epi, in, in_slot_stride, in_img_stride, out, out_slot_stride, out_img_stride, n_slots, n_img, st
    if (in_u8 && tconv_is(L, 4, 32, 8, 4, 84, 21, 2)) return launch_conv_tc<4, 32, 8, 4, 84, 21, 2, true, 2, 16>(ARGS);
    if (in_u8 && tconv_is(L, 4, 16, 8, 4, 84, 21, 2)) return launch_conv_tc<4, 16, 8, 4, 84, 21, 2, true, 2, 16>(ARGS);
    if (!in_u8 && tconv_is(L, 32, 64, 4, 2, 21, 11, 1)) return launch_conv_tc<32, 64, 4, 2, 21, 11, 1, false, 1, 16>(ARGS);
    if (!in_u8 && tconv_is(L, 16, 32, 4, 2, 21, 11, 1)) return launch_conv_tc<16, 32, 4, 2, 21, 11, 1, false, 1, 16>(ARGS);
    if (!in_u8 && tconv_is(L, 64, 64, 3, 1, 11, 11, 1)) return launch_conv_tc<64, 64, 3, 1, 11, 11, 1, false, 1, 16>(ARGS);
#undef ARGS
    return DNE_ERR_UNSUP;
}

// =====================================================================================================
// Dense layer, shared-theta part on the tensor cores:  part[split][m][n] = sum_{k in split} X[m][k] * W[k][n]
// (same contract as dense_theta_gemm_kernel).  CTA tile 128 x 128, k-chunks of 16, 3xTF32, operands staged by the
// threads (A rows are K-contiguous float4 loads; B is transposed to [n][k] quads on the fly), three smem stages.  The
// two warpgroups stage together and each issues the wgmmas of one m64 half of the tile: a stage is rewritten three
// chunks after it was read, by which time every warpgroup has waited for those wgmmas (wgmma_wait<1>) and passed a
// block barrier since -- one __syncthreads per chunk.
// =====================================================================================================
constexpr int TG_BM = 128, TG_BN = 128, TG_KC = 16, TG_NST = 3;
constexpr int TG_A_PLANE = TG_BM * 16, TG_B_PLANE = TG_BN * 16;
constexpr int TG_A_BYTES = (TG_KC / 4) * TG_A_PLANE, TG_B_BYTES = (TG_KC / 4) * TG_B_PLANE;
constexpr int TG_STAGE_BYTES = 2 * TG_A_BYTES + 2 * TG_B_BYTES;
constexpr int TG_SMEM_BYTES = TG_NST * TG_STAGE_BYTES + 128;

// stage chunk (rawA, rawB) into stage st, split hi / lo
__device__ __forceinline__ void tg_stage(uint32_t s0, int st, int tid, const float4 (&rawA)[2], const float (&rawB)[2][4]) {
    const uint32_t sA_hi = s0 + st * TG_STAGE_BYTES, sA_lo = sA_hi + TG_A_BYTES, sB_hi = sA_lo + TG_A_BYTES, sB_lo = sB_hi + TG_B_BYTES;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int u = tid + i * TG_THREADS;
        float4 hi, lo;
        split_tf32_fast(rawA[i].x, hi.x, lo.x);
        split_tf32_fast(rawA[i].y, hi.y, lo.y);
        split_tf32_fast(rawA[i].z, hi.z, lo.z);
        split_tf32_fast(rawA[i].w, hi.w, lo.w);
        sts128(sA_hi + u * 16, hi);                              // (u / TG_BM) * TG_A_PLANE + (u % TG_BM) * 16 == u * 16
        sts128(sA_lo + u * 16, lo);
        split_tf32_fast(rawB[i][0], hi.x, lo.x);
        split_tf32_fast(rawB[i][1], hi.y, lo.y);
        split_tf32_fast(rawB[i][2], hi.z, lo.z);
        split_tf32_fast(rawB[i][3], hi.w, lo.w);
        sts128(sB_hi + u * 16, hi);
        sts128(sB_lo + u * 16, lo);
    }
}
// this warpgroup's m64 half of the 128 x 128 tile: A_hi*B_hi + A_lo*B_hi + A_hi*B_lo over one chunk
__device__ __forceinline__ void tg_mma(uint32_t s0, int st, int half, float (&acc)[64], bool overwrite) {
    const uint32_t sA = s0 + st * TG_STAGE_BYTES + half * 1024, sB = s0 + st * TG_STAGE_BYTES + 2 * TG_A_BYTES;
    wgmma_fence();
#pragma unroll
    for (int k8 = 0; k8 < TG_KC / 8; ++k8) {
        const uint64_t dAh = smem_desc(sA + 2 * k8 * TG_A_PLANE, TG_A_PLANE, 128), dBh = smem_desc(sB + 2 * k8 * TG_B_PLANE, TG_B_PLANE, 128);
        wgmma_tf32<128>(acc, dAh, dBh, !(overwrite && k8 == 0));
        wgmma_tf32<128>(acc, dAh + (uint64_t)(TG_A_BYTES >> 4), dBh, 1);
        wgmma_tf32<128>(acc, dAh, dBh + (uint64_t)(TG_B_BYTES >> 4), 1);
    }
    wgmma_commit();
}

__global__ void __launch_bounds__(TG_THREADS, 1)
theta_gemm_tc_kernel(const float* __restrict__ X, int M, int K, int N, const float* __restrict__ W, int k_per_split,
                     float* __restrict__ part) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 127) & ~(uintptr_t)127);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int half = warp >> 2, wq = warp & 3;
    const int m0 = blockIdx.y * TG_BM, n0 = blockIdx.x * TG_BN, split = blockIdx.z;
    const int kbeg = split * k_per_split, kend = min(K, kbeg + k_per_split);
    const int nchunk = (kend - kbeg + TG_KC - 1) / TG_KC;
    const uint32_t s0 = smem_u32(smem);

    // A: 128 rows x 4 k-quads = 512 units; B: 128 n x 4 k-quads = 512 units -> 2 + 2 units per thread
    float4 rawA[2];
    float rawB[2][4];
    auto load_chunk = [&](int c) {
        const int k0 = kbeg + c * TG_KC;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int u = tid + i * TG_THREADS;
            const int r = u % TG_BM, q = u / TG_BM;
            const int m = m0 + r, k = k0 + 4 * q;
            rawA[i] = (m < M && k < kend) ? *reinterpret_cast<const float4*>(X + (int64_t)m * K + k)
                                          : make_float4(0.f, 0.f, 0.f, 0.f);
            const int n = n0 + (u % TG_BN), kb = k0 + 4 * (u / TG_BN);
#pragma unroll
            for (int j = 0; j < 4; ++j) rawB[i][j] = (n < N && kb + j < kend) ? W[(int64_t)(kb + j) * N + n] : 0.0f;
        }
    };
    float acc[64];
#pragma unroll
    for (int x = 0; x < 64; ++x) acc[x] = 0.0f;
    if (nchunk > 0) load_chunk(0);
    for (int c = 0; c < nchunk; ++c) {
        const int st = c % TG_NST;
        tg_stage(s0, st, tid, rawA, rawB);
        if (c + 1 < nchunk) load_chunk(c + 1);
        fence_proxy_async_smem();
        __syncthreads();
        tg_mma(s0, st, half, acc, false);                    // acc starts at zero: no non-wgmma write inside the pipeline
        wgmma_wait<1>();
    }
    wgmma_wait<0>();
    fence_regs<64>(acc);
    float* P = part + (int64_t)split * M * N;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int m = m0 + half * 64 + wq * 16 + (lane >> 2) + 8 * h;
        if (m < M) {
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int n = n0 + 8 * j + 2 * (lane & 3);         // N % 4 == 0: n < N implies n + 1 < N
                if (n < N) *reinterpret_cast<float2*>(P + (int64_t)m * N + n) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
            }
        }
    }
}

// returns 0 on launch, DNE_ERR_UNSUP if the shape is not covered (caller falls back to the SIMT GEMM)
int dne_launch_theta_gemm_tc(const float* X, int M, int K, int N, const float* W, int k_per_split, int n_split,
                             float* part, cudaStream_t st) {
    if (K % 4 != 0 || N % 4 != 0 || k_per_split % TG_KC != 0) return DNE_ERR_UNSUP;
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_done_dev[64] = {};
    bool& attr_done = attr_done_dev[dev < 64 ? dev : 63];
    if (!attr_done) {
        cudaFuncSetAttribute(theta_gemm_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (cudaFuncSetAttribute(theta_gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TG_SMEM_BYTES) != cudaSuccess)
            return DNE_ERR_CUDA;
        attr_done = true;
    }
    dim3 grid((N + TG_BN - 1) / TG_BN, (M + TG_BM - 1) / TG_BM, n_split);
    theta_gemm_tc_kernel<<<grid, TG_THREADS, TG_SMEM_BYTES, st>>>(X, M, K, N, W, k_per_split, part);
    return 0;
}

// =====================================================================================================
// Per-member dense layer of the virtual-batch-norm reference pass on the tensor cores (policies.py:322-328,399; the fc
// of ESAtariPolicy / ModelVirtualBN): out[slot][m][n] = sum_k X[slot][m][k] * fl(theta_w + fl(s*noise))[k][n] + bias_n
// for the M = n_ref reference rows of every member.  Same tile engine as theta_gemm_tc_kernel (CTA tile 128 x 128,
// 3xTF32, thread-staged operands, three smem stages) with blockIdx.z = member: the B operand is the member's PERTURBED
// weight matrix, formed from the theta rows and the member's noise rows while staging; the whole K range in one CTA.
// =====================================================================================================
__global__ void __launch_bounds__(TG_THREADS, 1)
member_gemm_tc_kernel(SlotArgs sa, int64_t off_w, int64_t off_b, const float* __restrict__ X, int64_t x_slot_stride, int M,
                      int K, int N, float* __restrict__ out, int64_t out_slot_stride) {
    const int slot = blockIdx.z;
    if (!slot_active(sa, slot)) return;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 127) & ~(uintptr_t)127);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int half = warp >> 2, wq = warp & 3;
    const int m0 = blockIdx.y * TG_BM, n0 = blockIdx.x * TG_BN;
    const int nchunk = (K + TG_KC - 1) / TG_KC;
    const float* th = slot_theta(sa, slot);
    const int64_t idx = sa.noise_idx[slot];
    const float s = sa.scale[slot];
    const float* tw = th + off_w;
    const float* nz = sa.noise + idx + off_w;
    const float* x = X + (int64_t)slot * x_slot_stride;
    const uint32_t s0 = smem_u32(smem);

    constexpr int MG_DRAIN = 16;
    float acc[64], accr[64];
#pragma unroll
    for (int xx = 0; xx < 64; ++xx) accr[xx] = 0.0f;
    float4 rawA[2];
    float rawB[2][4];
    auto load_chunk = [&](int c) {
        const int k0 = c * TG_KC;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int u = tid + i * TG_THREADS;
            const int r = u % TG_BM, q = u / TG_BM;
            const int m = m0 + r, k = k0 + 4 * q;
            rawA[i] = (m < M && k < K) ? *reinterpret_cast<const float4*>(x + (int64_t)m * K + k) : make_float4(0.f, 0.f, 0.f, 0.f);
            const int n = n0 + (u % TG_BN), kb = k0 + 4 * (u / TG_BN);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int64_t f = (int64_t)(kb + j) * N + n;
                rawB[i][j] = (n < N && kb + j < K) ? perturbed(tw[f], s, nz[f]) : 0.0f;
            }
        }
    };
    load_chunk(0);
    for (int c = 0; c < nchunk; ++c) {
        const int st = c % TG_NST;
        tg_stage(s0, st, tid, rawA, rawB);
        if (c + 1 < nchunk) load_chunk(c + 1);
        fence_proxy_async_smem();
        __syncthreads();
        tg_mma(s0, st, half, acc, (c % MG_DRAIN) == 0);
        if ((c % MG_DRAIN) == MG_DRAIN - 1 || c == nchunk - 1) {
            // fold the tensor-core accumulator into fp32 registers every MG_DRAIN chunks (K = 256): the tensor core's
            // accumulator add is not round-to-nearest, and over K = 3872 its bias reached 4e-5 (VBN statistics are compared
            // at 2e-5)
            wgmma_wait<0>();
            fence_regs<64>(acc);
#pragma unroll
            for (int xx = 0; xx < 64; ++xx) accr[xx] += acc[xx];
        } else {
            wgmma_wait<1>();
        }
    }
    float* o = out + (int64_t)slot * out_slot_stride;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const int n = n0 + 8 * j + 2 * (lane & 3);               // N % 4 == 0: n < N implies n + 1 < N
        if (n >= N) continue;
        const float b0 = off_b >= 0 ? perturbed(th[off_b + n], s, sa.noise[idx + off_b + n]) : 0.0f;
        const float b1 = off_b >= 0 ? perturbed(th[off_b + n + 1], s, sa.noise[idx + off_b + n + 1]) : 0.0f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + half * 64 + wq * 16 + (lane >> 2) + 8 * h;
            if (m < M) *reinterpret_cast<float2*>(o + (int64_t)m * N + n) = make_float2(accr[4 * j + 2 * h] + b0, accr[4 * j + 2 * h + 1] + b1);
        }
    }
}

// returns 0 on launch, DNE_ERR_UNSUP if the shape is not covered (caller falls back to the SIMT member GEMM)
int dne_launch_member_gemm_tc(const SlotArgs& sa, int64_t off_w, int64_t off_b, const float* X, int64_t x_slot_stride, int M,
                              int K, int N, float* out, int64_t out_slot_stride, int n_slots, cudaStream_t st) {
    if (K % 4 != 0 || N % 4 != 0 || K < TG_KC || (x_slot_stride & 3) || (out_slot_stride & 3) || (((uintptr_t)X | (uintptr_t)out) & 15))
        return DNE_ERR_UNSUP;
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_done_dev[64] = {};
    bool& attr_done = attr_done_dev[dev < 64 ? dev : 63];
    if (!attr_done) {
        cudaFuncSetAttribute(member_gemm_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if (cudaFuncSetAttribute(member_gemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, TG_SMEM_BYTES) != cudaSuccess)
            return DNE_ERR_CUDA;
        attr_done = true;
    }
    dim3 grid((N + TG_BN - 1) / TG_BN, (M + TG_BM - 1) / TG_BM, n_slots);
    member_gemm_tc_kernel<<<grid, TG_THREADS, TG_SMEM_BYTES, st>>>(sa, off_w, off_b, X, x_slot_stride, M, K, N, out, out_slot_stride);
    return 0;
}
