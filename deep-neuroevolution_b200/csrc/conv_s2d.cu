// conv_s2d.cu -- the member convolutions as shifted-window implicit GEMMs on the Hopper tensor cores (wgmma, accumulators
// in the registers of two MMA warpgroups), A operand fed by TMA, persistent warp-specialised CTAs.  Replaces
// conv_tc_kernel (tc_conv.cu) on the per-tick path.
//
// Same contraction as the reference's per-member conv2d (policies.py:321-327,451-453; models/dqn.py:41-45,
// models/base.py:54-75: extract_image_patches + batched matmul; TF 'SAME', NHWC, HWIO):
//   out[m][n] = act( sum_{ky,kx,ci} in[oy*S-P+ky][ox*S-P+kx][ci] * w[ky][kx][ci][n] + b[n] ),   w = theta + s*noise[idx:]
//
// What differs from conv_tc_kernel:
//   * NO im2col copy.  The (zero padded) input is space-to-depth'ed by the stride S, which turns the KSxKS/stride-S
//     convolution into a (KS/S)x(KS/S)/stride-1 convolution over a W x W pixel grid with S*S*CIN channels.  The image
//     is kept in shared memory as channel-octet planes  img[plane][pixel][8 x fp16]  -- which IS the wgmma K-major
//     no-swizzle canonical layout of a matrix whose rows are the pixels (8 pixels = one 128-byte core matrix, SBO = 128,
//     next channel octet LBO = PIXP*16 bytes; a 16-byte row holds 8 fp16 channels).  Output position m = oy*W + ox reads
//     pixel m + ty*W + tx for tap (ty, tx): the SAME image at a start address shifted by (ty*W+tx)*16 bytes.  One smem
//     descriptor per (tap, channel octet, m64 tile); rows with ox >= HOUT are junk accumulator rows that the epilogue
//     skips (dev/tc_window.cu is the hardware self-test of this addressing; tests/test_gpu_tc.py::test_tcgen05_shifted_window_operand).
//     Staging traffic per member drops from KS*KS/(S*S) x the input (conv3: 9x) to 1x.
//   * for every layer but the first the image is not staged by threads at all: the PRODUCING layer's epilogue writes the
//     next layer's image (already space-to-depth'ed, zero padded, split into fp16 hi / lo planes) to global memory in
//     exactly the shared-memory layout, and a producer thread brings it in with cp.async.bulk (TMA), one channel-octet
//     group per mbarrier, so the MMAs of member i overlap the loads of member i+1 (a group's buffer is released by the
//     MMA warps once their wgmmas reading it have completed).  The first layer converts the uint8 frame (exact in fp16:
//     one plane, /255 applied to the accumulator).
//   * the member's raw weights are not fetched by the staging threads either: a second producer thread streams the
//     chunk's theta rows and noise rows (16-byte aligned supersets of the arbitrarily aligned slices) with cp.async.bulk
//     into the ring stage that will hold the operand tile, NSTB chunks deep; converter warps read the raw rows from shared
//     memory, perturb + split, and overwrite the SAME stage with the canonical [B_hi ; B_lo] tile.
//   * persistent CTAs (one per SM), warpgroup-specialised: two MMA warpgroups (each owns every other m64 tile of the
//     member's rows and runs the fused epilogue through a shared-memory staging tile), one converter warpgroup, and a
//     producer warpgroup (image TMA warp + weight TMA warp).  setmaxnreg moves registers from the converter / producer
//     warpgroups to the MMA warpgroups, whose accumulators take 128 registers per thread.  A groups (TMA or converters <-> MMA) and the B ring
//     (converters <-> MMA) run ahead of the MMA warpgroups, so staging of member i+1 overlaps the MMAs and epilogue of i.
//   * arithmetic: wgmma kind f16 on 2 x fp16 splits (wgmma.cuh: x = h0 + h1*2^-11, 22 significand bits; uint8 pixels
//     are exact in fp16 and need one plane) -- twice the MAC rate and half the operand bytes of a 3xTF32 formulation:
//     main accumulator D0 = A_h0*B_h0, correction accumulator D1 = A_h0*B_h1 + A_h1*B_h0 (B_h0 and B_h1 stacked along N:
//     one N = 2*COUT MMA + one N = COUT MMA per K = 16 step), result = D0 + 2^-11 * D1.  fp16 x fp16 products are exact
//     in the fp32 accumulators.
#include "common.cuh"
#include "forward.cuh"
#include "epilogue.cuh"
#include "wgmma.cuh"

using namespace wg;

namespace {

// warpgroup roles: 0-1 MMA + epilogue, 2 converters (B tiles; first layer: also the uint8 frame), 3 producers (warp 12:
// image / frame TMA, warp 13: weight TMA; warps 14-15 idle)
constexpr int S2D_MMA_THREADS = 256;
constexpr int S2D_CONV_WARPS = 4;
constexpr int S2D_CONV_THREADS = S2D_CONV_WARPS * 32;
constexpr int S2D_THREADS = 512;
constexpr int S2D_REGS_MMA = 176, S2D_REGS_AUX = 80;        // setmaxnreg split: 2 * 176 + 2 * 80 = 512 = 65536 / 128
constexpr int S2D_FRAME_BYTES = 84 * 84 * 4;                            // the uint8 frame stack of the first layer
constexpr int S2D_FRAME_STRIDE = (S2D_FRAME_BYTES + 127) / 128 * 128;
constexpr int S2D_MAX_GROUPS = 8;
constexpr int S2D_MAX_BST = 8;       // ring depth: a stage cycles through TMA latency -> conversion -> MMA, ~4.6K cycles (conv3): 4 stages were the limit
constexpr int S2D_SMEM_BUDGET = 222 * 1024;                 // + static shared memory <= 227 KB

constexpr int cmin(int a, int b) { return a < b ? a : b; }
constexpr int cmax(int a, int b) { return a > b ? a : b; }

// Geometry of one layer's space-to-depth image (shared by the consumer kernel, the producing epilogue and the host).
struct S2dGeom {
    int S, PADB, W, KT, CIN, CP, NG, NPIX, PIXP, PARTS, LBO, GROUP_BYTES, IMG_BYTES, HIN;
};
__host__ __device__ constexpr S2dGeom s2d_geom(int CIN, int KS, int S, int HIN, int HOUT, int PAD, bool in_u8) {
    S2dGeom g{};
    const int HP = (HOUT - 1) * S + KS;
    // plane = 8 channels (one 16-byte fp16 row per pixel); group = 16 channels = one K = 16 MMA step = 2 planes per part
    g.S = S; g.PADB = PAD; g.W = HP / S; g.KT = KS / S; g.CIN = CIN; g.CP = S * S * CIN; g.NG = g.CP / 16;
    g.NPIX = g.W * g.W; g.PIXP = (g.NPIX + 7) / 8 * 8; g.PARTS = in_u8 ? 1 : 2; g.LBO = g.PIXP * 16;
    g.GROUP_BYTES = g.PARTS * 2 * g.LBO; g.IMG_BYTES = g.NG * g.GROUP_BYTES; g.HIN = HIN;
    return g;
}

constexpr int s2d_taps_per_chunk(int ntap, int piece_stride) {       // largest divisor of ntap whose raw landing zone fits ~26 KB
    int best = 1;
    for (int t = 1; t <= ntap; ++t)
        if (ntap % t == 0 && 2 * t * piece_stride <= 26000) best = t;
    return best;
}

template <int CIN, int COUT, int KS, int S, int HIN, int HOUT, int PAD, bool IN_U8>
struct S2dCfg {
    static constexpr S2dGeom G = s2d_geom(CIN, KS, S, HIN, HOUT, PAD, IN_U8);
    static_assert(((HOUT - 1) * S + KS) % S == 0 && KS % S == 0, "space-to-depth needs S | KS and S | padded size");
    static_assert(CIN % 4 == 0 && COUT % 16 == 0 && G.CP % 16 == 0 && G.NG <= S2D_MAX_GROUPS, "tile constraints");
    static constexpr int W = G.W, KT = G.KT, NTAP = KT * KT, NG = G.NG, PIXP = G.PIXP, LBO_A = G.LBO;
    static constexpr int PARTS = G.PARTS, GROUP_BYTES = G.GROUP_BYTES, IMG_BYTES = G.IMG_BYTES;
    static constexpr int MMAX = (HOUT - 1) * (W + 1);            // largest valid accumulator row
    static constexpr int MT = MMAX / 64 + 1;                     // m64 tiles; MMA warpgroup w owns tiles w, w + 2, ...
    static constexpr int NTW = (MT + 1) / 2;                     // tiles of MMA warpgroup 0 (warpgroup 1: MT / 2)
    static constexpr int ACC = COUT / 2;                         // accumulator floats per thread and tile, main and correction each
    static_assert(2 * NTW * ACC <= 128, "accumulators exceed the MMA warpgroups' register budget");
    static constexpr int MAXOFF = (KT - 1) * (W + 1);
    static constexpr int REACH = MT * 64 + MAXOFF;               // pixels a descriptor may touch from a plane start
    static constexpr int SLACK = REACH > PIXP ? ((REACH - PIXP) * 16 + 127) / 128 * 128 : 0;
    static constexpr int A_REGION = IMG_BYTES + SLACK;
    static constexpr int LBO_B = 2 * COUT * 16;                  // [B_h0 ; B_h1] stacked along N, 8 fp16 k values per row
    // raw landing zone of a chunk inside its ring stage: per tap one piece of 16 contiguous fp32 weight rows for theta and
    // one for the noise; each piece is the 16-byte aligned superset of its rows (+16 bytes)
    static constexpr int PIECE = 16 * COUT * 4;
    static constexpr int PIECE_STRIDE = PIECE + 16;
    static constexpr int TPC = s2d_taps_per_chunk(NTAP, PIECE_STRIDE);   // taps per chunk
    static constexpr int NCPG = NTAP / TPC;                      // chunks per channel group
    static constexpr int NCH = NG * NCPG;                        // chunks per member
    static constexpr int B_TILE = TPC * 2 * LBO_B;               // TPC taps x 16 k = TPC*2 k-octet planes
    static constexpr int RAW_BYTES = 2 * TPC * PIECE_STRIDE;
    static constexpr int BST_BYTES = (cmax(B_TILE, RAW_BYTES) + 127) / 128 * 128;
    static constexpr int FRAME_REGION = IN_U8 ? 2 * S2D_FRAME_STRIDE : 0;        // double-buffered raw uint8 frame
    // epilogue staging, one m64 tile [64][COUT] fp32 per MMA warpgroup: apart from the A region (the next member's image
    // is loading while the epilogue runs) and from the ring
    static constexpr int STAGE_BYTES = 64 * COUT * 4;
    static constexpr int STAGE_REGION = 2 * STAGE_BYTES;
    static constexpr int NSTB = cmin(S2D_MAX_BST, (S2D_SMEM_BUDGET - A_REGION - FRAME_REGION - STAGE_REGION - 256) / BST_BYTES);
    static_assert(NSTB >= 5, "shared memory: B ring too shallow to hide a stage's TMA -> conversion -> MMA cycle");
    static constexpr int SMEM_BYTES = A_REGION + NSTB * BST_BYTES + FRAME_REGION + STAGE_REGION + 256;
    static_assert(SMEM_BYTES <= S2D_SMEM_BUDGET, "shared memory budget");
    static constexpr int B_UNITS = COUT * TPC * 2;               // (column n, k octet) units per chunk
    // converter groups: chunk c is converted by group c % NGRP (independent streams hide the per-chunk hand-off latency)
    static constexpr int NGRP = 2;
    static constexpr int WPG = S2D_CONV_WARPS / NGRP, TG = 32 * WPG;
    static constexpr int B_UPT = (B_UNITS + TG - 1) / TG;
    static_assert(TG % COUT == 0 && NCH % NGRP == 0, "B unit map: a thread keeps its column; groups alternate chunks");
    static_assert(!IN_U8 || NCPG == 1, "the uint8 frame is staged per channel group by the group's (only) chunk");
};

// Where the epilogue writes: NHWC floats (feeding a dense layer) or the NEXT conv layer's image.
struct S2dOut {
    float* base;
    int64_t slot_stride;        // floats
    int next_img;               // 0: NHWC [HOUT*HOUT][COUT];  1: image of the next layer (geometry below)
    int nS, nPADB, nW, nPIXP, nHP;
    float* xc;                  // nullable (NHWC mode only): the same vector as the A operand of the TMA-fed theta GEMM,
    int xc_ko;                  //   Xc[slot / 128][k octet][h0 | h1][slot % 128][8 x fp16]  (theta_gemm_tma.cu), xc_ko = K / 8
};

// ------------------------------------------------------------------------------------------------------------------
// The fused epilogue of one member runs in two steps per m64 tile.  (1) registers -> shared memory: each MMA warpgroup
// folds its accumulators (main + 2^-11 * correction) into a staging tile [64][COUT] fp32 of its own.  This is the only
// part that has to be straight-line code (the accumulators are registers).  (2) shared memory -> global: a rolled loop
// over (row, channel octet) of the staged tile applies (/255) + bias (+BN) + activation to eight values and writes them
// as one 16-byte row of each fp16 split plane of the next layer's image, or as NHWC floats plus the Xc copy.  Its body is
// the same for every tile and member, so it stays in the instruction cache: the per-register path it replaces was fetched
// cold once per member, and that fetch set the epilogue's time.
//
// Octet o of staging row r sits at octet o ^ s2d_stage_swz(r): the fragment stores of a half warp (rows r .. r + 3, the
// same octet) then hit 32 distinct banks.
template <int COUT>
__device__ __forceinline__ int s2d_stage_swz(int r) {
    static_assert(COUT == 16 || COUT % 32 == 0, "staging swizzle");
    return COUT == 16 ? (r >> 1) & 1 : r & 3;
}

// step (1) for tile j of this warpgroup: fragment row wq*16 + lane/4 + 8h, columns 8i + 2*(lane&3) + {0, 1}
template <int COUT, int NTW, int ACC>
__device__ __forceinline__ void s2d_stage_tile(const float (&acc)[NTW][ACC], const float (&cor)[NTW][ACC], int j, int wq,
                                               int lane, uint32_t stage) {
#pragma unroll
    for (int jj = 0; jj < NTW; ++jj) {
        if (jj != j) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = wq * 16 + (lane >> 2) + 8 * h;
            const uint32_t row = stage + (uint32_t)(r * COUT + 2 * (lane & 3)) * 4;
#pragma unroll
            for (int i = 0; i < COUT / 8; ++i) {
                const int k = 4 * i + 2 * h;
                const float v0 = fmaf(cor[jj][k], F16_LO_INV, acc[jj][k]);
                const float v1 = fmaf(cor[jj][k + 1], F16_LO_INV, acc[jj][k + 1]);
                asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(row + (uint32_t)((i ^ s2d_stage_swz<COUT>(r)) * 32)),
                             "f"(v0), "f"(v1) : "memory");
            }
        }
    }
}

// step (2) for tile t: thread k of the warpgroup takes row k % 64 and the octets k / 64, k / 64 + 2, ...
template <int COUT, int HOUT, int W, bool IN_U8>
__device__ __forceinline__ void s2d_store_tile(int t, int k, uint32_t stage, const float* sb, const float* sm, const float* si,
                                               const float* sg, const float* se, int act, bool bn, const S2dOut& so,
                                               float* outp, int slot) {
    constexpr float IN_SCALE = IN_U8 ? (1.0f / 255.0f) : 1.0f;
    constexpr int NO = COUT / 8;
    const int ri = k & 63, m = t * 64 + ri;
    const int oy = m / W, ox = m - oy * W;
    if (oy >= HOUT || ox >= HOUT) return;                        // junk accumulator row
    const uint32_t row = stage + (uint32_t)(ri * COUT) * 4;
    const int swz = s2d_stage_swz<COUT>(ri);
    // the fp16 split rows of octet 0: the next image's pixel (hi plane, lo plane 2 * nPIXP further) or the Xc row pair
    uint4* p_hi = nullptr;
    int lo_off = 0, step = 0;                                    // step: uint4 between the rows of consecutive octets
    if (so.next_img) {
        const int Y = oy + so.nPADB, X = ox + so.nPADB;
        const int pix = (Y / so.nS) * so.nW + (X / so.nS);
        const int pp = (Y % so.nS) * so.nS + (X % so.nS);        // channel octets pp * NO .. of the next image
        p_hi = reinterpret_cast<uint4*>(outp) + (int64_t)pp * (NO / 2) * 4 * so.nPIXP + pix;
        lo_off = 2 * so.nPIXP;
        step = so.nPIXP;
    } else if (so.xc) {
        p_hi = reinterpret_cast<uint4*>(so.xc) + ((int64_t)(slot >> 7) * so.xc_ko + (oy * HOUT + ox) * NO) * 256 + (slot & 127);
        lo_off = 128;
        step = 256;
    }
#pragma unroll 1
    for (int o = k >> 6; o < NO; o += 2) {
        float v[8];
        {
            float4 x0, x1;
            const uint32_t a = row + (uint32_t)((o ^ swz) * 32);
            asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x0.x), "=f"(x0.y), "=f"(x0.z), "=f"(x0.w) : "r"(a));
            asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x1.x), "=f"(x1.y), "=f"(x1.z), "=f"(x1.w) : "r"(a + 16));
            v[0] = x0.x; v[1] = x0.y; v[2] = x0.z; v[3] = x0.w; v[4] = x1.x; v[5] = x1.y; v[6] = x1.z; v[7] = x1.w;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const int n = 8 * o + e;
            float r = v[e];
            if (IN_U8) r *= IN_SCALE;
            r += sb[n];
            if (bn) r = (r - sm[n]) * si[n] * sg[n] + se[n];   // policies.py:322
            v[e] = act == DNE_ACT_RELU ? fmaxf(r, 0.0f) : (act == DNE_ACT_TANH ? tanhf(r) : r);
        }
        if (!so.next_img) {
            float4* dst = reinterpret_cast<float4*>(outp + (int64_t)(oy * HOUT + ox) * COUT + 8 * o);
            dst[0] = make_float4(v[0], v[1], v[2], v[3]);
            dst[1] = make_float4(v[4], v[5], v[6], v[7]);
        }
        if (p_hi) {
            // next image: octet pp * NO + o is plane (o & 1) of plane pair (pp * NO + o) / 2 (NO is even)
            const int po = so.next_img ? ((o >> 1) * 4 + (o & 1)) * step : o * step;
            uint4 hi, lo;
            split_f16x8(v, hi, lo);
            p_hi[po] = hi;
            p_hi[po + lo_off] = lo;
        }
    }
}

template <int CIN, int COUT, int KS, int S, int HIN, int HOUT, int PAD, bool IN_U8>
__global__ void __launch_bounds__(S2D_THREADS, 1)
conv_s2d_kernel(SlotArgs sa, int64_t off_w, LayerEpi epi, const void* __restrict__ in_base, int64_t in_slot_stride,
                S2dOut so, int n_slots, int vdiv, int in_mod) {
    // vdiv > 1 (virtual-batch-norm reference pass, vbn_kernels.cu): the launch covers n_slots = members * vdiv VIRTUAL
    // slots; virtual slot v is image v % vdiv of member v / vdiv -- the member indexes the slot table (theta row, noise
    // index, scale, active flag, BN statistics), v indexes the input / output buffers.  in_mod > 0: the first layer's frames
    // are shared by all members (frame v % in_mod).
    using Cfg = S2dCfg<CIN, COUT, KS, S, HIN, HOUT, PAD, IN_U8>;
    constexpr int NG = Cfg::NG, NSTB = Cfg::NSTB, MT = Cfg::MT, NTW = Cfg::NTW, W = Cfg::W, KT = Cfg::KT;
    constexpr int TPC = Cfg::TPC, NCPG = Cfg::NCPG, NCH = Cfg::NCH;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 127) & ~(uintptr_t)127);
    __shared__ uint64_t a_full[NG], a_empty[NG], raw_full[NSTB], b_full[NSTB], b_empty[NSTB];
    __shared__ uint64_t frame_full[2], frame_empty[2];
    // per-channel epilogue parameters, double buffered by member parity
    __shared__ __align__(16) float s_bias[2][COUT], s_mean[2][COUT], s_inv[2][COUT], s_gamma[2][COUT], s_beta[2][COUT];

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    pdl_trigger();                                               // common.cuh: the next kernel of the tick may be scheduled
    const uint32_t sA = smem_u32(smem), sB = sA + Cfg::A_REGION;
    uint8_t* const gB = smem + Cfg::A_REGION;                                    // generic view of the ring (bulk copies)
    uint8_t* const gFrame = gB + NSTB * Cfg::BST_BYTES;
    uint8_t* const gStage = gFrame + Cfg::FRAME_REGION;                         // epilogue staging of the MMA warpgroups

    if (tid == 0) {
        for (int i = 0; i < NG; ++i) {
            mbar_init(&a_full[i], IN_U8 ? Cfg::WPG : 1);          // the converting group (uint8 frame) or the TMA producer
            mbar_init(&a_empty[i], S2D_MMA_THREADS);              // every MMA thread arrives (no divergent branch between wgmmas)
        }
        for (int i = 0; i < NSTB; ++i) {
            mbar_init(&raw_full[i], 1);                           // weight producer (expect_tx)
            mbar_init(&b_full[i], Cfg::WPG);                      // the warps of the converting group
            mbar_init(&b_empty[i], S2D_MMA_THREADS);
        }
        for (int i = 0; i < 2; ++i) {
            mbar_init(&frame_full[i], 1);
            mbar_init(&frame_empty[i], S2D_CONV_WARPS);
        }
        fence_mbar_init();
    }
    __syncthreads();
    if (warp < 8) regs_inc<S2D_REGS_MMA>();                      // warpgroup-uniform: every warp of a warpgroup runs the same one
    else regs_dec<S2D_REGS_AUX>();

    if (warp < 8) {
        // ============ MMA warpgroups: wgmma into registers, then the fused epilogue of the member ============
        const int w = warp >> 2, wq = warp & 3;
        const int et = tid;                                      // 0 .. 255
        const int act = epi.act;
        const bool bn = epi.bn != DNE_BN_NONE;
        // main and correction accumulators are separate register blocks: a wgmma into a sub-block of another wgmma's
        // accumulators leaves ptxas without registers for the pipeline and serialises every wgmma
        float acc[NTW][Cfg::ACC], cor[NTW][Cfg::ACC];
        uint32_t cb = 0, it = 0;
        pdl_wait();                                              // before the first global write (the zero padding below)
        for (int slot = blockIdx.x; slot < n_slots; slot += gridDim.x) {
            const int ms = slot / vdiv;
            if (!slot_active(sa, ms)) continue;
            const uint32_t pb = it & 1;
            {
                const float* th = slot_theta(sa, ms);
                const int64_t idx = sa.noise_idx[ms];
                const float s = sa.scale[ms];
                for (int c = et; c < COUT; c += S2D_MMA_THREADS) {
                    const ChanEpi ce = make_chan_epi(sa, epi, ms, COUT, c, th, idx, s);
                    s_bias[pb][c] = ce.bias; s_mean[pb][c] = ce.mean; s_inv[pb][c] = ce.inv; s_gamma[pb][c] = ce.gamma; s_beta[pb][c] = ce.beta;
                }
            }
            float* outp = so.base + slot * so.slot_stride;
            if (so.next_img) {
                // zero padding of the next layer's image: pixels (Y, X) of its padded grid that no output maps to
                const int nHP = so.nHP, no = COUT / 8;
                for (int b = et; b < nHP * nHP; b += S2D_MMA_THREADS) {
                    const int Y = b / nHP, X = b - Y * nHP;
                    if (Y >= so.nPADB && Y < so.nPADB + HOUT && X >= so.nPADB && X < so.nPADB + HOUT) continue;
                    const int pix = (Y / so.nS) * so.nW + (X / so.nS), pp = (Y % so.nS) * so.nS + (X % so.nS);
                    for (int q = 0; q < no; ++q) {
                        const int co = pp * no + q;                                   // channel octet of the next image
                        uint4* p = reinterpret_cast<uint4*>(outp) + (size_t)((co >> 1) * 4 + (co & 1)) * so.nPIXP + pix;
                        p[0] = make_uint4(0u, 0u, 0u, 0u);
                        p[(size_t)2 * so.nPIXP] = make_uint4(0u, 0u, 0u, 0u);
                    }
                }
            }
            // ---- main loop: one chunk = TPC taps x 16 channels of one channel group ----
            for (int c = 0; c < NCH; ++c, ++cb) {
                const int g = c / NCPG, tc = c - g * NCPG;
                const uint32_t st = cb % NSTB;
                if (tc == 0) mbar_wait(&a_full[g], it & 1);
                mbar_wait(&b_full[st], (cb / NSTB) & 1);
                wgmma_fence();
#pragma unroll
                for (int tl = 0; tl < TPC; ++tl) {
                    const int tap = tc * TPC + tl;
                    const int toff = (tap / KT) * W + (tap % KT);
                    const uint64_t dB = smem_desc(sB + st * Cfg::BST_BYTES + tl * 2 * Cfg::LBO_B, Cfg::LBO_B, 128);
#pragma unroll
                    for (int j = 0; j < NTW; ++j) {
                        // no branch around the wgmmas (a warp-divergent path serialises them): with an odd tile count,
                        // warpgroup 1 recomputes the last tile into an accumulator its epilogue skips
                        const int t = min(w + 2 * j, MT - 1);
                        const uint64_t dA = smem_desc(sA + g * Cfg::GROUP_BYTES + (t * 64 + toff) * 16, Cfg::LBO_A, 128);
                        const uint32_t first = (c | tl) != 0;
                        wgmma_f16<COUT>(acc[j], dA, dB, first);                                                  // A_h0 * B_h0
                        wgmma_f16<COUT>(cor[j], dA, dB + (uint64_t)((COUT * 16) >> 4), first);                   // A_h0 * B_h1 -> correction
                        if (!IN_U8) wgmma_f16<COUT>(cor[j], dA + (uint64_t)((2 * Cfg::LBO_A) >> 4), dB, 1);     // A_h1 * B_h0 -> correction
                    }
                }
                wgmma_commit();
                wgmma_wait<1>();                                 // the previous chunk's wgmmas have read their operands
                if (c > 0) {
                    const int pg = (c - 1) / NCPG;
                    mbar_arrive(&b_empty[(cb - 1) % NSTB]);
                    if ((c - 1) - pg * NCPG == NCPG - 1) mbar_arrive(&a_empty[pg]);
                }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int j = 0; j < NTW; ++j) {
                fence_regs<Cfg::ACC>(acc[j]);
                fence_regs<Cfg::ACC>(cor[j]);
            }
            mbar_arrive(&b_empty[(cb - 1) % NSTB]);
            mbar_arrive(&a_empty[NG - 1]);
            named_bar_sync(2, S2D_MMA_THREADS);                  // per-channel parameters (and padding) of this member ready,
                                                                 // and the staging tiles of the previous member read
            // ---- epilogue, one tile at a time: registers -> staging tile -> (/255) + bias (+BN) + activation -> global ----
            {
                const float *sb = s_bias[pb], *sm = s_mean[pb], *si = s_inv[pb], *sg = s_gamma[pb], *se = s_beta[pb];
                const uint32_t stage = smem_u32(gStage) + w * Cfg::STAGE_BYTES;
#pragma unroll 1
                for (int j = 0; j < NTW; ++j) {
                    const int t = w + 2 * j;
                    if (t >= MT) break;                          // warpgroup-uniform
                    if (j > 0) named_bar_sync(5 + w, 128);       // the previous tile is read
                    s2d_stage_tile<COUT, NTW, Cfg::ACC>(acc, cor, j, wq, lane, stage);
                    named_bar_sync(5 + w, 128);
                    s2d_store_tile<COUT, HOUT, W, IN_U8>(t, tid & 127, stage, sb, sm, si, sg, se, act, bn, so, outp, slot);
                }
            }
            ++it;
        }
    } else if (warp == 12) {
        // ================= image producer (TMA): the member's image, one channel-octet group per bulk copy; =================
        // ================= first layer: the member's raw uint8 frame (double buffered)                      =================
        if (lane == 0) {
            pdl_wait();                                          // the image / frame is written by the previous kernel of the tick
            uint32_t it = 0;
            for (int slot = blockIdx.x; slot < n_slots; slot += gridDim.x) {
                if (!slot_active(sa, slot / vdiv)) continue;
                if (IN_U8) {
                    const uint32_t fb = it & 1;
                    mbar_wait(&frame_empty[fb], ((it >> 1) & 1) ^ 1);
                    mbar_arrive_expect_tx(&frame_full[fb], S2D_FRAME_BYTES);
                    const int fslot = in_mod > 0 ? slot % in_mod : slot;
                    bulk_g2s(gFrame + fb * S2D_FRAME_STRIDE, (const uint8_t*)in_base + fslot * in_slot_stride, S2D_FRAME_BYTES,
                             &frame_full[fb]);
                } else {
                    const uint8_t* src = (const uint8_t*)((const float*)in_base + slot * in_slot_stride);
                    for (int g = 0; g < NG; ++g) {
                        mbar_wait(&a_empty[g], (it & 1) ^ 1);
                        mbar_arrive_expect_tx(&a_full[g], Cfg::GROUP_BYTES);
                        bulk_g2s(smem + g * Cfg::GROUP_BYTES, src + (size_t)g * Cfg::GROUP_BYTES, Cfg::GROUP_BYTES, &a_full[g]);
                    }
                }
                ++it;
            }
        }
    } else if (warp == 13) {
        // ================= weight producer (TMA): raw theta rows + raw noise rows of every chunk, NSTB chunks deep =================
        if (lane == 0) {
            uint32_t cb = 0;
            for (int slot = blockIdx.x; slot < n_slots; slot += gridDim.x) {
                const int ms = slot / vdiv;
                if (!slot_active(sa, ms)) continue;
                const float* th = slot_theta(sa, ms) + off_w;
                const float* nz = sa.noise + sa.noise_idx[ms] + off_w;
                const int a_t = (int)(((uintptr_t)th >> 2) & 3), a_n = (int)(((uintptr_t)nz >> 2) & 3);
                for (int c = 0; c < NCH; ++c, ++cb) {
                    const int g = c / NCPG, tc = c - g * NCPG;
                    const uint32_t st = cb % NSTB;
                    mbar_wait(&b_empty[st], ((cb / NSTB) & 1) ^ 1);
                    mbar_arrive_expect_tx(&raw_full[st], Cfg::RAW_BYTES);
                    uint8_t* dst = gB + st * Cfg::BST_BYTES;
                    const int cp = 16 * g, pp = cp / CIN, ci = cp % CIN, py = pp / S, px = pp % S;
#pragma unroll
                    for (int tl = 0; tl < TPC; ++tl) {
                        const int tap = tc * TPC + tl;
                        const int ty = tap / KT, tx = tap % KT;
                        const int kk = ((ty * S + py) * KS + (tx * S + px)) * CIN + ci;          // first of 16 contiguous weight rows
                        bulk_g2s(dst + tl * Cfg::PIECE_STRIDE, th + (int64_t)kk * COUT - a_t, Cfg::PIECE_STRIDE, &raw_full[st]);
                        bulk_g2s(dst + (TPC + tl) * Cfg::PIECE_STRIDE, nz + (int64_t)kk * COUT - a_n, Cfg::PIECE_STRIDE, &raw_full[st]);
                    }
                }
            }
        }
    } else if (warp < 12) {
        // ================= converter warps: raw rows -> perturbed, split [B_hi ; B_lo] tile, in place =================
        // =================                  (first layer: also the uint8 frame -> image planes)       =================
        constexpr int TG = Cfg::TG, NGRP = Cfg::NGRP;
        const int ct = tid - S2D_MMA_THREADS;                    // 0 .. S2D_CONV_THREADS - 1
        const int grp = ct / TG, tg = ct - grp * TG;
        // zero fill, once: the uint8 variant relies on the zero padding of its image never being overwritten (the
        // converter warps are its only writers); the TMA-fed variants only need finite values in the slack behind the last
        // plane, which is read into junk accumulator rows.  Only the converter warps wait for it.
        {
            constexpr int Z0 = IN_U8 ? 0 : Cfg::IMG_BYTES, Z1 = Cfg::A_REGION;
            for (int i = Z0 / 16 + ct; i < Z1 / 16; i += S2D_CONV_THREADS) sts128(sA + i * 16, make_float4(0.f, 0.f, 0.f, 0.f));
            fence_proxy_async_smem();
            named_bar_sync(1, S2D_CONV_THREADS);
        }
        const int n = tg % COUT;                                 // this thread's output channel in every unit
        constexpr int KQ_STEP = TG / COUT;
        const int kq0 = tg / COUT;
        uint32_t it = 0;
        for (int slot = blockIdx.x; slot < n_slots; slot += gridDim.x) {
            const int ms = slot / vdiv;
            if (!slot_active(sa, ms)) continue;
            const float* th = slot_theta(sa, ms) + off_w;
            const float* nz = sa.noise + sa.noise_idx[ms] + off_w;
            const int a_t = (int)(((uintptr_t)th >> 2) & 3), a_n = (int)(((uintptr_t)nz >> 2) & 3);
            const float s = sa.scale[ms];
            if (IN_U8) mbar_wait(&frame_full[it & 1], (it >> 1) & 1);
            for (int c = grp; c < NCH; c += NGRP) {
                const int g = c / NCPG;
                const uint32_t cb = it * NCH + c, st = cb % NSTB;
                if (IN_U8) {
                    // ---- the uint8 frame, channel group g = py (all four px phases): plane h holds the pixel pair
                    // px in {2h, 2h+1}: 8 bytes -> 8 fp16 channels = one 16-byte row ----
                    static_assert(!IN_U8 || (CIN == 4 && S == 4 && HIN == 84), "uint8 staging is written for the 84x84x4 frame stack, stride 4");
                    const uint32_t frame = smem_u32(gFrame + (it & 1) * S2D_FRAME_STRIDE);
                    const int py = g;
                    mbar_wait(&a_empty[g], (it & 1) ^ 1);
                    for (int u = tg; u < 2 * W * W; u += TG) {
                        const int h = u / (W * W), pix = u - h * (W * W);
                        const int yq = pix / W, xq = pix - yq * W;
                        const int y = 4 * yq + py - PAD, x0 = 4 * xq + 2 * h - PAD;
                        if (y >= 0 && y < HIN && x0 >= 0 && x0 < HIN) {
                            uint32_t p0, p1;
                            asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(p0), "=r"(p1) : "r"(frame + (y * HIN + x0) * 4));
                            auto h2 = [](uint32_t lo8, uint32_t hi8) {        // two bytes -> two fp16 (exact)
                                return (uint32_t)__half_as_ushort(__ushort2half_rn((unsigned short)lo8)) |
                                       ((uint32_t)__half_as_ushort(__ushort2half_rn((unsigned short)hi8)) << 16);
                            };
                            const uint4 row = make_uint4(h2(p0 & 255u, (p0 >> 8) & 255u), h2((p0 >> 16) & 255u, p0 >> 24),
                                                         h2(p1 & 255u, (p1 >> 8) & 255u), h2((p1 >> 16) & 255u, p1 >> 24));
                            sts128u(sA + g * Cfg::GROUP_BYTES + h * Cfg::LBO_A + pix * 16, row);
                        }
                    }
                    fence_proxy_async_smem();
                    __syncwarp();
                    if (lane == 0) {
                        mbar_arrive(&a_full[g]);
                        if (c + NGRP >= NCH) mbar_arrive(&frame_empty[it & 1]);    // this warp's last read of the raw frame
                    }
                }
                mbar_wait(&raw_full[st], (cb / NSTB) & 1);
                const uint32_t sBs = sB + st * Cfg::BST_BYTES;
                float w[Cfg::B_UPT][8];
#pragma unroll
                for (int i = 0; i < Cfg::B_UPT; ++i) {
                    const int kp = kq0 + i * KQ_STEP;            // local k octet: tap kp >> 1 of the chunk, rows 8*(kp & 1) .. +7 of its piece
                    if (kp < TPC * 2) {
                        const uint32_t pt = sBs + (kp >> 1) * Cfg::PIECE_STRIDE + (uint32_t)((a_t + (8 * (kp & 1)) * COUT + n) * 4);
                        const uint32_t pn = sBs + (TPC + (kp >> 1)) * Cfg::PIECE_STRIDE + (uint32_t)((a_n + (8 * (kp & 1)) * COUT + n) * 4);
#pragma unroll
                        for (int j = 0; j < 8; ++j) w[i][j] = perturbed(lds32(pt + j * COUT * 4), s, lds32(pn + j * COUT * 4));
                    }
                }
                named_bar_sync(3 + grp, TG);                     // every raw value of the stage is in registers: overwrite it
#pragma unroll
                for (int i = 0; i < Cfg::B_UPT; ++i) {
                    const int kp = kq0 + i * KQ_STEP;
                    if (kp < TPC * 2) {
                        uint4 hi, lo;
                        split_f16x8(w[i], hi, lo);
                        sts128u(sBs + kp * Cfg::LBO_B + n * 16, hi);
                        sts128u(sBs + kp * Cfg::LBO_B + (COUT + n) * 16, lo);
                    }
                }
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) mbar_arrive(&b_full[st]);
            }
            ++it;
        }
    }
}

template <int CIN, int COUT, int KS, int S, int HIN, int HOUT, int PAD, bool IN_U8>
int launch_s2d(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, const void* in, int64_t in_slot_stride,
               const S2dOut& so, int n_slots, int sm_count, cudaStream_t st, int vdiv, int in_mod) {
    using Cfg = S2dCfg<CIN, COUT, KS, S, HIN, HOUT, PAD, IN_U8>;
    auto kern = conv_s2d_kernel<CIN, COUT, KS, S, HIN, HOUT, PAD, IN_U8>;
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_done[64] = {};                              // per device (one context per device and process)
    if (dev < 64 && !attr_done[dev]) {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES) != cudaSuccess)
            return DNE_ERR_CUDA;
        attr_done[dev] = true;
    }
    const int grid = n_slots < sm_count ? n_slots : sm_count;
    // the first layer follows host copies / the previous tick's graph: launched fully serialized.  The weight producer and
    // the converter warps of the later layers never wait: theta and the noise table are not written inside a tick.
    // (dne_set_option("chain_ticks", 1): the caller guarantees that the stream's previous kernel is the previous tick's head --
    // nothing that writes theta, the noise table or the slot table -- and the first layer joins the chain too.)
    if (dne_launch_chain(kern, dim3(grid), dim3(S2D_THREADS), (size_t)Cfg::SMEM_BYTES, st, !IN_U8 || g_dne_chain_ticks, sa, (int64_t)L.off_w, epi, in,
                         in_slot_stride, so, n_slots, vdiv, in_mod) != cudaSuccess)
        return DNE_ERR_CUDA;
    DNE_LAUNCHED(1);
    return 0;
}

bool shape_is(const dne_layer_desc& L, int cin, int cout, int ks, int stride, int hin, int hout, int pad) {
    return L.kind == DNE_CONV && L.cin == cin && L.cout == cout && L.ksize == ks && L.stride == stride && L.hin == hin &&
           L.hout == hout && L.pad == pad;
}

}  // namespace

// ---- host interface (forward.cuh) ---------------------------------------------------------------------------------
// Shapes compiled in: the Nature-DQN family of the reference (models/dqn.py:25-47, policies.py:321-327,451-453).
bool dne_s2d_supported(const dne_layer_desc& L, bool in_u8) {
    if (in_u8) return shape_is(L, 4, 32, 8, 4, 84, 21, 2) || shape_is(L, 4, 16, 8, 4, 84, 21, 2);
    return shape_is(L, 32, 64, 4, 2, 21, 11, 1) || shape_is(L, 16, 32, 4, 2, 21, 11, 1) || shape_is(L, 64, 64, 3, 1, 11, 11, 1);
}

// Bytes of layer L's INPUT image (what the producing epilogue writes per slot); 0 if L is not an s2d conv layer.
size_t dne_s2d_image_bytes(const dne_layer_desc& L) {
    if (!dne_s2d_supported(L, false)) return 0;
    const S2dGeom g = s2d_geom(L.cin, L.ksize, L.stride, L.hin, L.hout, L.pad, false);
    return (size_t)g.IMG_BYTES;
}

// Geometry of layer L's input image for an external writer (vbn_image_kernel): S, PADB, W, PIXP, HP = W * S.
void dne_s2d_image_geom(const dne_layer_desc& L, int* nS, int* nPADB, int* nW, int* nPIXP, int* nHP) {
    const S2dGeom g = s2d_geom(L.cin, L.ksize, L.stride, L.hin, L.hout, L.pad, false);
    *nS = g.S; *nPADB = g.PADB; *nW = g.W; *nPIXP = g.PIXP; *nHP = g.W * g.S;
}

// next: the following conv layer if it consumes an image (nullptr: write NHWC floats).
int dne_launch_conv_layer_s2d(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, bool in_u8, const void* in,
                              int64_t in_slot_stride, float* out, int64_t out_slot_stride, const dne_layer_desc* next,
                              int n_slots, int sm_count, cudaStream_t st, float* xc, int vdiv, int in_mod) {
    S2dOut so;
    so.xc = next ? nullptr : xc;
    so.xc_ko = (L.hout * L.hout * L.cout) / 8;
    so.base = out;
    so.slot_stride = out_slot_stride;
    so.next_img = next ? 1 : 0;
    so.nS = so.nPADB = so.nW = so.nPIXP = so.nHP = 1;
    if (next) {
        const S2dGeom g = s2d_geom(next->cin, next->ksize, next->stride, next->hin, next->hout, next->pad, false);
        so.nS = g.S; so.nPADB = g.PADB; so.nW = g.W; so.nPIXP = g.PIXP; so.nHP = g.W * g.S;
    }
#define ARGS sa, L, epi, in, in_slot_stride, so, n_slots, sm_count, st, (vdiv < 1 ? 1 : vdiv), in_mod
    if (in_u8 && shape_is(L, 4, 32, 8, 4, 84, 21, 2)) return launch_s2d<4, 32, 8, 4, 84, 21, 2, true>(ARGS);
    if (in_u8 && shape_is(L, 4, 16, 8, 4, 84, 21, 2)) return launch_s2d<4, 16, 8, 4, 84, 21, 2, true>(ARGS);
    if (!in_u8 && shape_is(L, 32, 64, 4, 2, 21, 11, 1)) return launch_s2d<32, 64, 4, 2, 21, 11, 1, false>(ARGS);
    if (!in_u8 && shape_is(L, 16, 32, 4, 2, 21, 11, 1)) return launch_s2d<16, 32, 4, 2, 21, 11, 1, false>(ARGS);
    if (!in_u8 && shape_is(L, 64, 64, 3, 1, 11, 11, 1)) return launch_s2d<64, 64, 3, 1, 11, 11, 1, false>(ARGS);
#undef ARGS
    return DNE_ERR_UNSUP;
}
