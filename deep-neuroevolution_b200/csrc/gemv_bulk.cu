// gemv_bulk.cu -- the HBM-bound GEMV of the decomposed dense layers, streaming the UNION of a launch's weight slices once.
//
// Same math as dense_noise_gemv_kernel (forward_kernels.cu): for every group of G slots that share one slice,
//     y_g[n] = sum_k x_g[k] * W[k][n],   W = base[E0 + k*N + n],   E0 = idx[slot0] + off (arbitrary alignment)
// The slices of one launch start at unrelated offsets of one table (noise slab, or the theta matrix for GA parents) and
// overlap: 128 random 15.9 MB fc slices of the 1 GB noise table cover it about 2 times over.  Streaming every slice on
// its own reads each covered byte ~2.3 times, and L2 (50 MB) absorbs almost none of it.  This kernel cuts the table into
// a fixed grid of rows of N floats (aligned to the table base), groups the rows into blocks of GU_BLK rows, and makes every
// block that some active group's slice intersects one work item: the item streams the block's covered rows ONCE into a
// shared-memory ring (producer warp, cp.async.bulk, full / empty mbarriers) and applies them to every covering group.
//
// Row R, table column c of group g (R_g = E0_g div N, rho_g = E0_g mod N) is weight
//     k = R - R_g - [c < rho_g],   n = (c - rho_g) mod N.
// Consumer thread t owns column quad 4t..4t+3 of every row, so for each group its four components always feed the same four
// outputs (rotated by rho_g), with multiplier x[k] or x[k-1].  x is staged per item over the block's rows, zero outside
// [0, K) -- rows of the block that a group does not cover contribute exactly zero.  Each staged float4 is read from shared
// memory once and used for every covering group (at most GU_VEC / G groups per pass; a block with more covering groups is
// streamed again for the rest).
//
// Partials: group g's piece i is block floor(R_g / GU_BLK) + i, written to part[group][i][G][N] for i < M (dne_gemv_pieces);
// pieces the group does not reach are written as zero.  The combine kernels add the M pieces in order: deterministic.
//
// The plan (which blocks, which groups cover each) depends only on the slot table, which nothing inside a tick writes, so
// every CTA derives it in its prologue -- before griddepcontrol.wait -- from the <= n_groups intervals: no host sync, and it
// cannot go stale when a caller rewrites the index tensors.  Items are dealt round-robin over the persistent CTAs.
#include <climits>
#include "common.cuh"
#include "forward.cuh"
#include "epilogue.cuh"
#include "wgmma.cuh"

using namespace wg;

int g_dne_gemv_bulk = 1;
int g_dne_gemv_ctas_per_sm = 2;
int g_dne_gemv_grid = 0;             // > 0: cap on the number of CTAs (dne_set_option("gemv_grid")): leaves whole SMs to another stream
int g_dne_gemv_stages = 5;           // shared-memory ring depth upper bound (2..GB_STAGES), dne_set_option("gemv_stages")

constexpr int GB_CONSUMERS = 256;
constexpr int GB_THREADS = GB_CONSUMERS + 32;      // + one producer warp
constexpr int GB_STAGES = 8;                       // maximum ring depth (barrier arrays); the launch picks n_stages <= this
constexpr int GB_STAGE_BYTES = 16384;
constexpr int GB_RPR = 4;                          // rows per reader per stage: (16384/4N) / (256/(N/4)) = 4 for every N
constexpr int GU_BLK = DNE_GEMV_BLOCK_ROWS;        // table rows per block (work item)
constexpr int GU_VEC = 8;                          // x vectors (covering groups x G) per pass: accumulator registers / 4
constexpr int GU_VB = 4;                           // x vectors per round of the cross-reader reduction
constexpr int GU_MIN_N = 64;                       // rows per stage 4096 / N <= 64
constexpr int GU_XS_LD_MAX = GU_BLK + 4096 / GU_MIN_N;
// shared array of the x staging [GU_VEC][XS_LD] and, after a pass's last stage, of the reduction [RW][GU_VB][N + 4]
constexpr int GU_XS_FLOATS = GU_VEC * GU_XS_LD_MAX > (1024 / GU_MIN_N) * GU_VB * (GU_MIN_N + 4)
                                 ? GU_VEC * GU_XS_LD_MAX : (1024 / GU_MIN_N) * GU_VB * (GU_MIN_N + 4);
constexpr int GU_PLAN_BYTES_PER_GROUP = 8 + 5 * 4; // E0, b0, b1, sorted, start, prefix

// Lists (one warp) the groups covering block b whose ordinal among them lies in [first, first + cap) into out[], in group
// order; returns the total number of covering groups.
__device__ __forceinline__ int gu_cover(const int* pb0, const int* pb1, int n_groups, int b, int first, int cap, int* out,
                                        int lane) {
    int total = 0;
    for (int h0 = 0; h0 < n_groups; h0 += 32) {
        const int h = h0 + lane;
        const bool c = h < n_groups && pb0[h] <= b && b <= pb1[h];
        const unsigned m = __ballot_sync(0xffffffffu, c);
        const int ord = total + __popc(m & ((1u << lane) - 1u));
        if (c && ord >= first && ord < first + cap) out[ord - first] = h;
        total += __popc(m);
    }
    __syncwarp();
    return total;
}

template <int G>
__global__ void __launch_bounds__(GB_THREADS, 2)
gemv_union_kernel(SlotArgs sa, GemvSrc src, const float* __restrict__ X, int64_t x_slot_stride, int K, int N,
                  int n_pieces, int n_groups, int n_slots, float* __restrict__ part, int n_stages,
                  const float* __restrict__ tpart, int t_split) {
    // tpart != nullptr ("fold"): the shared-theta GEMM's split-K partials [t_split][n_slots][N] are folded into this
    // kernel's output, part[group][piece][g][n] = s_g * (noise partial of the piece) + sum_{j = piece (mod n_pieces)} tpart[j]:
    // the combine kernel then adds n_pieces values per output instead of n_pieces + t_split.  Fixed summation order.
    constexpr int CAP = GU_VEC / G;                    // covering groups per pass
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 127) & ~(uintptr_t)127);
    float* stage_base = reinterpret_cast<float*>(smem);
    int64_t* pE0 = reinterpret_cast<int64_t*>(smem + n_stages * GB_STAGE_BYTES);
    int* pb0 = reinterpret_cast<int*>(pE0 + n_groups);      // first / last block of each group (INT_MAX / -1: inactive)
    int* pb1 = pb0 + n_groups;
    int* psort = pb1 + n_groups;                             // groups by (first block, index)
    int* pstart = psort + n_groups;                          // first block sorted entry i adds to the union
    int* ppre = pstart + n_groups;                           // blocks added by the sorted entries before i
    __shared__ uint64_t full_bar[GB_STAGES], empty_bar[GB_STAGES];
    __shared__ __align__(16) float xs[GU_XS_FLOATS];   // xs[v][1 + L] = x_v[k] at block row L; reused by the reduction
    __shared__ int cov_c[CAP], cov_p[CAP];                  // this pass's groups: consumers / producer
    __shared__ int rho_c[CAP];
    __shared__ int s_total, s_row0, s_nelem, s_items;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NQ = N >> 2;
    const int RW = GB_CONSUMERS / NQ;                  // row readers per stage
    const int RB = GB_RPR * RW;                        // rows per stage
    const int XS_LD = GU_BLK + RB;
    pdl_trigger();                                     // common.cuh: PDL chain of the tick

    if (tid == 0) {
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], GB_CONSUMERS / 32);
        }
        fence_mbar_init();
    }
    // ---- plan, step 1: every group's slice start and block interval ----
    for (int g = tid; g < n_groups; g += GB_THREADS) {
        const int slot0 = g * G;
        bool any = false;
#pragma unroll
        for (int m = 0; m < G; ++m) any = any || (slot0 + m < n_slots && slot_active(sa, slot0 + m));
        const int64_t E0 = (src.idx64 ? src.idx64[slot0] : (src.idx32 ? (int64_t)src.idx32[slot0] * src.mul : 0)) + src.off;
        pE0[g] = E0;
        pb0[g] = any ? (int)(E0 / N / GU_BLK) : INT_MAX;
        pb1[g] = any ? (int)((E0 + (int64_t)K * N - 1) / N / GU_BLK) : -1;
    }
    __syncthreads();
    // ---- step 2: rank sort by (first block, group) ----
    for (int g = tid; g < n_groups; g += GB_THREADS) {
        const int key = pb0[g];
        int r = 0;
        for (int h = 0; h < n_groups; ++h) {
            const int kh = pb0[h];
            r += (kh < key) || (kh == key && h < g);
        }
        psort[r] = g;
    }
    __syncthreads();
    // ---- step 3 (warp 0): blocks each sorted entry adds to the union, and their prefix sum = item numbering ----
    if (warp == 0) {
        int carry_max = -1, carry_sum = 0;
        for (int i0 = 0; i0 < n_groups; i0 += 32) {
            const int i = i0 + lane;
            const int g = i < n_groups ? psort[i] : 0;
            const int b0 = i < n_groups ? pb0[g] : INT_MAX, b1 = i < n_groups ? pb1[g] : -1;
            int mx = b1;                                  // inclusive max scan of the last blocks
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int o = __shfl_up_sync(0xffffffffu, mx, d);
                if (lane >= d) mx = max(mx, o);
            }
            int before = __shfl_up_sync(0xffffffffu, mx, 1);
            if (lane == 0) before = -1;
            before = max(before, carry_max);
            const int start = max(b0, before + 1);
            const int add = (b0 != INT_MAX && b1 >= start) ? b1 - start + 1 : 0;
            int sum = add;                                // inclusive sum scan
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const int o = __shfl_up_sync(0xffffffffu, sum, d);
                if (lane >= d) sum += o;
            }
            if (i < n_groups) { pstart[i] = start; ppre[i] = carry_sum + sum - add; }
            carry_sum += __shfl_sync(0xffffffffu, sum, 31);
            carry_max = max(carry_max, __shfl_sync(0xffffffffu, mx, 31));
        }
        if (lane == 0) s_items = carry_sum;
    }
    __syncthreads();
    const int n_items = s_items;
    auto item_block = [&](int q) {                     // sorted entry i with ppre[i] <= q < ppre[i] + added_i (the last such)
        int lo = 0, hi = n_groups;                     // first index with ppre > q
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ppre[mid] <= q) lo = mid + 1; else hi = mid;
        }
        return pstart[lo - 1] + (q - ppre[lo - 1]);
    };
    // rows [row0, row0 + n_elem / N) of the table cover the pass: from the first covered row of block b to the last,
    // ending at the 16-byte-rounded end of the furthest slice (never past the table)
    auto pass_range = [&](int b, const int* gl, int ng, int64_t& row0, int& n_elem) {
        int64_t r_first = INT64_MAX, e_last = 0;
        for (int i = 0; i < ng; ++i) {
            const int64_t E0 = pE0[gl[i]];
            r_first = min(r_first, E0 / N);
            e_last = max(e_last, (E0 + (int64_t)K * N + 3) & ~(int64_t)3);
        }
        const int64_t blk0 = (int64_t)b * GU_BLK;
        row0 = max(r_first, blk0);
        const int64_t e_end = min(e_last, (blk0 + GU_BLK) * N);
        n_elem = (int)(e_end - row0 * N);
    };

    if (warp == GB_CONSUMERS / 32) {
        // ===================== producer warp =====================
        uint32_t it = 0;
        for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
            const int b = item_block(item);
            int total = CAP;
            for (int first = 0; first < total; first += CAP) {
                total = gu_cover(pb0, pb1, n_groups, b, first, CAP, cov_p, lane);
                int64_t row0;
                int n_elem;
                pass_range(b, cov_p, min(CAP, total - first), row0, n_elem);
                const float* gsrc = src.base + row0 * N;
                for (int e0 = 0; e0 < n_elem; e0 += RB * N, ++it) {
                    if (lane == 0) {
                        const int s = it % n_stages;
                        mbar_wait(&empty_bar[s], ((it / n_stages) & 1) ^ 1);
                        const uint32_t bytes = (uint32_t)min(RB * N, n_elem - e0) * 4;
                        mbar_arrive_expect_tx(&full_bar[s], bytes);
                        bulk_g2s(stage_base + (size_t)s * (GB_STAGE_BYTES / 4), gsrc + e0, bytes, &full_bar[s]);
                    }
                }
                __syncwarp();                          // cov_p is rewritten by the next pass
            }
        }
        return;
    }

    // ===================== consumer warps =====================
    // (the producer above streams weight rows -- written before the tick -- without waiting; X and part need the chain)
    pdl_wait();
    const int t = tid % NQ, rw = tid / NQ;
    const int red_ld = N + 4;
    float* red = xs;                                   // [RW][GU_VB][N + 4], after the last stage of a pass
    uint32_t it = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int b = item_block(item);
        int total = CAP;
        for (int first = 0; first < total; first += CAP) {
            if (warp == 0) {
                const int tot = gu_cover(pb0, pb1, n_groups, b, first, CAP, cov_c, lane);
                if (lane == 0) {
                    const int ng = min(CAP, tot - first);
                    int64_t row0;
                    int n_elem;
                    pass_range(b, cov_c, ng, row0, n_elem);
                    s_total = tot;
                    s_row0 = (int)(row0 - (int64_t)b * GU_BLK);     // block-relative
                    s_nelem = n_elem;
                    for (int i = 0; i < ng; ++i) rho_c[i] = (int)(pE0[cov_c[i]] % N);
                }
            }
            named_bar_sync(1, GB_CONSUMERS);                               // barrier A: pass plan
            total = s_total;
            const int ng = min(CAP, total - first), nv = ng * G;
            const int lrow0 = s_row0, n_elem = s_nelem;
            // stage x_v over block rows -1 .. XS_LD-2: xs[v][L + 1] = x_v[k], k = row - R_g, zero outside [0, K)
            for (int i = tid; i < nv * XS_LD; i += GB_CONSUMERS) {
                const int v = i / XS_LD, L = i - v * XS_LD - 1;
                const int g = cov_c[v / G], slot = g * G + v % G;
                const int64_t k = (int64_t)b * GU_BLK + L - pE0[g] / N;
                xs[v * XS_LD + L + 1] = (k >= 0 && k < K && slot < n_slots) ? X[(int64_t)slot * x_slot_stride + k] : 0.0f;
            }
            named_bar_sync(1, GB_CONSUMERS);                               // barrier B: xs staged

            float acc[GU_VEC][4];
#pragma unroll
            for (int v = 0; v < GU_VEC; ++v)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[v][c] = 0.0f;

            for (int e0 = 0; e0 < n_elem; e0 += RB * N, ++it) {
                const int s = it % n_stages;
                const int stage_elems = min(RB * N, n_elem - e0);
                const int rl0 = rw * GB_RPR;           // this reader's first row inside the stage (contiguous rows)
                const int xb0 = lrow0 + e0 / N + rl0;  // xs index of x[k - 1] for the reader's first row
                mbar_wait(&full_bar[s], (it / n_stages) & 1);
                // explicit ld.shared (a C++ pointer into the re-aligned dynamic smem compiles to generic LD.E)
                const uint32_t rows_a = wg::smem_u32(stage_base) + s * GB_STAGE_BYTES + (rl0 * NQ + t) * 16;
                float4 w[GB_RPR];
#pragma unroll
                for (int j = 0; j < GB_RPR; ++j)       // columns past the streamed end (last row of the pass) are zero
                    w[j] = ((rl0 + j) * N + 4 * t < stage_elems) ? wg::lds128(rows_a + j * NQ * 16) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                for (int gi = 0; gi < CAP; ++gi) {
                    if (gi < ng) {
                        const int rho = rho_c[gi];     // components c < rho carry row k - 1
                        const bool p0 = 4 * t < rho, p1 = 4 * t + 1 < rho, p2 = 4 * t + 2 < rho, p3 = 4 * t + 3 < rho;
#pragma unroll
                        for (int m = 0; m < G; ++m) {
                            const int v = gi * G + m;
                            float xm[GB_RPR + 1];
#pragma unroll
                            for (int j = 0; j <= GB_RPR; ++j) xm[j] = xs[v * XS_LD + xb0 + j];
#pragma unroll
                            for (int j = 0; j < GB_RPR; ++j) {
                                acc[v][0] = fmaf(p0 ? xm[j] : xm[j + 1], w[j].x, acc[v][0]);
                                acc[v][1] = fmaf(p1 ? xm[j] : xm[j + 1], w[j].y, acc[v][1]);
                                acc[v][2] = fmaf(p2 ? xm[j] : xm[j + 1], w[j].z, acc[v][2]);
                                acc[v][3] = fmaf(p3 ? xm[j] : xm[j + 1], w[j].w, acc[v][3]);
                            }
                        }
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty_bar[s]);           // this warp is done reading stage s
            }
            // cross-reader reduction in fixed order, GU_VB vectors per round (red aliases xs: wait for every reader)
            for (int vb0 = 0; vb0 < nv; vb0 += GU_VB) {
                named_bar_sync(1, GB_CONSUMERS);                           // barrier C: xs / red free
#pragma unroll
                for (int v = 0; v < GU_VEC; ++v) {
                    if (v >= vb0 && v < vb0 + GU_VB && v < nv) {
                        const int rho = rho_c[v / G];
                        float* row = red + (rw * GU_VB + (v - vb0)) * red_ld;
#pragma unroll
                        for (int c = 0; c < 4; ++c) {
                            const int n = 4 * t + c - rho;
                            row[n < 0 ? n + N : n] = acc[v][c];
                        }
                    }
                }
                named_bar_sync(1, GB_CONSUMERS);                           // barrier D
                for (int i = tid; i < GU_VB * N; i += GB_CONSUMERS) {
                    const int vl = i / N, n = i - vl * N, v = vb0 + vl;
                    if (v >= nv) break;
                    const int g = cov_c[v / G], m = v % G, slot = g * G + m;
                    const int piece = b - pb0[g];
                    float sum = 0.0f;
                    for (int w2 = 0; w2 < RW; ++w2) sum += red[(w2 * GU_VB + vl) * red_ld + n];
                    if (tpart) {
                        float ts = 0.0f;
                        if (slot < n_slots)
                            for (int j = piece; j < t_split; j += n_pieces) ts += tpart[((int64_t)j * n_slots + slot) * N + n];
                        sum = fmaf(slot < n_slots ? sa.scale[slot] : 0.0f, sum, ts);
                    }
                    part[(((int64_t)g * n_pieces + piece) * G + m) * N + n] = sum;
                }
            }
            // pieces past a group's last block: zero (+ the folded theta partials), written with the group's last block
            for (int gi = 0; gi < ng; ++gi) {
                const int g = cov_c[gi];
                if (pb1[g] != b) continue;
                for (int piece = b - pb0[g] + 1; piece < n_pieces; ++piece)
                    for (int i = tid; i < G * N; i += GB_CONSUMERS) {
                        const int m = i / N, n = i - m * N, slot = g * G + m;
                        float ts = 0.0f;
                        if (tpart && slot < n_slots)
                            for (int j = piece; j < t_split; j += n_pieces) ts += tpart[((int64_t)j * n_slots + slot) * N + n];
                        part[(((int64_t)g * n_pieces + piece) * G + m) * N + n] = ts;
                    }
            }
            named_bar_sync(1, GB_CONSUMERS);                               // barrier E: red[], xs[], cov_c[] reusable
        }
    }
}

int dne_gemv_pieces(int K) { return (K + 1 + GU_BLK - 1) / GU_BLK + 1; }

int dne_launch_gemv_union(const SlotArgs& sa, const GemvSrc& src, int G, const float* X, int64_t x_slot_stride, int K,
                          int N, int n_pieces, int n_slots, float* part, int sm_count, cudaStream_t st,
                          const float* fold_theta, int fold_n_split) {
    // shape cover: 4 | N, N/4 divides 256, one stage = GB_RPR rows per reader, at most GU_BLK / 4 rows per stage
    if (N % 4 != 0 || N < GU_MIN_N || N * 4 > GB_STAGE_BYTES || (GB_CONSUMERS % (N / 4)) != 0) return DNE_ERR_UNSUP;
    const int RW = GB_CONSUMERS / (N / 4);
    if (GB_RPR * RW * N * 4 != GB_STAGE_BYTES || n_pieces != dne_gemv_pieces(K) || (G != 1 && G != 2)) return DNE_ERR_UNSUP;
    const int n_groups = (n_slots + G - 1) / G;
    if (n_groups <= 0) return 0;
    // shared memory: static (xs + barriers) + ring + plan; as many ring stages as fit next to the chosen CTAs per SM
    const size_t static_smem = (size_t)GU_XS_FLOATS * 4 + 1024;
    const size_t plan = (size_t)n_groups * GU_PLAN_BYTES_PER_GROUP + 128;
    const size_t per_sm = 227 * 1024;
    int cps = g_dne_gemv_ctas_per_sm, n_stages = 0;
    for (; cps >= 1; --cps) {
        const size_t budget = per_sm / cps - 1024;
        n_stages = budget > static_smem + plan ? (int)((budget - static_smem - plan) / GB_STAGE_BYTES) : 0;
        if (n_stages > g_dne_gemv_stages) n_stages = g_dne_gemv_stages;
        if (n_stages >= 2) break;
    }
    if (cps < 1) return DNE_ERR_UNSUP;
    const size_t smem = (size_t)n_stages * GB_STAGE_BYTES + plan;
    int grid = cps * sm_count;
    if (g_dne_gemv_grid > 0 && grid > g_dne_gemv_grid) grid = g_dne_gemv_grid;
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_done_dev[64][3] = {};                        // per device: one process may drive several GPUs
    bool* attr_done = attr_done_dev[dev < 64 ? dev : 63];
    auto launch = [&](auto kern) -> int {
        if (!attr_done[G]) {
            cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(per_sm - static_smem - 1024)) != cudaSuccess)
                return DNE_ERR_CUDA;
            attr_done[G] = true;
        }
        if (dne_launch_chain(kern, dim3(grid), dim3(GB_THREADS), smem, st, true, sa, src, X, x_slot_stride, K, N, n_pieces,
                             n_groups, n_slots, part, n_stages, fold_theta, fold_theta ? fold_n_split : 0) != cudaSuccess)
            return DNE_ERR_CUDA;
        return 0;
    };
    return G == 2 ? launch(gemv_union_kernel<2>) : launch(gemv_union_kernel<1>);
}
