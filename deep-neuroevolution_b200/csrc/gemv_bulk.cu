// gemv_bulk.cu -- the HBM-bound noise GEMV with a TMA bulk-copy (cp.async.bulk) shared-memory pipeline.
//
// Same math and partial layout as dense_noise_gemv_kernel (forward_kernels.cu):
//     part[group][chunk][g][n] = sum_{k in chunk} x_g[k] * W[k][n],   W = slab[E0 + k*N + n], E0 arbitrary alignment
// but the weight rows do not pass through registers on their way in: a producer warp streams the 16B-ALIGNED superset
// of the chunk (contiguous RB-row blocks, one cp.async.bulk each) into a ring of shared-memory stages, completion
// tracked by mbarriers (full / empty), and 8 consumer warps read the rows back with conflict-free LDS.128.  The bytes
// in flight are STAGES x 16 KB per CTA regardless of register allocation (the plain-LDG kernel is limited by how many
// loads ptxas keeps in flight: measured 64 % of HBM peak; Little's law wants > 44 KB per SM).
// CTAs are persistent: a static round-robin over (group, chunk) work items, the ring runs across item boundaries.
//
// Alignment trick (see forward_kernels.cu): thread t always owns aligned column quad q = 4t..4t+3.  Element (r, q) of
// the aligned stream is weight (k = r, n = q - a) for q >= a and (k = r - 1, n = N + q - a) for q < a, a = E0 & 3.
// Only quad 0 has the second kind; it keeps a second accumulator fed from the SAME staged rows with multiplier x[r-1].
#include "common.cuh"
#include "forward.cuh"
#include "epilogue.cuh"
#include "wgmma.cuh"

using namespace wg;

int g_dne_gemv_bulk = 1;
int g_dne_gemv_ctas_per_sm = 2;
int g_dne_gemv_balance = 1;          // choose the grid size that balances the round-robin item deal (dne_set_option("gemv_balance"))
int g_dne_gemv_grid = 0;             // > 0: cap on the number of CTAs (dne_set_option("gemv_grid")): leaves whole SMs to another stream
int g_dne_gemv_stages = 6;           // shared-memory ring depth (2..GB_STAGES), dne_set_option("gemv_stages")
int g_dne_gemv_prefetch = 0;         // L2 prefetch distance in stages (cp.async.bulk.prefetch.L2), dne_set_option("gemv_prefetch")

constexpr int GB_CONSUMERS = 256;
constexpr int GB_THREADS = GB_CONSUMERS + 32;      // + one producer warp
constexpr int GB_STAGES = 8;                       // maximum ring depth (barrier arrays); the launch picks n_stages <= this
constexpr int GB_STAGE_BYTES = 16384;
constexpr int GB_RPR = 4;                          // rows per reader per stage: (16384/4N) / (256/(N/4)) = 4 for every N
constexpr int GB_FOLD_O = 4, GB_FOLD_S = 3;         // fold: outputs per consumer thread (G*N <= 1024), theta splits per chunk
constexpr int GB_MAX_ROWS = 512;                   // rows per work item (x staging buffer)

template <int G>
__global__ void __launch_bounds__(GB_THREADS)
gemv_bulk_kernel(SlotArgs sa, GemvSrc src, const float* __restrict__ X, int64_t x_slot_stride, int K, int N,
                 int rows_per_chunk, int n_chunks, int n_groups, float* __restrict__ part, int n_stages, int pf_dist,
                 const float* __restrict__ tpart, int t_split, int n_slots) {
    // tpart != nullptr ("fold"): the shared-theta GEMM's split-K partials [t_split][n_slots][N] are folded into this
    // kernel's output, part[group][chunk][g][n] = s_g * (noise partial of the chunk) + sum_{j = chunk (mod n_chunks)} tpart[j]:
    // the combine kernel then adds n_chunks values per output instead of n_chunks + t_split (its latency-bound L2 round
    // trips were 5 of 7 for the theta partials).  The <= GB_FOLD_S loads per output are issued at the top of the item and
    // consumed after its last stage.  Fixed summation order: deterministic.
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 127) & ~(uintptr_t)127);
    float* stage_base = reinterpret_cast<float*>(smem);
    float* red = reinterpret_cast<float*>(smem + n_stages * GB_STAGE_BYTES);        // [RW][G][N+4]
    __shared__ uint64_t full_bar[GB_STAGES], empty_bar[GB_STAGES];
    __shared__ float xs[G][GB_MAX_ROWS + 8];           // xs[g][1 + r] = x_g[k_beg + r];  xs[g][0] = x_g[k_beg - 1]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int NQ = N >> 2;
    const int RW = GB_CONSUMERS / NQ;                  // row readers per stage
    const int RB = GB_RPR * RW;                        // rows per stage
    const int n_items = n_groups * n_chunks;
    pdl_trigger();                                     // common.cuh: PDL chain of the tick

    if (tid == 0) {
        for (int s = 0; s < n_stages; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], GB_CONSUMERS / 32);
        }
        fence_mbar_init();
    }
    __syncthreads();

    auto item_active = [&](int item) {
        const int slot0 = (item / n_chunks) * G;
        bool any = false;
#pragma unroll
        for (int g = 0; g < G; ++g) any = any || slot_active(sa, slot0 + g);
        return any;
    };
    auto item_base = [&](int item, int& k_beg, int& rows, int& a) -> const float* {
        const int group = item / n_chunks, chunk = item % n_chunks;
        const int slot0 = group * G;
        k_beg = chunk * rows_per_chunk;
        rows = min(K, k_beg + rows_per_chunk) - k_beg;
        const int64_t E0 = (src.idx64 ? src.idx64[slot0] : (src.idx32 ? (int64_t)src.idx32[slot0] * src.mul : 0)) + src.off;
        a = (int)(E0 & 3);
        return src.base + (E0 - a) + (int64_t)k_beg * N;       // 16B-aligned start of the chunk's aligned rows
    };

    if (warp == GB_CONSUMERS / 32) {
        // ===================== producer warp (one elected lane) =====================
        if (lane == 0) {
            // L2 prefetch cursor: runs pf_dist stage-blocks ahead of the copy cursor (across work-item boundaries), so the
            // HBM latency is covered by L2 and the shared-memory ring only has to cover the L2 -> SM latency.  That lets a
            // shallow ring (1 CTA/SM, <= 64 KB) stream at HBM rate and leaves shared memory for a co-resident conv CTA.
            int p_item = blockIdx.x - gridDim.x, p_r0 = 0, p_rows = 0;
            const float* p_base = nullptr;
            auto p_next_item = [&]() {
                do { p_item += gridDim.x; } while (p_item < n_items && !item_active(p_item));
                if (p_item < n_items) { int kb, a_; p_base = item_base(p_item, kb, p_rows, a_); p_r0 = 0; }
            };
            auto p_step = [&]() {                                // prefetch the cursor's block, then advance it
                if (p_item >= n_items) return;
                bulk_prefetch_l2(p_base + (int64_t)p_r0 * N, (uint32_t)min(RB, p_rows - p_r0) * N * 4);
                p_r0 += RB;
                if (p_r0 >= p_rows) p_next_item();
            };
            if (pf_dist > 0) {
                p_next_item();
                for (int d = 0; d < pf_dist; ++d) p_step();
            }
            uint32_t it = 0;
            for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
                if (!item_active(item)) continue;
                int k_beg, rows, a;
                const float* base = item_base(item, k_beg, rows, a);
                for (int r0 = 0; r0 < rows; r0 += RB, ++it) {
                    if (pf_dist > 0) p_step();
                    const int s = it % n_stages;
                    mbar_wait(&empty_bar[s], ((it / n_stages) & 1) ^ 1);
                    const uint32_t bytes = (uint32_t)min(RB, rows - r0) * N * 4;
                    mbar_arrive_expect_tx(&full_bar[s], bytes);
                    bulk_g2s(stage_base + (size_t)s * (GB_STAGE_BYTES / 4), base + (int64_t)r0 * N, bytes, &full_bar[s]);
                }
            }
        }
        return;
    }

    // ===================== consumer warps =====================
    // (the producer above streams weight rows -- written before the tick -- without waiting; X and part need the chain)
    pdl_wait();
    const int t = tid % NQ, rw = tid / NQ;
    const int red_ld = N + 4;
    uint32_t it = 0;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        if (!item_active(item)) continue;
        const int group = item / n_chunks, chunk = item % n_chunks;
        const int slot0 = group * G;
        int k_beg, rows, a;
        const float* base = item_base(item, k_beg, rows, a);

        float tv[GB_FOLD_O][GB_FOLD_S];
        if (tpart) {
#pragma unroll
            for (int o = 0; o < GB_FOLD_O; ++o) {
                const int i = tid + o * GB_CONSUMERS;
                const int g = i / N, n = i - g * N;
                const bool ok = i < G * N && slot0 + g < n_slots;
#pragma unroll
                for (int k = 0; k < GB_FOLD_S; ++k) {
                    const int j = chunk + k * n_chunks;
                    // volatile asm: the load is issued HERE (the compiler otherwise sinks it to its use after the streaming
                    // loop and exposes one L2 round trip per item: measured +8 us per GEMV launch)
                    float v = 0.0f;
                    if (ok && j < t_split)
                        asm volatile("ld.global.cg.f32 %0, [%1];" : "=f"(v) : "l"(tpart + ((int64_t)j * n_slots + slot0 + g) * N + n) : "memory");
                    tv[o][k] = v;
                }
            }
        }
        // stage x_g[k_beg-1 .. k_beg+rows) (the previous item's readers are past their last xs read: barrier C below)
        for (int i = tid; i < G * (rows + 1); i += GB_CONSUMERS) {
            const int g = i / (rows + 1), r = i % (rows + 1);
            const int k = k_beg - 1 + r;
            xs[g][r] = (k >= 0) ? X[(int64_t)(slot0 + g) * x_slot_stride + k] : 0.0f;
        }
        named_bar_sync(1, GB_CONSUMERS);                                   // barrier A

        float acc[G][4], wrap[G][4];
#pragma unroll
        for (int g = 0; g < G; ++g)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[g][c] = wrap[g][c] = 0.0f;
        const bool do_wrap = (t == 0) && (a != 0);

        for (int r0 = 0; r0 < rows; r0 += RB, ++it) {
            const int s = it % n_stages;
            const int nr = min(RB, rows - r0);
            const int rl0 = rw * GB_RPR;                 // this reader's first row inside the stage (contiguous rows)
            // x multipliers: xm[g][j] = x[r0+rl0+j] (row itself), xm[g][-1 -> index 0] = x[r0+rl0-1] (wrap of the first row)
            float xm[G][GB_RPR + 1];
#pragma unroll
            for (int g = 0; g < G; ++g)
#pragma unroll
                for (int j = 0; j <= GB_RPR; ++j) xm[g][j] = xs[g][r0 + rl0 + j];        // xs index = 1 + (row - 1)
            mbar_wait(&full_bar[s], (it / n_stages) & 1);
            // explicit ld.shared (a C++ pointer into the re-aligned dynamic smem compiles to generic LD.E)
            const uint32_t rows_a = wg::smem_u32(stage_base) + s * GB_STAGE_BYTES + (rl0 * NQ + t) * 16;
            if (nr == RB) {
                float4 v[GB_RPR];
#pragma unroll
                for (int j = 0; j < GB_RPR; ++j) v[j] = wg::lds128(rows_a + j * NQ * 16);
#pragma unroll
                for (int j = 0; j < GB_RPR; ++j)
#pragma unroll
                    for (int g = 0; g < G; ++g) {
                        acc[g][0] = fmaf(xm[g][j + 1], v[j].x, acc[g][0]);
                        acc[g][1] = fmaf(xm[g][j + 1], v[j].y, acc[g][1]);
                        acc[g][2] = fmaf(xm[g][j + 1], v[j].z, acc[g][2]);
                        acc[g][3] = fmaf(xm[g][j + 1], v[j].w, acc[g][3]);
                    }
                if (do_wrap) {
#pragma unroll
                    for (int j = 0; j < GB_RPR; ++j)
#pragma unroll
                        for (int g = 0; g < G; ++g) {     // aligned row r carries weight row r-1 in its columns q < a
                            const float xp = (r0 + rl0 + j >= 1) ? xm[g][j] : 0.0f;
                            wrap[g][0] = fmaf(xp, v[j].x, wrap[g][0]);
                            wrap[g][1] = fmaf(xp, v[j].y, wrap[g][1]);
                            wrap[g][2] = fmaf(xp, v[j].z, wrap[g][2]);
                            wrap[g][3] = fmaf(xp, v[j].w, wrap[g][3]);
                        }
                }
            } else {
                for (int j = 0; j < GB_RPR; ++j) {
                    if (rl0 + j < nr) {
                        const float4 v = wg::lds128(rows_a + j * NQ * 16);
#pragma unroll
                        for (int g = 0; g < G; ++g) {
                            acc[g][0] = fmaf(xm[g][j + 1], v.x, acc[g][0]);
                            acc[g][1] = fmaf(xm[g][j + 1], v.y, acc[g][1]);
                            acc[g][2] = fmaf(xm[g][j + 1], v.z, acc[g][2]);
                            acc[g][3] = fmaf(xm[g][j + 1], v.w, acc[g][3]);
                            if (do_wrap && (r0 + rl0 + j >= 1)) {
                                wrap[g][0] = fmaf(xm[g][j], v.x, wrap[g][0]);
                                wrap[g][1] = fmaf(xm[g][j], v.y, wrap[g][1]);
                                wrap[g][2] = fmaf(xm[g][j], v.z, wrap[g][2]);
                                wrap[g][3] = fmaf(xm[g][j], v.w, wrap[g][3]);
                            }
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty_bar[s]);           // this warp is done reading stage s
        }
        // the chunk's last weight row (k = rows-1) wraps into aligned row `rows`, the first row of the NEXT chunk:
        // one 16-byte load per item
        if (do_wrap && rw == 0) {
            const float4 v = ldg_stream_f4(base + (int64_t)rows * N);
#pragma unroll
            for (int g = 0; g < G; ++g) {
                const float x = xs[g][rows];                      // x[k_beg + rows - 1]
                wrap[g][0] = fmaf(x, v.x, wrap[g][0]);
                wrap[g][1] = fmaf(x, v.y, wrap[g][1]);
                wrap[g][2] = fmaf(x, v.z, wrap[g][2]);
                wrap[g][3] = fmaf(x, v.w, wrap[g][3]);
            }
        }
        // cross-reader reduction in fixed order, then this item's partial [G][N]
#pragma unroll
        for (int g = 0; g < G; ++g) {
            float* row = red + (rw * G + g) * red_ld;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const int q = 4 * t + c;
                if (q >= a) row[q - a] = acc[g][c];
            }
            if (t == 0) {
#pragma unroll
                for (int c = 0; c < 4; ++c)
                    if (c < a) row[N + c - a] = wrap[g][c];
            }
        }
        named_bar_sync(1, GB_CONSUMERS);                                   // barrier B
        float* out = part + ((int64_t)group * n_chunks + chunk) * G * N;
        if (tpart) {
#pragma unroll
            for (int o = 0; o < GB_FOLD_O; ++o) {
                const int i = tid + o * GB_CONSUMERS;
                if (i < G * N) {
                    const int g = i / N, n = i - g * N;
                    float sum = 0.0f;
                    for (int w = 0; w < RW; ++w) sum += red[(w * G + g) * red_ld + n];
                    float ts = tv[o][0];
#pragma unroll
                    for (int k = 1; k < GB_FOLD_S; ++k) ts += tv[o][k];
                    out[i] = fmaf(slot0 + g < n_slots ? sa.scale[slot0 + g] : 0.0f, sum, ts);
                }
            }
        } else {
            for (int i = tid; i < G * N; i += GB_CONSUMERS) {
                const int g = i / N, n = i % N;
                float sum = 0.0f;
                for (int w = 0; w < RW; ++w) sum += red[(w * G + g) * red_ld + n];
                out[i] = sum;
            }
        }
        named_bar_sync(1, GB_CONSUMERS);                                   // barrier C: red[] and xs[] reusable
    }
}

bool dne_gemv_bulk_can_fold(int G, int N, int n_chunks, int n_split) {
    return G * N <= GB_FOLD_O * GB_CONSUMERS && n_split >= 1 && n_split <= GB_FOLD_S * n_chunks;
}

int dne_launch_gemv_bulk(const SlotArgs& sa, const GemvSrc& src, int G, const float* X, int64_t x_slot_stride, int K,
                         int N, int rows_per_chunk, int n_chunks, int n_slots, float* part, int sm_count,
                         cudaStream_t st, const float* fold_theta, int fold_n_split) {
    if (fold_theta && !dne_gemv_bulk_can_fold(G, N, n_chunks, fold_n_split)) return DNE_ERR_UNSUP;
    // shape cover: 4 | N, N/4 divides 256, one stage = GB_RPR rows per reader
    if (N % 4 != 0 || N * 4 > GB_STAGE_BYTES || (GB_CONSUMERS % (N / 4)) != 0) return DNE_ERR_UNSUP;
    const int RW = GB_CONSUMERS / (N / 4);
    if (GB_RPR * RW * N * 4 != GB_STAGE_BYTES || rows_per_chunk > GB_MAX_ROWS) return DNE_ERR_UNSUP;
    const int n_groups = (n_slots + G - 1) / G;
    const int n_stages = g_dne_gemv_stages;
    const size_t smem = (size_t)n_stages * GB_STAGE_BYTES + (size_t)RW * G * (N + 4) * sizeof(float) + 128;
    const int n_items = n_groups * n_chunks;
    int grid = g_dne_gemv_ctas_per_sm * sm_count;
    if (g_dne_gemv_grid > 0 && grid > g_dne_gemv_grid) grid = g_dne_gemv_grid;
    if (grid > n_items) grid = n_items;
    else if (g_dne_gemv_balance) {
        // the items are dealt round-robin: pick the grid size in [7/8 * grid, grid] that leaves the fewest idle item slots in
        // the last round (62 pairs x 32 chunks on 296 CTAs: 7 rounds with 88 idle slots; on 284 CTAs: 4 idle slots)
        int best = grid;
        long best_waste = (long)((n_items + grid - 1) / grid) * grid - n_items;
        for (int g = grid - 1; g >= grid - grid / 8 && best_waste > 0; --g) {
            const long waste = (long)((n_items + g - 1) / g) * g - n_items;
            if (waste < best_waste) { best_waste = waste; best = g; }
        }
        grid = best;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    static bool attr_done_dev[64][3] = {};                        // per device: one process may drive several GPUs
    bool* attr_done = attr_done_dev[dev < 64 ? dev : 63];
    if (G == 2) {
        if (!attr_done[2]) {
            cudaFuncSetAttribute(gemv_bulk_kernel<2>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            if (cudaFuncSetAttribute(gemv_bulk_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (GB_STAGES * 16 + 12) * 1024) != cudaSuccess)
                return DNE_ERR_CUDA;
            attr_done[2] = true;
        }
        if (dne_launch_chain(gemv_bulk_kernel<2>, dim3(grid), dim3(GB_THREADS), smem, st, true, sa, src, X, x_slot_stride, K, N,
                             rows_per_chunk, n_chunks, n_groups, part, n_stages, g_dne_gemv_prefetch, fold_theta, fold_n_split, n_slots) != cudaSuccess)
            return DNE_ERR_CUDA;
    } else {
        if (!attr_done[1]) {
            cudaFuncSetAttribute(gemv_bulk_kernel<1>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            if (cudaFuncSetAttribute(gemv_bulk_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (GB_STAGES * 16 + 12) * 1024) != cudaSuccess)
                return DNE_ERR_CUDA;
            attr_done[1] = true;
        }
        if (dne_launch_chain(gemv_bulk_kernel<1>, dim3(grid), dim3(GB_THREADS), smem, st, true, sa, src, X, x_slot_stride, K, N,
                             rows_per_chunk, n_chunks, n_groups, part, n_stages, g_dne_gemv_prefetch, fold_theta, fold_n_split, n_slots) != cudaSuccess)
            return DNE_ERR_CUDA;
    }
    return 0;
}
