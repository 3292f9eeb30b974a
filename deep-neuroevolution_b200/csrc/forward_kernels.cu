// forward_kernels.cu -- fused perturb + batched per-member policy forward + action select.
//
// Replaces, for all env slots of one tick at once (reference: one sess.run at batch 1 per worker step):
//   es_distributed/es.py:412-419          v = sigma*noise[idx:idx+P]; set_trainable_flat(theta +/- v)
//   es_distributed/policies.py:319-330    ESAtariPolicy forward (conv/BN/relu, fc, argmax)       :449-459 GAAtariPolicy
//   es_distributed/policies.py:150-162    MujocoPolicy forward (ob-norm, tanh MLP)
//   gpu_implementation/neuroevolution/models/dqn.py:25-47 + base.py:54-99   Model / LargeModel
//   gpu_implementation/gym_tensorflow/ops/indexedmatmul.cpp:148-213          per-slot batched matmul
//
// Design (DESIGN.md "forward"): a member's weights are theta + s*noise[idx:idx+P] and are NEVER written to
// HBM.  Convolutions (small weights, large reuse) build the member's weight tile in shared memory and run an
// implicit GEMM.  Dense layers (97.8% of the weight bytes, M=1 per member) are algebraically split:
//     x.(theta_w + s*N) = x.theta_w  +  s * (x.N)
// x.theta_w over all slots is one ordinary GEMM with a SHARED B operand (theta stays L2 resident);
// x.N is a streaming GEMV over the member's noise slice, the HBM-bound part, and an antithetic pair
// (+s, -s on the same slice) reads the slice ONCE for both members.
#include "common.cuh"
#include "forward.cuh"
#include "epilogue.cuh"

// ---------------------------------------------------------------------------------------------------
// Convolution as implicit GEMM, one member per blockIdx.y, BM output positions per CTA.
//   A[m][k] = in[oy*S-PAD+ky][ox*S-PAD+kx][ci]   (TF SAME, NHWC; k = (ky,kx,ci), HWIO flat order: tf_util.py:135)
//   B[k][n] = theta_w[k*COUT+n] + s*noise[idx+off_w+k*COUT+n]     built in shared memory per k-tile
// fp32 SIMT register tile TM x TN.  (The wgmma version of this contraction replaces this kernel.)
// ---------------------------------------------------------------------------------------------------
constexpr int CONV_BK = 16;

template <int CIN, int COUT, int KS, int STRIDE, int HIN, int HOUT, int PAD, bool IN_U8, int BM, int TM, int TN>
__global__ void __launch_bounds__((BM / TM) * (COUT / TN))
conv_kernel(SlotArgs sa, int64_t off_w, LayerEpi epi, const void* __restrict__ in_base, int64_t in_slot_stride,
            int64_t in_img_stride, float* __restrict__ out_base, int64_t out_slot_stride, int64_t out_img_stride) {
    constexpr int THREADS = (BM / TM) * (COUT / TN);
    constexpr int M = HOUT * HOUT;
    constexpr int K = KS * KS * CIN;
    constexpr int BK = CONV_BK;
    static_assert(K % BK == 0 && CIN % 4 == 0 && TM % 4 == 0, "tile constraints");
    constexpr int A_UNITS = BM * BK / 4;                       // float4 (4 consecutive ci) units
    constexpr int A_PER_THREAD = (A_UNITS + THREADS - 1) / THREADS;
    constexpr int B_ELEMS = BK * COUT;
    constexpr int B_PER_THREAD = (B_ELEMS + THREADS - 1) / THREADS;

    const int slot = blockIdx.y;
    if (!slot_active(sa, slot)) return;
    const int img = blockIdx.z;                                // reference-batch image (VBN pass) or 0
    const int m_tile = blockIdx.x * BM;
    const int tid = threadIdx.x;
    const int tx = tid % (COUT / TN), ty = tid / (COUT / TN);

    __shared__ __align__(16) float As[BK][BM];
    __shared__ __align__(16) float Bs[BK][COUT];

    const float* th = slot_theta(sa, slot);
    const int64_t idx = sa.noise_idx[slot];
    const float s = sa.scale[slot];
    const float* nz = sa.noise + idx + off_w;
    const float* tw = th + off_w;

    // per-thread A gather coordinates (fixed across k-tiles)
    int a_iy0[A_PER_THREAD], a_ix0[A_PER_THREAD];
    bool a_ok[A_PER_THREAD];
#pragma unroll
    for (int i = 0; i < A_PER_THREAD; ++i) {
        const int u = tid + i * THREADS;
        const int m = m_tile + (u % BM);
        a_ok[i] = (u < A_UNITS) && (m < M);
        const int oy = m / HOUT, ox = m % HOUT;
        a_iy0[i] = oy * STRIDE - PAD;
        a_ix0[i] = ox * STRIDE - PAD;
    }
    const uint8_t* in_u8 = nullptr;
    const float* in_f = nullptr;
    if (IN_U8) in_u8 = (const uint8_t*)in_base + slot * in_slot_stride + img * in_img_stride;
    else in_f = (const float*)in_base + slot * in_slot_stride + img * in_img_stride;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.0f;

    for (int k0 = 0; k0 < K; k0 += BK) {
        // ---- A tile: im2col gather, 4 consecutive input channels per unit ----
#pragma unroll
        for (int i = 0; i < A_PER_THREAD; ++i) {
            const int u = tid + i * THREADS;
            if (u < A_UNITS) {
                const int ml = u % BM, kq = u / BM;
                const int k = k0 + 4 * kq;
                const int ci = k % CIN, t = k / CIN;
                const int kx = t % KS, ky = t / KS;
                const int iy = a_iy0[i] + ky, ix = a_ix0[i] + kx;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (a_ok[i] && iy >= 0 && iy < HIN && ix >= 0 && ix < HIN) {
                    const int e = (iy * HIN + ix) * CIN + ci;
                    if (IN_U8) {
                        const uchar4 q = *reinterpret_cast<const uchar4*>(in_u8 + e);
                        v.x = __fdiv_rn((float)q.x, 255.0f);     // atari_wrappers.py:186
                        v.y = __fdiv_rn((float)q.y, 255.0f);
                        v.z = __fdiv_rn((float)q.z, 255.0f);
                        v.w = __fdiv_rn((float)q.w, 255.0f);
                    } else {
                        v = *reinterpret_cast<const float4*>(in_f + e);
                    }
                }
                As[4 * kq + 0][ml] = v.x;
                As[4 * kq + 1][ml] = v.y;
                As[4 * kq + 2][ml] = v.z;
                As[4 * kq + 3][ml] = v.w;
            }
        }
        // ---- B tile: member weights, contiguous BK*COUT run of the flat vector ----
#pragma unroll
        for (int i = 0; i < B_PER_THREAD; ++i) {
            const int e = tid + i * THREADS;
            if (e < B_ELEMS) {
                const int64_t f = (int64_t)k0 * COUT + e;
                (&Bs[0][0])[e] = perturbed(tw[f], s, nz[f]);
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TN];
#pragma unroll
            for (int i = 0; i < TM; i += 4) {
                const float4 q = *reinterpret_cast<const float4*>(&As[k][ty * TM + i]);
                a[i] = q.x; a[i + 1] = q.y; a[i + 2] = q.z; a[i + 3] = q.w;
            }
#pragma unroll
            for (int j = 0; j < TN; ++j) b[j] = Bs[k][tx * TN + j];
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    // ---- epilogue: bias (+BN) + activation, NHWC store ----
    float* out = out_base + slot * out_slot_stride + img * out_img_stride;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
        const int n = tx * TN + j;
        const ChanEpi ce = make_chan_epi(sa, epi, slot, COUT, n, th, idx, s);
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            const int m = m_tile + ty * TM + i;
            if (m < M) out[(int64_t)m * COUT + n] = ce.apply(acc[i][j]);
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Dense layer, shared-theta part:  Ypart[split][m][n] = sum_{k in split} X[m][k] * theta_w[k][n]
// Ordinary fp32 SIMT GEMM, 128x128x16 tiles, 8x8 per thread, split-K with deterministic partials.
// ---------------------------------------------------------------------------------------------------
constexpr int DG_BM = 128, DG_BN = 128, DG_BK = 16, DG_T = 8, DG_THREADS = 256;

__global__ void __launch_bounds__(DG_THREADS)
dense_theta_gemm_kernel(const float* __restrict__ X, int M, int K, int N, const float* __restrict__ W,
                        int k_per_split, float* __restrict__ part) {
    __shared__ __align__(16) float As[DG_BK][DG_BM];
    __shared__ __align__(16) float Bs[DG_BK][DG_BN];
    const int tid = threadIdx.x;
    const int tx = tid % (DG_BN / DG_T), ty = tid / (DG_BN / DG_T);
    const int m0 = blockIdx.y * DG_BM, n0 = blockIdx.x * DG_BN;
    const int split = blockIdx.z;
    const int kbeg = split * k_per_split, kend = min(K, kbeg + k_per_split);

    float acc[DG_T][DG_T];
#pragma unroll
    for (int i = 0; i < DG_T; ++i)
#pragma unroll
        for (int j = 0; j < DG_T; ++j) acc[i][j] = 0.0f;

    for (int k0 = kbeg; k0 < kend; k0 += DG_BK) {
        // A: 128 rows x 16 k = 512 float4 units (K % 4 == 0 guaranteed by the caller)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int u = tid + i * DG_THREADS;
            const int ml = u % DG_BM, kq = u / DG_BM;
            const int m = m0 + ml, k = k0 + 4 * kq;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < M && k < kend) v = *reinterpret_cast<const float4*>(X + (int64_t)m * K + k);
            As[4 * kq + 0][ml] = v.x;
            As[4 * kq + 1][ml] = v.y;
            As[4 * kq + 2][ml] = v.z;
            As[4 * kq + 3][ml] = v.w;
        }
        // B: 16 x 128 scalars (no alignment assumption on off_w)
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int e = tid + i * DG_THREADS;
            const int kl = e / DG_BN, nl = e % DG_BN;
            const int k = k0 + kl, n = n0 + nl;
            Bs[kl][nl] = (k < kend && n < N) ? W[(int64_t)k * N + n] : 0.0f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < DG_BK; ++k) {
            float a[DG_T], b[DG_T];
            const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * DG_T]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * DG_T + 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][tx * DG_T]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[k][tx * DG_T + 4]);
            a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
            b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
#pragma unroll
            for (int i = 0; i < DG_T; ++i)
#pragma unroll
                for (int j = 0; j < DG_T; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* P = part + (int64_t)split * M * N;
#pragma unroll
    for (int i = 0; i < DG_T; ++i) {
        const int m = m0 + ty * DG_T + i;
        if (m >= M) continue;
#pragma unroll
        for (int j = 0; j < DG_T; ++j) {
            const int n = n0 + tx * DG_T + j;
            if (n < N) P[(int64_t)m * N + n] = acc[i][j];
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Dense layer, noise part (THE HBM-bound kernel):  a_g[n] = sum_k x_g[k] * noise[idx + off_w + k*N + n]
// for the G members of a group that share one noise slice (G=2: antithetic pair, slice read once).
//
// The slice starts at an arbitrary element offset, so [idx+off_w, ...) is generally not 16-byte aligned and
// TMA / vector loads cannot address it directly.  We stream the 16B-ALIGNED superset instead: with
// E0 = idx+off_w, a = E0 & 3, E0' = E0 - a, "aligned row" r is slab[E0' + r*N, +N) and thread t always loads
// the same aligned float4 column q = 4t..4t+3 of every row.  Element (r, q) is weight (k = r, n = q - a) if
// q >= a, else (k = r-1, n = N + q - a).  So every thread accumulates acc[c] += x[r] * S[r][4t+c] with fixed
// columns, and only thread 0 keeps a second accumulator with multiplier x[r-1] for its (at most 3) wrapped
// columns.  blockDim = (N/4) * RW: RW row-interleaved readers per column quad, reduced through shared memory.
// Grid = (chunks of the K rows, groups).  Partials are written per chunk (deterministic, no atomics).
// ---------------------------------------------------------------------------------------------------
// The same kernel also streams the PARENT weights for GA slots (theta rows selected per slot): the "slab" is then
// the theta matrix and the per-group element offset is theta_idx * P (GemvSrc).

template <int G, int U>
__global__ void __launch_bounds__(256)
dense_noise_gemv_kernel(SlotArgs sa, GemvSrc src, const float* __restrict__ X, int64_t x_slot_stride, int K,
                        int N, int rows_per_chunk, float* __restrict__ part) {
    extern __shared__ float smem[];
    const int group = blockIdx.y, chunk = blockIdx.x, n_chunks = gridDim.x;
    const int slot0 = group * G;
    bool any = false;
#pragma unroll
    for (int g = 0; g < G; ++g) any = any || slot_active(sa, slot0 + g);
    if (!any) return;

    const int NQ = N >> 2;                 // float4 columns
    const int RW = blockDim.x / NQ;        // row readers
    const int t = threadIdx.x % NQ, rw = threadIdx.x / NQ;
    const int k_beg = chunk * rows_per_chunk;
    const int k_end = min(K, k_beg + rows_per_chunk);
    const int rows = k_end - k_beg;

    // stage x[k_beg-1 .. k_end) for the G members: xs[g][0] = x[k_beg-1] (0 if k_beg == 0)
    float* xs = smem;                                   // [G][rows_per_chunk + 1]
    const int xs_ld = rows_per_chunk + 1;
    for (int i = threadIdx.x; i < G * (rows + 1); i += blockDim.x) {
        const int g = i / (rows + 1), r = i % (rows + 1);
        const int k = k_beg - 1 + r;
        xs[g * xs_ld + r] = (k >= 0) ? X[(int64_t)(slot0 + g) * x_slot_stride + k] : 0.0f;
    }
    __syncthreads();

    const int64_t E0 = (src.idx64 ? src.idx64[slot0] : (src.idx32 ? (int64_t)src.idx32[slot0] * src.mul : 0)) + src.off;
    const int a = (int)(E0 & 3);
    const float* S = src.base + (E0 - a) + 4 * t;       // aligned column quad of this thread

    float acc[G][4];
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[g][c] = 0.0f;

    int r = rw;   // row index local to the chunk, this reader takes rows rw, rw+RW, ...
    for (; r + (U - 1) * RW < rows; r += U * RW) {
        float4 v[U];
        static_assert(U == 8, "batched load helper is written for 8 rows");
        ldg_stream_f4x8(S + (int64_t)(k_beg + r) * N, (int64_t)RW * N, v);
#pragma unroll
        for (int u = 0; u < U; ++u) {
#pragma unroll
            for (int g = 0; g < G; ++g) {
                const float x = xs[g * xs_ld + 1 + r + u * RW];
                acc[g][0] = fmaf(x, v[u].x, acc[g][0]);
                acc[g][1] = fmaf(x, v[u].y, acc[g][1]);
                acc[g][2] = fmaf(x, v[u].z, acc[g][2]);
                acc[g][3] = fmaf(x, v[u].w, acc[g][3]);
            }
        }
    }
    for (; r < rows; r += RW) {
        const float4 v = ldg_stream_f4(S + (int64_t)(k_beg + r) * N);
#pragma unroll
        for (int g = 0; g < G; ++g) {
            const float x = xs[g * xs_ld + 1 + r];
            acc[g][0] = fmaf(x, v.x, acc[g][0]);
            acc[g][1] = fmaf(x, v.y, acc[g][1]);
            acc[g][2] = fmaf(x, v.z, acc[g][2]);
            acc[g][3] = fmaf(x, v.w, acc[g][3]);
        }
    }
    // wrapped columns (q < a): weight (k = r-1, n = N+q-a).  Chunk rows k in [k_beg,k_end) <-> aligned rows
    // r = k+1 in [k_beg+1, k_end].  Only column quad 0 has them; done by the warp-0 lanes t == 0.
    float wrap[G][4];
#pragma unroll
    for (int g = 0; g < G; ++g)
#pragma unroll
        for (int c = 0; c < 4; ++c) wrap[g][c] = 0.0f;
    if (t == 0 && a != 0) {
        for (int rr = rw; rr < rows; rr += RW) {          // aligned row k_beg+1+rr, multiplier x[k_beg+rr]
            const float4 v = ldg_stream_f4(S + (int64_t)(k_beg + 1 + rr) * N);
#pragma unroll
            for (int g = 0; g < G; ++g) {
                const float x = xs[g * xs_ld + 1 + rr];
                wrap[g][0] = fmaf(x, v.x, wrap[g][0]);
                wrap[g][1] = fmaf(x, v.y, wrap[g][1]);
                wrap[g][2] = fmaf(x, v.z, wrap[g][2]);
                wrap[g][3] = fmaf(x, v.w, wrap[g][3]);
            }
        }
    }
    // cross-reader reduction (fixed order) and store of this chunk's partial [G][N]
    __syncthreads();                                     // xs no longer needed: reuse smem
    float* red = smem;                                   // [RW][G][N + 4]
    const int red_ld = N + 4;
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
    __syncthreads();
    float* out = part + ((int64_t)group * n_chunks + chunk) * G * N;
    for (int i = threadIdx.x; i < G * N; i += blockDim.x) {
        const int g = i / N, n = i % N;
        float sum = 0.0f;
        for (int w = 0; w < RW; ++w) sum += red[(w * G + g) * red_ld + n];
        out[i] = sum;
    }
}

// combine:  y[m][n] = act(bn( sum_split Ytheta + s_m * sum_chunk Ynoise + bias ))
// theta partials are [split][slot][N] (shared-theta GEMM, Gt == 0) or [group][chunk][Gt][N] (per-parent GEMV).
__global__ void __launch_bounds__(256)
dense_combine_kernel(SlotArgs sa, LayerEpi epi, int n_slots, int N, int G, const float* __restrict__ part_theta,
                     int n_split, int Gt, const float* __restrict__ part_noise, int n_chunks,
                     float* __restrict__ out, int64_t out_slot_stride) {
    const int slot = blockIdx.y;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N || !slot_active(sa, slot)) return;
    float yt = 0.0f;
    if (Gt == 0) {
        for (int sp = 0; sp < n_split; ++sp) yt += part_theta[((int64_t)sp * n_slots + slot) * N + n];
    } else {
        const float* pt = part_theta + (((int64_t)(slot / Gt) * n_split) * Gt + (slot % Gt)) * N + n;
        for (int c = 0; c < n_split; ++c) yt += pt[(int64_t)c * Gt * N];
    }
    const int group = slot / G, g = slot % G;
    float yn = 0.0f;
    const float* pn = part_noise + (((int64_t)group * n_chunks) * G + g) * N + n;
    for (int c = 0; c < n_chunks; ++c) yn += pn[(int64_t)c * G * N];
    const float s = sa.scale[slot];
    const float* th = slot_theta(sa, slot);
    const ChanEpi ce = make_chan_epi(sa, epi, slot, N, n, th, sa.noise_idx[slot], s);
    // n_split < 0: the GEMV folded s * (noise partial) + theta partials into part_noise (gemv_bulk.cu)
    out[(int64_t)slot * out_slot_stride + n] = ce.apply(n_split < 0 ? yn : fmaf(s, yn, yt));
}

// ---------------------------------------------------------------------------------------------------
// Small / irregular dense layer (output heads: 512x18, 256x17; anything with N % 4 != 0), one CTA per slot and tile
// of up to DS_MAXN output columns, fused w = theta + s*noise, optional argmax (policies.py:330: first max on ties, NaN
// counts as max; only for N <= DS_MAXN, a single tile).
// ---------------------------------------------------------------------------------------------------
constexpr int DS_THREADS = 256, DS_MAXN = 256;

// Column tile blockIdx.y covers columns [n0, n0 + NT).  Thread t < RG*NT owns output column n0 + t % NT and row group
// rg = t / NT (RG = 256 / NT row groups).  With a single tile (N <= 256), one iteration of the k loop covers RG
// consecutive rows = RG*N CONTIGUOUS weights, so the theta / noise loads are flat and perfectly coalesced whatever N
// is (18, 17, ...); wider layers read NT contiguous weights per row.
__global__ void __launch_bounds__(DS_THREADS)
dense_small_kernel(SlotArgs sa, int64_t off_w, LayerEpi epi, const float* __restrict__ X, int64_t x_slot_stride,
                   int K, int N, float* __restrict__ out, int64_t out_slot_stride, int32_t* __restrict__ actions) {
    const int slot = blockIdx.x;
    if (!slot_active(sa, slot)) return;
    __shared__ float red[DS_THREADS];
    __shared__ float ys[DS_MAXN];
    const int n0 = blockIdx.y * DS_MAXN;
    const int NT = min(DS_MAXN, N - n0);
    const int RG = DS_THREADS / NT;
    const int t = threadIdx.x;
    const int n = t % NT, rg = t / NT;
    const float* th = slot_theta(sa, slot);
    const int64_t idx = sa.noise_idx[slot];
    const float s = sa.scale[slot];
    const float* tw = th + off_w + n0;
    const float* nz = sa.noise + idx + off_w + n0;
    const float* x = X + (int64_t)slot * x_slot_stride;
    float acc0 = 0.0f, acc1 = 0.0f;
    if (rg < RG) {
        int k = rg;
        for (; k + RG < K; k += 2 * RG) {                      // two independent rows in flight
            const int64_t f0 = (int64_t)k * N + n, f1 = (int64_t)(k + RG) * N + n;
            const float t0 = tw[f0], n0 = nz[f0], t1 = tw[f1], n1 = nz[f1];
            acc0 = fmaf(x[k], perturbed(t0, s, n0), acc0);
            acc1 = fmaf(x[k + RG], perturbed(t1, s, n1), acc1);
        }
        if (k < K) {
            const int64_t f0 = (int64_t)k * N + n;
            acc0 = fmaf(x[k], perturbed(tw[f0], s, nz[f0]), acc0);
        }
    }
    red[t] = acc0 + acc1;
    __syncthreads();
    if (t < NT) {
        float sum = 0.0f;
        for (int g = 0; g < RG; ++g) sum += red[g * NT + t];
        const ChanEpi ce = make_chan_epi(sa, epi, slot, N, n0 + t, th, idx, s);
        const float y = ce.apply(sum);
        ys[t] = y;
        if (out) out[(int64_t)slot * out_slot_stride + n0 + t] = y;
    }
    __syncthreads();
    if (actions && threadIdx.x == 0) {             // N <= DS_MAXN (dne_launch_dense_layer): one tile holds every column
        int best = 0;
        float bv = ys[0];
        for (int j = 1; j < N; ++j) {
            const float v = ys[j];
            if (bv != bv) break;                   // a NaN already is the maximum (numpy argmax)
            if (v > bv || v != v) { bv = v; best = j; }
        }
        actions[slot] = best;
    }
}

// combine + output head in one kernel (one CTA per slot): the hidden vector y[N1] of dense_combine_kernel is built in
// shared memory and fed straight to the head (512x18 / 256x18 / 256x17) and its argmax -- one launch and one global round
// trip less per tick.  Both phases are latency bound (L2 partials; theta + noise rows of the head), so every thread keeps 8
// independent loads in flight and adds them in index order (the sums are order-deterministic).
constexpr int DCH_MAXK = 1024, DCH_THREADS = 512, DCH_B = 8, DCH_HR = 20;
__global__ void __launch_bounds__(DCH_THREADS, 2)
dense_combine_head_kernel(SlotArgs sa, LayerEpi epi1, int n_slots, int N1, int G, const float* __restrict__ part_theta,
                          int n_split, int Gt, const float* __restrict__ part_noise, int n_chunks,
                          float* __restrict__ hidden_out, int64_t hidden_stride,
                          int64_t off_w2, LayerEpi epi2, int N2, float* __restrict__ out, int64_t out_slot_stride,
                          int32_t* __restrict__ actions) {
    const int slot = blockIdx.x;
    if (!slot_active(sa, slot)) return;                // (an exited CTA counts as triggered / never blocks a dependent)
    __shared__ float xs[DCH_MAXK];
    __shared__ float red[DCH_THREADS];
    __shared__ float ys[DS_MAXN];
    const int t = threadIdx.x;
    const float* th = slot_theta(sa, slot);
    const int64_t idx = sa.noise_idx[slot];
    const float s = sa.scale[slot];
    // The head's weights do not depend on phase 1: when a thread's share of rows fits in registers (K / RG <= DCH_HR), its
    // theta / noise loads (HBM latency) are issued FIRST and overlap the L2 round trips of the partial sums below.
    const int K = N1, N = N2;
    const int RG = DCH_THREADS / N;
    const int hn_ = t % N, rg = t / N;
    const float* tw = th + off_w2;
    const float* nz = sa.noise + idx + off_w2;
    const int rows_pt = (K + RG - 1) / RG;
    const bool pre = rows_pt <= DCH_HR;
    float hw[DCH_HR], hz[DCH_HR];
    if (pre && rg < RG) {
#pragma unroll
        for (int j = 0; j < DCH_HR; ++j) {
            const int k = rg + j * RG;
            const int64_t f = (int64_t)k * N + hn_;
            hw[j] = k < K ? tw[f] : 0.0f;
            hz[j] = k < K ? nz[f] : 0.0f;
        }
    }
    // ---- phase 1: y = act(bn(sum_split Ytheta + s * sum_chunk Ynoise + bias))  (dense_combine_kernel) ----
    pdl_wait();                                        // common.cuh: the partial sums come from the previous kernels of the tick
    // partial sums: DCH_B predicated loads in flight, added in index order (same order as a sequential loop)
    auto sum_strided = [](const float* p, int64_t stride, int count) {
        float acc = 0.0f;
        for (int c = 0; c < count; c += DCH_B) {
            float v[DCH_B];
#pragma unroll
            for (int j = 0; j < DCH_B; ++j) v[j] = (c + j < count) ? p[(int64_t)(c + j) * stride] : 0.0f;
#pragma unroll
            for (int j = 0; j < DCH_B; ++j)
                if (c + j < count) acc += v[j];
        }
        return acc;
    };
    for (int n = t; n < N1; n += DCH_THREADS) {
        const ChanEpi ce = make_chan_epi(sa, epi1, slot, N1, n, th, idx, s);      // its two loads go out before the partials
        const float* pt;
        int64_t pt_stride;
        if (Gt == 0) { pt = part_theta + (int64_t)slot * N1 + n; pt_stride = (int64_t)n_slots * N1; }
        else { pt = part_theta + (((int64_t)(slot / Gt) * n_split) * Gt + (slot % Gt)) * N1 + n; pt_stride = (int64_t)Gt * N1; }
        const int group = slot / G, g = slot % G;
        const float* pn = part_noise + (((int64_t)group * n_chunks) * G + g) * N1 + n;
        const float yt = sum_strided(pt, pt_stride, n_split);          // n_split < 0 (folded into the noise partials): no loads
        const float yn = sum_strided(pn, (int64_t)G * N1, n_chunks);
        const float y = ce.apply(n_split < 0 ? yn : fmaf(s, yn, yt));
        xs[n] = y;
        if (hidden_out) hidden_out[(int64_t)slot * hidden_stride + n] = y;
    }
    __syncthreads();
    // ---- phase 2: the head on x = xs.  Thread t < RG*N owns output column n = t % N and row group rg = t / N (rows rg,
    // rg + RG, ...: a batch of rows is a contiguous run of weights, so the loads are flat and coalesced) ----
    const int n = hn_;
    float acc = 0.0f;
    if (rg < RG) {
        if (pre) {
#pragma unroll
            for (int j = 0; j < DCH_HR; ++j) {
                const int k = rg + j * RG;
                if (k < K) acc = fmaf(xs[k], perturbed(hw[j], s, hz[j]), acc);
            }
        } else {
            int k = rg;
            for (; k + (DCH_B - 1) * RG < K; k += DCH_B * RG) {
                float a[DCH_B], b[DCH_B];
#pragma unroll
                for (int j = 0; j < DCH_B; ++j) {
                    const int64_t f = (int64_t)(k + j * RG) * N + n;
                    a[j] = tw[f];
                    b[j] = nz[f];
                }
#pragma unroll
                for (int j = 0; j < DCH_B; ++j) acc = fmaf(xs[k + j * RG], perturbed(a[j], s, b[j]), acc);
            }
            for (; k < K; k += RG) {
                const int64_t f = (int64_t)k * N + n;
                acc = fmaf(xs[k], perturbed(tw[f], s, nz[f]), acc);
            }
        }
    }
    red[t] = acc;
    __syncthreads();
    if (t < N) {
        float sum = 0.0f;
        for (int g = 0; g < RG; ++g) sum += red[g * N + t];
        const ChanEpi ce = make_chan_epi(sa, epi2, slot, N, t, th, idx, s);
        const float y = ce.apply(sum);
        ys[t] = y;
        if (out) out[(int64_t)slot * out_slot_stride + t] = y;
    }
    __syncthreads();
    if (actions && threadIdx.x == 0) {
        int best = 0;
        float bv = ys[0];
        for (int j = 1; j < N; ++j) {
            const float v = ys[j];
            if (bv != bv) break;                   // a NaN already is the maximum (numpy argmax)
            if (v > bv || v != v) { bv = v; best = j; }
        }
        actions[slot] = best;
    }
}

// MujocoPolicy observation normalisation (policies.py:151): clip((o - mean) / std, -5, 5).  Without statistics (mean
// NULL: SimpleClassifier / LinearClassifier, models/simple.py) the observation goes through unchanged and unclipped.
__global__ void ob_norm_kernel(const float* __restrict__ obs, const float* __restrict__ mean,
                               const float* __restrict__ stdv, int64_t total, int dim, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int d = (int)(i % dim);
    float v = obs[i];
    if (mean) v = fminf(fmaxf(__fdiv_rn(__fsub_rn(v, mean[d]), stdv[d]), -5.0f), 5.0f);
    out[i] = v;
}

// Observation statistics for the running normaliser (es.py:356-363: task_ob_stat.increment(obs.sum(0), square(obs).sum(0),
// len(obs)) over the episodes sampled with probability calc_obstat_prob): per tick, add the observations of the listed
// slots into float64 running sums.  One thread per observation dimension, slots in list order: deterministic.
__global__ void ob_stat_accum_kernel(const float* __restrict__ obs, int dim, const int32_t* __restrict__ slots, int m,
                                     double* __restrict__ sum, double* __restrict__ sumsq) {
    const int d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= dim) return;
    double a = 0.0, b = 0.0;
    for (int i = 0; i < m; ++i) {
        const double v = (double)obs[(int64_t)slots[i] * dim + d];
        a += v;
        b += v * v;
    }
    sum[d] += a;
    sumsq[d] += b;
}

extern "C" int dne_ob_stat_accumulate(const float* d_obs, int ob_dim, const int32_t* d_slots, int m, double* d_sum,
                                      double* d_sumsq, void* stream) {
    DNE_CHECK_ARG(d_obs && d_slots && d_sum && d_sumsq && ob_dim > 0 && m >= 0, "bad arguments");
    if (m == 0) return DNE_OK;
    ob_stat_accum_kernel<<<(ob_dim + 127) / 128, 128, 0, (cudaStream_t)stream>>>(d_obs, ob_dim, d_slots, m, d_sum, d_sumsq);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}

// =====================================================================================================
// host side: layer dispatch
// =====================================================================================================
struct ConvKey { int cin, cout, ks, stride, hin, hout, pad; };

template <int CIN, int COUT, int KS, int STRIDE, int HIN, int HOUT, int PAD, bool IN_U8, int BM, int TM, int TN>
static void launch_conv(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, const void* in,
                        int64_t in_slot_stride, int64_t in_img_stride, float* out, int64_t out_slot_stride,
                        int64_t out_img_stride, int n_slots, int n_img, cudaStream_t st) {
    constexpr int THREADS = (BM / TM) * (COUT / TN);
    dim3 grid((HOUT * HOUT + BM - 1) / BM, n_slots, n_img);
    conv_kernel<CIN, COUT, KS, STRIDE, HIN, HOUT, PAD, IN_U8, BM, TM, TN><<<grid, THREADS, 0, st>>>(
        sa, L.off_w, epi, in, in_slot_stride, in_img_stride, out, out_slot_stride, out_img_stride);
    DNE_LAUNCHED(1);
}

static bool conv_is(const dne_layer_desc& L, int cin, int cout, int ks, int stride, int hin, int hout, int pad) {
    return L.cin == cin && L.cout == cout && L.ksize == ks && L.stride == stride && L.hin == hin &&
           L.hout == hout && L.pad == pad;
}

// in_u8: the layer reads uint8 observations.  Returns 0 or DNE_ERR_UNSUP.
int g_dne_conv_tc = 2;     // 2: shifted-window wgmma + TMA (conv_s2d.cu), 1: im2col-staged wgmma (tc_conv.cu), 0: fp32 SIMT

int dne_launch_conv_layer(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, bool in_u8,
                          const void* in, int64_t in_slot_stride, int64_t in_img_stride, float* out,
                          int64_t out_slot_stride, int64_t out_img_stride, int n_slots, int n_img,
                          cudaStream_t st) {
    if (g_dne_conv_tc) {
        const int rc = dne_launch_conv_layer_tc(sa, L, epi, in_u8, in, in_slot_stride, in_img_stride, out,
                                                out_slot_stride, out_img_stride, n_slots, n_img, st);
        if (rc != DNE_ERR_UNSUP) return rc;
    }
    return dne_launch_conv_layer_simt(sa, L, epi, in_u8, in, in_slot_stride, in_img_stride, out, out_slot_stride,
                                      out_img_stride, n_slots, n_img, st);
}

int dne_launch_conv_layer_simt(const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi, bool in_u8,
                          const void* in, int64_t in_slot_stride, int64_t in_img_stride, float* out,
                          int64_t out_slot_stride, int64_t out_img_stride, int n_slots, int n_img,
                          cudaStream_t st) {
#define ARGS sa, L, epi, in, in_slot_stride, in_img_stride, out, out_slot_stride, out_img_stride, n_slots, n_img, st
    if (in_u8 && conv_is(L, 4, 32, 8, 4, 84, 21, 2)) { launch_conv<4, 32, 8, 4, 84, 21, 2, true, 128, 8, 4>(ARGS); return 0; }
    if (in_u8 && conv_is(L, 4, 16, 8, 4, 84, 21, 2)) { launch_conv<4, 16, 8, 4, 84, 21, 2, true, 128, 8, 2>(ARGS); return 0; }
    if (!in_u8 && conv_is(L, 32, 64, 4, 2, 21, 11, 1)) { launch_conv<32, 64, 4, 2, 21, 11, 1, false, 128, 8, 4>(ARGS); return 0; }
    if (!in_u8 && conv_is(L, 16, 32, 4, 2, 21, 11, 1)) { launch_conv<16, 32, 4, 2, 21, 11, 1, false, 128, 8, 4>(ARGS); return 0; }
    if (!in_u8 && conv_is(L, 64, 64, 3, 1, 11, 11, 1)) { launch_conv<64, 64, 3, 1, 11, 11, 1, false, 128, 8, 4>(ARGS); return 0; }
#undef ARGS
    return DNE_ERR_UNSUP;
}

// ---- dense-layer planning (shared by the ws query and the launcher) -----------------------------------
DensePlan dne_plan_dense(const dne_layer_desc& L, int n_slots, int paired, bool shared_theta, int sm_count) {
    DensePlan p;
    memset(&p, 0, sizeof(p));
    const int K = L.cin, N = L.cout;
    // paired < 0 marks the output head (needs the argmax epilogue of dense_small_kernel)
    p.decomposed = (paired >= 0) && (N % 4 == 0) && (K % 4 == 0) && ((int64_t)K * N >= 16384) && (N / 4 <= 256);
    if (!p.decomposed) return p;
    // paired bit 0: slots (2p,2p+1) share the noise index; bit 1: they share the theta row (GA parent)
    p.G = (paired & 1) ? 2 : 1;
    p.Gt = shared_theta ? 0 : ((paired & 2) ? 2 : 1);
    // split-K so that the GEMM grid is one wave of the TMA-fed kernel (one CTA per SM, each owning a PAIR of 128-row M tiles
    // of one N tile: theta_gemm_tma.cu) = two waves of the 128x128-tile kernels at M = 256
    const int m_tiles = (n_slots + DG_BM - 1) / DG_BM;
    const int tiles = ((m_tiles + 1) / 2) * ((N + DG_BN - 1) / DG_BN);
    const int k_tiles = (K + DG_BK - 1) / DG_BK;
    int split = (sm_count + tiles - 1) / tiles;
    if (split > k_tiles) split = k_tiles;
    if (split < 1) split = 1;
    int kt_per = (k_tiles + split - 1) / split;
    kt_per += kt_per & 1;                                // k_per_split % 32 == 0: the TMA-fed fp16 GEMM moves K chunks of 32
    p.k_per_split = kt_per * DG_BK;
    p.n_split = (K + p.k_per_split - 1) / p.k_per_split;
    // partials per group: the union GEMV's pieces (one per table block a slice can touch); the SIMT GEMV writes the same
    // number of partials, each over rows_per_chunk rows of K
    p.n_chunks = dne_gemv_pieces(K);
    p.rows_per_chunk = (K + p.n_chunks - 1) / p.n_chunks;
    const int nq = N / 4;
    p.rw = 1;
    while (nq * p.rw * 2 <= 256 && p.rw * 2 <= 8) p.rw *= 2;
    while (nq * p.rw < 64 && p.rw < 8) p.rw *= 2;
    p.part_theta_floats = (size_t)p.n_split * n_slots * N;
    if (p.Gt) {                                        // per-parent theta streamed by the GEMV kernel
        p.n_split = p.n_chunks;
        p.part_theta_floats = (size_t)((n_slots + p.Gt - 1) / p.Gt) * p.n_chunks * p.Gt * N;
    }
    const int groups = (n_slots + p.G - 1) / p.G;
    p.part_noise_floats = (size_t)groups * p.n_chunks * p.G * N;
    return p;
}

bool dne_head_fusable(const dne_layer_desc& L, const DensePlan& p, const dne_layer_desc& head, const DensePlan& hp) {
    return p.decomposed && !hp.decomposed && L.cout <= DCH_MAXK && head.cin == L.cout && head.cout <= DS_MAXN;
}

int dne_launch_dense_layer(const dne_ctx* ctx, const SlotArgs& sa, const dne_layer_desc& L, const LayerEpi& epi,
                           const DensePlan& p, const float* X, int64_t x_slot_stride, float* out,
                           int64_t out_slot_stride, int32_t* actions, float* part_theta, float* part_noise,
                           int n_slots, cudaStream_t st, const DenseHead* head, const TgmOperands* tgm) {
    const int K = L.cin, N = L.cout;
    if (!p.decomposed) {
        if (actions && N > DS_MAXN) return DNE_ERR_UNSUP;          // the argmax runs over one column tile
        dense_small_kernel<<<dim3(n_slots, (N + DS_MAXN - 1) / DS_MAXN), DS_THREADS, 0, st>>>(
            sa, L.off_w, epi, X, x_slot_stride, K, N, out, out_slot_stride, actions);
        DNE_LAUNCHED(1);
        return 0;
    }
    if (x_slot_stride != K || actions) return DNE_ERR_UNSUP;   // heads always go through dense_small_kernel
    const int threads = (N / 4) * p.rw;
    auto gemv_smem = [&](int G) {
        size_t sm1 = (size_t)G * (p.rows_per_chunk + 1) * sizeof(float);
        size_t sm2 = (size_t)p.rw * G * (N + 4) * sizeof(float);
        return sm1 > sm2 ? sm1 : sm2;
    };
    if (p.Gt == 0) {
        // TMA-fed wgmma GEMM when both operands are pre-arranged (dne_theta_prepare + conv_s2d epilogue); else
        // thread-staged tensor cores (wgmma, 3xTF32) when enabled, fp32 SIMT otherwise
        if (tgm && dne_launch_theta_gemm_tma(tgm->Xc, tgm->Wc, n_slots, K, N, p.k_per_split, p.n_split, part_theta, st) == 0) {
        } else if (!(g_dne_conv_tc && dne_launch_theta_gemm_tc(X, n_slots, K, N, sa.theta + L.off_w, p.k_per_split, p.n_split,
                                                        part_theta, st) == 0)) {
            dim3 grid((N + DG_BN - 1) / DG_BN, (n_slots + DG_BM - 1) / DG_BM, p.n_split);
            dense_theta_gemm_kernel<<<grid, DG_THREADS, 0, st>>>(X, n_slots, K, N, sa.theta + L.off_w, p.k_per_split,
                                                                part_theta);
        }
    } else {
        GemvSrc ts{sa.theta, nullptr, sa.theta_idx, sa.P, L.off_w};
        dim3 grid(p.n_chunks, (n_slots + p.Gt - 1) / p.Gt);
        if (g_dne_gemv_bulk && dne_launch_gemv_union(sa, ts, p.Gt, X, x_slot_stride, K, N, p.n_chunks, n_slots, part_theta,
                                                     ctx->sm_count, st) == 0) {
        } else if (p.Gt == 2)
            dense_noise_gemv_kernel<2, 8><<<grid, threads, gemv_smem(2), st>>>(sa, ts, X, x_slot_stride, K, N,
                                                                              p.rows_per_chunk, part_theta);
        else
            dense_noise_gemv_kernel<1, 8><<<grid, threads, gemv_smem(1), st>>>(sa, ts, X, x_slot_stride, K, N,
                                                                              p.rows_per_chunk, part_theta);
    }
    bool folded = false;
    {
        GemvSrc ns{sa.noise, sa.noise_idx, nullptr, 0, L.off_w};
        dne_ctx* mctx = const_cast<dne_ctx*>(ctx);
        const bool first_gemv = !ctx->ev_record_done;
        if (first_gemv && ctx->ev_mode == 0 && ctx->ev_record) {     // mode 0: the HBM-bound part of this call starts
            cudaEventRecord((cudaEvent_t)ctx->ev_record, st);
            mctx->ev_record_done = 1;
        }
        if (first_gemv && ctx->ev_mode == 1 && ctx->ev_wait) {       // mode 1: take turns on the memory system
            cudaStreamWaitEvent(st, (cudaEvent_t)ctx->ev_wait, 0);
            mctx->ev_wait = nullptr;
        }
        const int groups = (n_slots + p.G - 1) / p.G;
        dim3 grid(p.n_chunks, groups);
        const bool prof = ctx->prof_on && ctx->ev_n < ctx->ev_cap;
        if (prof) cudaEventRecord(ctx->ev[2 * ctx->ev_n], st);
        // fold the theta GEMM's split-K partials into the GEMV output (gemv_bulk.cu)
        folded = g_dne_gemv_bulk && g_dne_fold_theta && p.Gt == 0;
        if (g_dne_gemv_bulk && dne_launch_gemv_union(sa, ns, p.G, X, x_slot_stride, K, N, p.n_chunks, n_slots, part_noise,
                                                     ctx->sm_count, st, folded ? part_theta : nullptr,
                                                     folded ? p.n_split : 0) == 0) {
        } else if ((folded = false), p.G == 2)
            dense_noise_gemv_kernel<2, 8><<<grid, threads, gemv_smem(2), st>>>(sa, ns, X, x_slot_stride, K, N,
                                                                              p.rows_per_chunk, part_noise);
        else
            dense_noise_gemv_kernel<1, 8><<<grid, threads, gemv_smem(1), st>>>(sa, ns, X, x_slot_stride, K, N,
                                                                              p.rows_per_chunk, part_noise);
        if (prof) {
            cudaEventRecord(ctx->ev[2 * ctx->ev_n + 1], st);
            const_cast<dne_ctx*>(ctx)->ev_n++;
        }
        if (first_gemv && ctx->ev_mode == 1 && ctx->ev_record) {
            cudaEventRecord((cudaEvent_t)ctx->ev_record, st);
            mctx->ev_record_done = 1;
        }
    }
    if (head) {          // combine + output head + argmax in one kernel (the hidden vector stays in shared memory)
        // PDL: the head's weight loads (theta / noise, not written inside a tick) go out before its pdl_wait()
        if (dne_launch_chain(dense_combine_head_kernel, dim3(n_slots), dim3(DCH_THREADS), 0, st, true, sa, epi, n_slots, N, p.G,
                             (const float*)part_theta, folded ? -1 : p.n_split, p.Gt, (const float*)part_noise, p.n_chunks, out, out_slot_stride,
                             (int64_t)head->L->off_w, head->epi, (int)head->L->cout, head->out, head->out_slot_stride,
                             head->actions) != cudaSuccess)
            return DNE_ERR_CUDA;
    } else {
        dim3 grid((N + 255) / 256, n_slots);
        dense_combine_kernel<<<grid, 256, 0, st>>>(sa, epi, n_slots, N, p.G, part_theta, folded ? -1 : p.n_split, p.Gt, part_noise,
                                                  p.n_chunks, out, out_slot_stride);
    }
    DNE_LAUNCHED(3);
    return 0;
}

void dne_launch_ob_norm(const float* obs, const float* mean, const float* stdv, int64_t total, int dim, float* out,
                        cudaStream_t st) {
    ob_norm_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(obs, mean, stdv, total, dim, out);
    DNE_LAUNCHED(1);
}
