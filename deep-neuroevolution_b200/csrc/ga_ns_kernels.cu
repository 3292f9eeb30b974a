// ga_ns_kernels.cu -- GA genome materialisation / mutation / truncation selection, k-NN novelty,
// Atari observation preprocess.  All are integer/byte or streaming float work (HBM bound; no GEMM shape).
//
//   dne_ga_materialize <- ga.py:256-264 + policies.py:42-44 + tf_util.py:122-130 (mode 1, CPU path)
//                         gpu_implementation/neuroevolution/models/base.py:140-146,155-156 + dqn.py:26-28 (mode 0)
//   dne_ga_mutate      <- models/base.py:155-156
//   dne_ga_truncate    <- ga.py:145-149 ; gpu_implementation/ga.py:180
//   dne_knn_novelty    <- nses.py:12-32
//   dne_preprocess_atari <- atari_wrappers.py:105,167-180 ; tf_atari.py:90 ; stack_frames.py:33-43
#include "common.cuh"

// ---- GA: seed-chain -> theta ---------------------------------------------------------------------------
// init of one variable.  kind 0: weights mode 0 (scale_by), 1: weights mode 1 (column normalise), 2: zero
__global__ void ga_init_scale_kernel(const float* __restrict__ nz, int64_t size, float scale, float* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < size) out[i] = __fmul_rn(nz[i], scale);            // base.py:141  noise*scale_by
}

// tf_util.py:122-130: out *= std / sqrt(square(out).sum(axis=0)) on the [rows, cout] view.  One thread per
// output column, rows accumulated sequentially in float32 -- the same order numpy uses for an axis-0 sum.
__global__ void ga_init_normc_kernel(const float* __restrict__ nz, int rows, int cout, float stdv,
                                     float* __restrict__ out) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= cout) return;
    float ss = 0.0f;
    for (int r = 0; r < rows; ++r) {
        const float v = nz[(int64_t)r * cout + n];
        ss = __fadd_rn(ss, __fmul_rn(v, v));
    }
    const float f = __fdiv_rn(stdv, __fsqrt_rn(ss));
    for (int r = 0; r < rows; ++r) out[(int64_t)r * cout + n] = __fmul_rn(nz[(int64_t)r * cout + n], f);
}

// theta[e] = fl(theta[e] + fl(p_k * noise[seed_k + e])) for k = 1..len-1, in chain order (base.py:143-145,
// ga.py:262-263): one float32 rounding per product and per add, like the reference's numpy expression.
__global__ void ga_chain_kernel(const float* __restrict__ noise, const int64_t* __restrict__ seeds,
                                const float* __restrict__ powers, int len, int64_t P, float* __restrict__ theta) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= P) return;
    float t = theta[e];
    for (int k = 1; k < len; ++k) t = __fadd_rn(t, __fmul_rn(powers[k], ldg_stream_f1(noise + seeds[k] + e)));
    theta[e] = t;
}

__global__ void ga_mutate_kernel(const float* __restrict__ parent, const float* __restrict__ nz, float power,
                                 int64_t P, float* __restrict__ out) {
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e < P) out[e] = __fadd_rn(parent[e], __fmul_rn(power, ldg_stream_f1(nz + e)));
}

__global__ void read_seed0_kernel(const int64_t* seeds, int64_t* out) { *out = seeds[0]; }

extern "C" int dne_ga_materialize(dne_ctx* ctx, const dne_net_desc* net, const int64_t* d_seeds,
                                  const float* d_powers, int len, const double* h_std, int mode, float* d_theta_out,
                                  void* stream) {
    if (ctx) dne_prep_invalidate_theta(ctx, d_theta_out);
    DNE_CHECK_ARG(ctx && ctx->noise && net && d_seeds && d_theta_out && len >= 1, "bad arguments");
    DNE_CHECK_ARG(len == 1 || d_powers, "powers required for chains longer than 1");
    DNE_CHECK_ARG(mode == 0 || mode == 1, "mode must be 0 (gpu path) or 1 (cpu path)");
    cudaStream_t st = (cudaStream_t)stream;
    // seed0 is needed on the host to address the per-variable init kernels; one 8-byte D2H copy.
    int64_t seed0 = 0;
    DNE_CUDA(cudaMemcpyAsync(&seed0, d_seeds, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    DNE_CUDA(cudaStreamSynchronize(st));
    DNE_CHECK_ARG(seed0 >= 0 && seed0 + net->num_params <= ctx->noise_count, "seed out of range");
    const float* nz = ctx->noise + seed0;
    DNE_CUDA(cudaMemsetAsync(d_theta_out, 0, sizeof(float) * net->num_params, st));   // biases / BN params -> 0
    for (int l = 0; l < net->n_layers; ++l) {
        const dne_layer_desc& L = net->layers[l];
        const int rows = (L.kind == DNE_CONV) ? L.ksize * L.ksize * L.cin : L.cin;
        const int64_t size = (int64_t)rows * L.cout;
        const double stdv = h_std ? h_std[l] : 1.0;
        if (mode == 0) {
            const float scale = (float)(stdv / sqrt((double)rows));           // dqn.py:27
            ga_init_scale_kernel<<<(unsigned)cdiv64(size, 256), 256, 0, st>>>(nz + L.off_w, size, scale,
                                                                             d_theta_out + L.off_w);
        } else {
            ga_init_normc_kernel<<<(L.cout + 127) / 128, 128, 0, st>>>(nz + L.off_w, rows, L.cout, (float)stdv,
                                                                      d_theta_out + L.off_w);
        }
        DNE_LAUNCH_CHECK1();
    }
    if (len > 1) {
        ga_chain_kernel<<<(unsigned)cdiv64(net->num_params, 256), 256, 0, st>>>(ctx->noise, d_seeds, d_powers, len,
                                                                               net->num_params, d_theta_out);
        DNE_LAUNCH_CHECK1();
    }
    return DNE_OK;
}

extern "C" int dne_ga_mutate(dne_ctx* ctx, const float* d_parent, int64_t seed, float power, int64_t P,
                             float* d_theta_out, void* stream) {
    if (ctx) dne_prep_invalidate_theta(ctx, d_theta_out);
    DNE_CHECK_ARG(ctx && ctx->noise && d_parent && d_theta_out && P > 0, "bad arguments");
    DNE_CHECK_ARG(seed >= 0 && seed + P <= ctx->noise_count, "seed out of range");
    ga_mutate_kernel<<<(unsigned)cdiv64(P, 256), 256, 0, (cudaStream_t)stream>>>(d_parent, ctx->noise + seed, power,
                                                                                P, d_theta_out);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}

// ---- GA: truncation selection --------------------------------------------------------------------------
// position of i in the stable descending order = #{j: f[j] > f[i]} + #{j < i: f[j] == f[i]}  (NaN last).
__device__ __forceinline__ bool desc_before(float a, float b) { return (a > b) || ((b != b) && (a == a)); }
__device__ __forceinline__ bool desc_eq(float a, float b) { return (a == b) || ((a != a) && (b != b)); }

__global__ void __launch_bounds__(256) ga_truncate_kernel(const float* __restrict__ f, int pop, int T,
                                                          int32_t* __restrict__ selected) {
    __shared__ float tile[1024];
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const float fi = (i < pop) ? f[i] : 0.0f;
    int r = 0;
    for (int base = 0; base < pop; base += 1024) {
        const int len = min(1024, pop - base);
        __syncthreads();
        for (int t = threadIdx.x; t < len; t += blockDim.x) tile[t] = f[base + t];
        __syncthreads();
        if (i < pop)
            for (int t = 0; t < len; ++t) {
                const float fj = tile[t];
                r += (desc_before(fj, fi) || (desc_eq(fj, fi) && (base + t) < i)) ? 1 : 0;
            }
    }
    if (i < pop && r < T) selected[r] = i;
}

extern "C" int dne_ga_truncate(const float* d_fitness, int pop, int T, int32_t* d_selected, void* stream) {
    DNE_CHECK_ARG(d_fitness && d_selected && pop >= 1 && T >= 1 && T <= pop, "bad arguments");
    ga_truncate_kernel<<<(pop + 255) / 256, 256, 0, (cudaStream_t)stream>>>(d_fitness, pop, T, d_selected);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}

// ---- k-NN novelty ----------------------------------------------------------------------------------------
// dist^2(q,a) = sum over rows t < max(len_q,len_a), cols d of (q[t][d]-a[t][d])^2 on last-row-padded uint8
// sequences == nses.py:12-20.  Exact integer arithmetic (abs-diff + dp4a), float64 sqrt.
constexpr int KNN_THREADS = 256;

__global__ void __launch_bounds__(KNN_THREADS)
knn_dist_kernel(const uint8_t* __restrict__ bc, const int32_t* __restrict__ bc_len, const uint8_t* __restrict__ ar,
                const int32_t* __restrict__ ar_len, int t_max, int D, double* __restrict__ dist, int A) {
    const int ai = blockIdx.x, qi = blockIdx.y;
    const int rows = min(t_max, max(bc_len[qi], ar_len[ai]));
    const int64_t nbytes = (int64_t)rows * D;
    const uint8_t* q = bc + (int64_t)qi * t_max * D;
    const uint8_t* a = ar + (int64_t)ai * t_max * D;
    unsigned long long total = 0;
    unsigned int acc = 0;
    int pending = 0;
    const int64_t nwords = nbytes >> 2;                       // D % 4 == 0 is checked by the host
    const uint32_t* q4 = reinterpret_cast<const uint32_t*>(q);
    const uint32_t* a4 = reinterpret_cast<const uint32_t*>(a);
    for (int64_t w = threadIdx.x; w < nwords; w += KNN_THREADS) {
        const uint32_t d = __vabsdiffu4(q4[w], a4[w]);
        acc = __dp4a(d, d, acc);
        if (++pending == 8192) { total += acc; acc = 0; pending = 0; }
    }
    total += acc;
    total = warp_sum(total);
    __shared__ unsigned long long sh[KNN_THREADS / 32];
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = total;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long s = 0;
        for (int i = 0; i < KNN_THREADS / 32; ++i) s += sh[i];
        dist[(int64_t)qi * A + ai] = sqrt((double)s);
    }
}

// mean of the k smallest distances per query (nses.py:28-32); k successive min-extractions, one CTA per query.
// Order of numpy's sort: numbers ascending, NaN after every number (a NaN BC coordinate gives NaN distances), so a NaN is
// taken only when no number is left and the mean is then NaN.  Taken entries are marked -1.0 (distances are never < 0).
__device__ __forceinline__ bool dist_before(double a, double b) { return (a < b) || ((b != b) && (a == a)); }
__device__ __forceinline__ bool dist_same(double a, double b) { return (a == b) || ((a != a) && (b != b)); }

__global__ void __launch_bounds__(KNN_THREADS)
knn_select_kernel(double* __restrict__ dist, int A, int k, float* __restrict__ novelty) {
    const int qi = blockIdx.x;
    double* d = dist + (int64_t)qi * A;
    __shared__ double sv[KNN_THREADS];
    __shared__ int si[KNN_THREADS];
    const int kk = min(k, A);
    double sum = 0.0;
    for (int it = 0; it < kk; ++it) {         // A - it >= 1 entries are untaken: every iteration finds one
        double bv = 0.0;
        int bi = -1;
        for (int j = threadIdx.x; j < A; j += KNN_THREADS) {
            const double v = d[j];
            if (!(v < 0.0) && (bi < 0 || dist_before(v, bv))) { bv = v; bi = j; }
        }
        sv[threadIdx.x] = bv;
        si[threadIdx.x] = bi;
        __syncthreads();
        for (int o = KNN_THREADS / 2; o > 0; o >>= 1) {
            if (threadIdx.x < o) {
                const int oi = si[threadIdx.x + o];
                const double ov = sv[threadIdx.x + o];
                const double mv = sv[threadIdx.x];
                const int mi = si[threadIdx.x];
                if (oi >= 0 && (mi < 0 || dist_before(ov, mv) || (dist_same(ov, mv) && oi < mi))) {
                    sv[threadIdx.x] = ov;
                    si[threadIdx.x] = oi;
                }
            }
            __syncthreads();
        }
        if (threadIdx.x == 0) {
            sum += sv[0];
            d[si[0]] = -1.0;                                    // mark as taken
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) novelty[qi] = (float)(sum / (double)kk);
}

extern "C" int dne_knn_ws_bytes(int q, int A, size_t* out_bytes) {
    DNE_CHECK_ARG(out_bytes && q >= 0 && A >= 0, "bad arguments");
    *out_bytes = align_up((size_t)q * (size_t)A * sizeof(double), 256);
    return DNE_OK;
}

extern "C" int dne_knn_novelty(const uint8_t* d_bc, const int32_t* d_bc_len, int q, const uint8_t* d_archive,
                               const int32_t* d_archive_len, int A, int t_max, int D, int k, float* d_novelty,
                               void* d_ws, size_t ws_bytes, void* stream) {
    DNE_CHECK_ARG(d_bc && d_bc_len && d_archive && d_archive_len && d_novelty && d_ws, "null pointer");
    DNE_CHECK_ARG(q >= 1 && A >= 1 && t_max >= 1 && D >= 4 && D % 4 == 0 && k >= 1, "bad sizes (D must be a multiple of 4)");
    if (ws_bytes < (size_t)q * A * sizeof(double)) {
        dne_set_error("dne_knn_novelty: workspace too small");
        return DNE_ERR_WS;
    }
    cudaStream_t st = (cudaStream_t)stream;
    double* dist = (double*)d_ws;
    knn_dist_kernel<<<dim3(A, q), KNN_THREADS, 0, st>>>(d_bc, d_bc_len, d_archive, d_archive_len, t_max, D, dist, A);
    DNE_LAUNCH_CHECK1();
    knn_select_kernel<<<q, KNN_THREADS, 0, st>>>(dist, A, k, d_novelty);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}

// Vector behaviour characterisations (MujocoPolicy: final (x, y) position, or the x/y trajectory: policies.py:292-299):
// float64 vectors of equal length D, distance = plain L2 (nses.py:12-20 with n == m), float64 arithmetic in index order.
__global__ void knn_dist_vec_kernel(const double* __restrict__ bc, const double* __restrict__ ar, int q, int A, int D,
                                    double* __restrict__ dist) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (int64_t)q * A) return;
    const int qi = (int)(i / A), ai = (int)(i % A);
    double s = 0.0;
    for (int d = 0; d < D; ++d) {
        const double t = __dsub_rn(bc[(int64_t)qi * D + d], ar[(int64_t)ai * D + d]);
        s = __dadd_rn(s, __dmul_rn(t, t));
    }
    dist[i] = sqrt(s);
}

extern "C" int dne_knn_novelty_vec(const double* d_bc, int q, const double* d_archive, int A, int D, int k, float* d_novelty,
                                   void* d_ws, size_t ws_bytes, void* stream) {
    DNE_CHECK_ARG(d_bc && d_archive && d_novelty && d_ws, "null pointer");
    DNE_CHECK_ARG(q >= 1 && A >= 1 && D >= 1 && k >= 1, "bad sizes");
    if (ws_bytes < (size_t)q * A * sizeof(double)) {
        dne_set_error("dne_knn_novelty_vec: workspace too small");
        return DNE_ERR_WS;
    }
    cudaStream_t st = (cudaStream_t)stream;
    double* dist = (double*)d_ws;
    const int64_t n = (int64_t)q * A;
    knn_dist_vec_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(d_bc, d_archive, q, A, D, dist);
    DNE_LAUNCH_CHECK1();
    knn_select_kernel<<<q, KNN_THREADS, 0, st>>>(dist, A, k, d_novelty);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}

// ---- Atari preprocess: max over two frames + frame stack, in place --------------------------------------
__global__ void preprocess_kernel(const uint8_t* __restrict__ prev, const uint8_t* __restrict__ cur,
                                  uchar4* __restrict__ stack, const uint8_t* __restrict__ reset_mask, int n_slots,
                                  int mode) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;     // pixel index over all slots
    const int64_t total = (int64_t)n_slots * 84 * 84;
    if (i >= total) return;
    const int slot = (int)(i / (84 * 84));
    const uint8_t a = cur[i], b = prev ? prev[i] : (uint8_t)0;
    const uint8_t nw = a > b ? a : b;                                      // atari_wrappers.py:105 / tf_atari.py:90
    uchar4 s = stack[i];
    if (reset_mask && reset_mask[slot]) {
        s = (mode == 0) ? make_uchar4(nw, nw, nw, nw)                      // atari_wrappers.py:167-172
                        : make_uchar4(0, 0, 0, nw);                        // stack_frames.py:33-37
    } else {
        s = make_uchar4(s.y, s.z, s.w, nw);                                // shift left, append
    }
    stack[i] = s;
}

extern "C" int dne_preprocess_atari(const uint8_t* d_prev, const uint8_t* d_cur, uint8_t* d_stack,
                                    const uint8_t* d_reset_mask, int n_slots, int mode, void* stream) {
    DNE_CHECK_ARG(d_cur && d_stack && n_slots >= 0 && (mode == 0 || mode == 1), "bad arguments");
    if (n_slots == 0) return DNE_OK;
    const int64_t total = (int64_t)n_slots * 84 * 84;
    preprocess_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, (cudaStream_t)stream>>>(
        d_prev, d_cur, reinterpret_cast<uchar4*>(d_stack), d_reset_mask, n_slots, mode);
    DNE_LAUNCH_CHECK1();
    return DNE_OK;
}
