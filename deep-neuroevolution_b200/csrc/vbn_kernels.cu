// vbn_kernels.cu -- virtual batch norm reference pass (ESAtariPolicy).
//
//   es_distributed/policies.py:322,324,328  layers.batch_norm(scale=True, is_training=is_ref, decay=0., epsilon=1e-3)
//   es_distributed/policies.py:332-335,399  the 128-observation reference batch is forwarded before every rollout
//   es_distributed/es.py:105-113,160-162    reference batch = 128 random-action observations, shared by all members
//
// Per member: forward the shared reference batch layer by layer with the member's perturbed weights; after each
// BN'd layer take the batch mean / biased variance per channel (these become the member's "moving" statistics
// because decay = 0), normalise, activate, continue.  This is the one sub-problem of the path with real weight
// reuse per member (M = n_ref*441 rows per member for conv1): a dense contraction.
//
// r02: with conv_tc = 2 (default) the convolutions of the pass run on the shifted-window wgmma kernels of the tick
// (conv_s2d.cu) over n_slots * n_ref VIRTUAL slots (virtual slot v = image v % n_ref of member v / n_ref: consecutive CTAs
// share a member, whose weight rows stay L2-hot), writing the raw pre-normalisation output as NHWC floats; after the batch
// statistics, vbn_image_kernel normalises + activates and writes the NEXT conv layer's space-to-depth fp16-split image
// (the layout the tick's conv epilogue produces), and the fc runs on member_gemm_tc_kernel (tc_conv.cu).  conv_tc = 1 keeps
// the r01 tensor-core kernels, conv_tc = 0 the fp32 SIMT referee.
#include "common.cuh"
#include "forward.cuh"
#include "wgmma.cuh"

__device__ __forceinline__ bool v_slot_active(const SlotArgs& a, int slot) { return !a.active || a.active[slot]; }
__device__ __forceinline__ const float* v_slot_theta(const SlotArgs& a, int slot) {
    return a.theta + (a.theta_idx ? (int64_t)a.theta_idx[slot] * a.P : 0);
}
__device__ __forceinline__ float v_perturbed(float th, float s, float n) { return __fadd_rn(th, __fmul_rn(s, n)); }

// ---- per-member GEMM: out[slot][m][n] = sum_k X[slot][m][k] * (theta_w + s*noise)[k][n] + bias_n ------------
constexpr int MG_BM = 128, MG_BN = 64, MG_BK = 16, MG_TM = 8, MG_TN = 4, MG_THREADS = 256;

__global__ void __launch_bounds__(MG_THREADS)
member_gemm_kernel(SlotArgs sa, int64_t off_w, int64_t off_b, const float* __restrict__ X, int64_t x_slot_stride,
                   int M, int K, int N, float* __restrict__ out, int64_t out_slot_stride) {
    const int slot = blockIdx.z;
    if (!v_slot_active(sa, slot)) return;
    __shared__ __align__(16) float As[MG_BK][MG_BM];
    __shared__ __align__(16) float Bs[MG_BK][MG_BN];
    const int tid = threadIdx.x;
    const int tx = tid % (MG_BN / MG_TN), ty = tid / (MG_BN / MG_TN);
    const int m0 = blockIdx.y * MG_BM, n0 = blockIdx.x * MG_BN;
    const float* th = v_slot_theta(sa, slot);
    const int64_t idx = sa.noise_idx[slot];
    const float s = sa.scale[slot];
    const float* tw = th + off_w;
    const float* nz = sa.noise + idx + off_w;
    const float* x = X + (int64_t)slot * x_slot_stride;

    float acc[MG_TM][MG_TN];
#pragma unroll
    for (int i = 0; i < MG_TM; ++i)
#pragma unroll
        for (int j = 0; j < MG_TN; ++j) acc[i][j] = 0.0f;

    for (int k0 = 0; k0 < K; k0 += MG_BK) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {                       // A: 128 x 16 = 512 float4 units
            const int u = tid + i * MG_THREADS;
            const int ml = u % MG_BM, kq = u / MG_BM;
            const int m = m0 + ml, k = k0 + 4 * kq;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < M && k < K) v = *reinterpret_cast<const float4*>(x + (int64_t)m * K + k);
            As[4 * kq + 0][ml] = v.x;
            As[4 * kq + 1][ml] = v.y;
            As[4 * kq + 2][ml] = v.z;
            As[4 * kq + 3][ml] = v.w;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {                       // B: 16 x 64 member weights
            const int e = tid + i * MG_THREADS;
            const int kl = e / MG_BN, nl = e % MG_BN;
            const int k = k0 + kl, n = n0 + nl;
            float w = 0.0f;
            if (k < K && n < N) {
                const int64_t f = (int64_t)k * N + n;
                w = v_perturbed(tw[f], s, nz[f]);
            }
            Bs[kl][nl] = w;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < MG_BK; ++k) {
            float a[MG_TM], b[MG_TN];
            const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * MG_TM]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[k][ty * MG_TM + 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][tx * MG_TN]);
            a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
            b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w;
#pragma unroll
            for (int i = 0; i < MG_TM; ++i)
#pragma unroll
                for (int j = 0; j < MG_TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
    float* o = out + (int64_t)slot * out_slot_stride;
#pragma unroll
    for (int j = 0; j < MG_TN; ++j) {
        const int n = n0 + tx * MG_TN + j;
        if (n >= N) continue;
        const float bias = (off_b >= 0) ? v_perturbed(th[off_b + n], s, sa.noise[idx + off_b + n]) : 0.0f;
#pragma unroll
        for (int i = 0; i < MG_TM; ++i) {
            const int m = m0 + ty * MG_TM + i;
            if (m < M) o[(int64_t)m * N + n] = acc[i][j] + bias;
        }
    }
}

// ---- batch statistics: mean and biased variance per (slot, channel) over `rows` rows ---------------------------
// grid (ceil(C/32), n_slots), 256 threads = 8 row-readers x 32 channels; float64 accumulation, two passes.
__global__ void __launch_bounds__(256)
vbn_stats_kernel(SlotArgs sa, const float* __restrict__ Y, int64_t y_slot_stride, int rows, int C,
                 float* __restrict__ vbn, int vbn_len, int bn_off) {
    const int slot = blockIdx.y;
    if (!v_slot_active(sa, slot)) return;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int c = blockIdx.x * 32 + lane;
    const float* y = Y + (int64_t)slot * y_slot_stride;
    __shared__ double sh[8][33];
    double sum = 0.0;
    if (c < C)
        for (int r = w; r < rows; r += 8) sum += (double)y[(int64_t)r * C + c];
    sh[w][lane] = sum;
    __syncthreads();
    double mean = 0.0;
    for (int i = 0; i < 8; ++i) mean += sh[i][lane];
    mean /= (double)rows;
    const float mean_f = (float)mean;
    __syncthreads();
    double ss = 0.0;
    if (c < C)
        for (int r = w; r < rows; r += 8) {
            const double d = (double)y[(int64_t)r * C + c] - (double)mean_f;
            ss += d * d;
        }
    sh[w][lane] = ss;
    __syncthreads();
    if (w == 0 && c < C) {
        double v = 0.0;
        for (int i = 0; i < 8; ++i) v += sh[i][lane];
        float* st = vbn + (int64_t)slot * vbn_len + bn_off;
        st[c] = mean_f;
        st[C + c] = (float)(v / (double)rows);
    }
}


// ---- batch statistics, r02: coalesced, many CTAs per member ------------------------------------------------------
// vbn_stats_partial_kernel: grid (VS_SPLIT, n_slots); CTA (sp, slot) reads a contiguous range of the member's rows as float4
// units (thread t keeps channel quad t % (C/4): C/4 divides 256 for the policies' channel counts 16 / 32 / 64 / 256 / 512) and
// accumulates sum and sum of squares in float64; fixed-order block reduction -> red[slot][sp][2][C] doubles.
// vbn_stats_final_kernel: adds the VS_SPLIT partials in index order; mean = S1/rows, var = S2/rows - mean^2 in float64
// (the two-pass form of vbn_stats_kernel, kept for C % 4 != 0, differs from it by (mean - fl(mean))^2 ~ 1e-15).
constexpr int VS_SPLIT = 16;
__global__ void __launch_bounds__(256)
vbn_stats_partial_kernel(SlotArgs sa, const float* __restrict__ Y, int64_t y_slot_stride, int rows, int C,
                         double* __restrict__ red) {
    const int slot = blockIdx.y, sp = blockIdx.x;
    if (!v_slot_active(sa, slot)) return;
    const int Q = C >> 2;                                  // channel quads per row
    const int64_t units = (int64_t)rows * Q;
    const int64_t per = ((units + VS_SPLIT - 1) / VS_SPLIT + 255) / 256 * 256;      // multiple of 256: a thread keeps its quad
    const int64_t u0 = (int64_t)sp * per, u1 = min(units, u0 + per);
    const float4* y = reinterpret_cast<const float4*>(Y + (int64_t)slot * y_slot_stride);
    double s1[4] = {0.0, 0.0, 0.0, 0.0}, s2[4] = {0.0, 0.0, 0.0, 0.0};
    for (int64_t u = u0 + threadIdx.x; u < u1; u += 256) {
        const float4 v = y[u];
        s1[0] += v.x; s1[1] += v.y; s1[2] += v.z; s1[3] += v.w;
        s2[0] += (double)v.x * v.x; s2[1] += (double)v.y * v.y; s2[2] += (double)v.z * v.z; s2[3] += (double)v.w * v.w;
    }
    __shared__ double sh[256][8];
#pragma unroll
    for (int j = 0; j < 4; ++j) { sh[threadIdx.x][j] = s1[j]; sh[threadIdx.x][4 + j] = s2[j]; }
    __syncthreads();
    // thread c < C owns channel c: quad c / 4 is held by the threads t = c / 4 (mod Q)
    for (int c = threadIdx.x; c < C; c += 256) {
        double a = 0.0, b = 0.0;
        for (int t = c >> 2; t < 256; t += Q) { a += sh[t][c & 3]; b += sh[t][4 + (c & 3)]; }
        double* r = red + (((int64_t)slot * VS_SPLIT + sp) * 2) * C;
        r[c] = a;
        r[C + c] = b;
    }
}

__global__ void vbn_stats_final_kernel(SlotArgs sa, const double* __restrict__ red, int rows, int C, float* __restrict__ vbn,
                                       int vbn_len, int bn_off) {
    const int slot = blockIdx.x;
    if (!v_slot_active(sa, slot)) return;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        double a = 0.0, b = 0.0;
        for (int sp = 0; sp < VS_SPLIT; ++sp) {
            const double* r = red + (((int64_t)slot * VS_SPLIT + sp) * 2) * C;
            a += r[c];
            b += r[C + c];
        }
        const double mean = a / (double)rows;
        double var = b / (double)rows - mean * mean;
        if (var < 0.0) var = 0.0;
        float* st = vbn + (int64_t)slot * vbn_len + bn_off;
        st[c] = (float)mean;
        st[C + c] = (float)var;
    }
}

// ---- normalise + scale/shift + activation in place --------------------------------------------------------------
__global__ void __launch_bounds__(256)
vbn_apply_kernel(SlotArgs sa, float* __restrict__ Y, int64_t y_slot_stride, int64_t elems, int C, int act,
                 int64_t off_beta, int64_t off_gamma, const float* __restrict__ vbn, int vbn_len, int bn_off) {
    const int slot = blockIdx.y;
    if (!v_slot_active(sa, slot)) return;
    const float* th = v_slot_theta(sa, slot);
    const int64_t idx = sa.noise_idx[slot];
    const float s = sa.scale[slot];
    const float* st = vbn + (int64_t)slot * vbn_len + bn_off;
    float* y = Y + (int64_t)slot * y_slot_stride;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < elems; e += (int64_t)gridDim.x * blockDim.x) {
        const int c = (int)(e % C);
        const float inv = __fdiv_rn(1.0f, __fsqrt_rn(st[C + c] + 1e-3f));
        // off_gamma < 0: ModelVirtualBN flavour (batchnorm.py:85-93): no gamma, off_beta is the post-normalisation bias 'b'
        const float gamma = off_gamma >= 0 ? v_perturbed(th[off_gamma + c], s, sa.noise[idx + off_gamma + c]) : 1.0f;
        const float beta = v_perturbed(th[off_beta + c], s, sa.noise[idx + off_beta + c]);
        y[e] = apply_act((y[e] - st[c]) * inv * gamma + beta, act);
    }
}

__global__ void act_inplace_kernel(float* __restrict__ y, int64_t total, int act) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total) y[i] = apply_act(y[i], act);
}

// ---- normalise + scale/shift + activation, written as the next conv layer's space-to-depth image -----------------
// One CTA per virtual slot (member * n_ref + image).  Same arithmetic as vbn_apply_kernel; same image layout as the
// next_img branch of the conv_s2d epilogue: img[channel-octet plane][pixel][8 x fp16], hi planes then lo planes per
// 16-channel group, zero padding written for the pixels no output maps to.
struct VbnImgGeom { int nS, nPADB, nW, nPIXP, nHP; };
__global__ void __launch_bounds__(256)
vbn_image_kernel(SlotArgs sa, const float* __restrict__ Y, int64_t y_vslot_stride, int n_ref, int HOUT, int C, int act, int bn,
                 int64_t off_beta, int64_t off_gamma, const float* __restrict__ vbn, int vbn_len, int bn_off,
                 float* __restrict__ img, int64_t img_vslot_stride, VbnImgGeom g) {
    const int v = blockIdx.x, slot = v / n_ref;
    if (!v_slot_active(sa, slot)) return;
    __shared__ float s_mean[64], s_inv[64], s_gamma[64], s_beta[64];
    const float* th = v_slot_theta(sa, slot);
    const int64_t idx = sa.noise_idx[slot];
    const float s = sa.scale[slot];
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float mean = 0.0f, inv = 1.0f, gamma = 1.0f, beta = 0.0f;
        if (bn != DNE_BN_NONE) {
            const float* st = vbn + (int64_t)slot * vbn_len + bn_off;
            mean = st[c];
            inv = __fdiv_rn(1.0f, __fsqrt_rn(st[C + c] + 1e-3f));
            gamma = off_gamma >= 0 ? v_perturbed(th[off_gamma + c], s, sa.noise[idx + off_gamma + c]) : 1.0f;
            beta = v_perturbed(th[off_beta + c], s, sa.noise[idx + off_beta + c]);
        }
        s_mean[c] = mean; s_inv[c] = inv; s_gamma[c] = gamma; s_beta[c] = beta;
    }
    __syncthreads();
    const float* y = Y + (int64_t)v * y_vslot_stride;
    uint4* out = reinterpret_cast<uint4*>(img + (int64_t)v * img_vslot_stride);
    const int no = C / 8;
    // zero padding of the image: pixels (Yp, Xp) of the padded grid that no output maps to
    for (int b = threadIdx.x; b < g.nHP * g.nHP; b += blockDim.x) {
        const int Yp = b / g.nHP, Xp = b - Yp * g.nHP;
        if (Yp >= g.nPADB && Yp < g.nPADB + HOUT && Xp >= g.nPADB && Xp < g.nPADB + HOUT) continue;
        const int pix = (Yp / g.nS) * g.nW + (Xp / g.nS), pp = (Yp % g.nS) * g.nS + (Xp % g.nS);
        for (int q = 0; q < no; ++q) {
            const int co = pp * no + q;
            uint4* p = out + (size_t)((co >> 1) * 4 + (co & 1)) * g.nPIXP + pix;
            p[0] = make_uint4(0u, 0u, 0u, 0u);
            p[(size_t)2 * g.nPIXP] = make_uint4(0u, 0u, 0u, 0u);
        }
    }
    for (int u = threadIdx.x; u < HOUT * HOUT * no; u += blockDim.x) {
        const int m = u / no, q = u - m * no;
        const int oy = m / HOUT, ox = m - oy * HOUT;
        const float4 a = *reinterpret_cast<const float4*>(y + (int64_t)m * C + 8 * q);
        const float4 b = *reinterpret_cast<const float4*>(y + (int64_t)m * C + 8 * q + 4);
        float e[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = 8 * q + j;
            float r = e[j];
            if (bn != DNE_BN_NONE) r = (r - s_mean[c]) * s_inv[c] * s_gamma[c] + s_beta[c];
            e[j] = apply_act(r, act);
        }
        uint4 hi, lo;
        wg::split_f16x8(e, hi, lo);
        const int Yp = oy + g.nPADB, Xp = ox + g.nPADB;
        const int pix = (Yp / g.nS) * g.nW + (Xp / g.nS), pp = (Yp % g.nS) * g.nS + (Xp % g.nS);
        const int co = pp * no + q;
        uint4* p = out + (size_t)((co >> 1) * 4 + (co & 1)) * g.nPIXP + pix;
        p[0] = hi;
        p[(size_t)2 * g.nPIXP] = lo;
    }
}

static int64_t v_layer_out_elems(const dne_layer_desc& L) {
    return L.kind == DNE_CONV ? (int64_t)L.hout * L.hout * L.cout : (int64_t)L.cout;
}

static int last_bn_layer(const dne_net_desc* net) {
    int last = -1;
    for (int l = 0; l < net->n_layers; ++l)
        if (net->layers[l].bn != DNE_BN_NONE) last = l;
    return last;
}

// Workspace layout of the pass: per layer the raw / normalised NHWC output [n_slots][n_ref][elems] and, on the s2d path,
// the space-to-depth image of every conv layer that follows a conv layer [n_slots * n_ref][image].  The size does not depend
// on dne_set_option("conv_tc"): the image regions are always reserved when the shapes allow the s2d path.
struct VbnPlan {
    bool s2d_shapes;                       // every conv layer up to the last BN layer has an s2d instantiation
    int last;
    size_t out_off[DNE_MAX_LAYERS], img_off[DNE_MAX_LAYERS], red_off, total;
};
static VbnPlan vbn_plan(const dne_net_desc* net, int n_slots, int n_ref) {
    VbnPlan p{};
    p.last = last_bn_layer(net);
    p.s2d_shapes = p.last >= 0;
    for (int l = 0; l <= p.last; ++l)
        if (net->layers[l].kind == DNE_CONV && !dne_s2d_supported(net->layers[l], l == 0)) p.s2d_shapes = false;
    size_t off = 0;
    for (int l = 0; l <= p.last; ++l) {
        p.out_off[l] = off;
        off += align_up((size_t)n_slots * n_ref * v_layer_out_elems(net->layers[l]) * sizeof(float), 256);
    }
    for (int l = 1; l <= p.last; ++l) {
        p.img_off[l] = 0;
        if (p.s2d_shapes && net->layers[l].kind == DNE_CONV && net->layers[l - 1].kind == DNE_CONV) {
            p.img_off[l] = off;
            off += align_up((size_t)n_slots * n_ref * dne_s2d_image_bytes(net->layers[l]), 256);
        }
    }
    int cmax = 1;
    for (int l = 0; l <= p.last; ++l) cmax = net->layers[l].cout > cmax ? net->layers[l].cout : cmax;
    p.red_off = off;                                       // float64 partial sums of the statistics: [n_slots][VS_SPLIT][2][C]
    off += align_up((size_t)n_slots * VS_SPLIT * 2 * cmax * sizeof(double), 256);
    p.total = off;
    return p;
}

extern "C" int dne_vbn_ws_bytes(const dne_net_desc* net, int n_slots, int n_ref, size_t* out_bytes) {
    DNE_CHECK_ARG(net && out_bytes && n_slots >= 0 && n_ref >= 1, "bad arguments");
    *out_bytes = vbn_plan(net, n_slots, n_ref).total;
    return DNE_OK;
}

extern "C" int dne_vbn_reference_pass(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                                      const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                      const uint8_t* d_active, int n_slots, const uint8_t* d_ref, int n_ref,
                                      float* d_vbn, void* d_ws, size_t ws_bytes, void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_ref && d_vbn && d_ws, "null pointer");
    DNE_CHECK_ARG(((uintptr_t)d_theta & 15) == 0, "d_theta must be 16-byte aligned");
    DNE_CHECK_ARG(net->ob_kind == DNE_OB_ATARI_U8 && n_ref >= 1 && n_slots >= 0, "bad arguments");
    if (n_slots == 0) return DNE_OK;
    const VbnPlan vp = vbn_plan(net, n_slots, n_ref);
    const int last = vp.last;
    DNE_CHECK_ARG(last >= 0 && net->vbn_len > 0, "net has no batch-norm layers");
    if (ws_bytes < vp.total) {
        dne_set_error("dne_vbn_reference_pass: workspace too small (%zu < %zu)", ws_bytes, vp.total);
        return DNE_ERR_WS;
    }
    DNE_CHECK_ARG(((uintptr_t)d_ws & 255) == 0, "d_ws must be 256-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    SlotArgs sa;
    sa.theta = d_theta;
    sa.noise = ctx->noise;
    sa.noise_idx = d_noise_idx;
    sa.scale = d_scale;
    sa.theta_idx = d_theta_idx;
    sa.active = d_active;
    sa.P = net->num_params;

    const bool s2d = vp.s2d_shapes && g_dne_conv_tc == 2 && (int64_t)n_slots * n_ref < (int64_t)1 << 30;
    const int n_virtual = n_slots * n_ref;
    char* ws = (char*)d_ws;
    const void* cur = d_ref;              // NHWC floats [n_slots][n_ref][cur_elems] (layer 0: the shared uint8 batch)
    const float* cur_img = nullptr;       // s2d path: the layer's input as space-to-depth images [n_slots * n_ref][image]
    int64_t cur_elems = 84 * 84 * 4;      // per image
    bool cur_u8 = true;
    for (int l = 0; l <= last; ++l) {
        const dne_layer_desc& L = net->layers[l];
        const int64_t oe = v_layer_out_elems(L);
        float* out = (float*)(ws + vp.out_off[l]);
        const int64_t out_slot_stride = (int64_t)n_ref * oe;
        LayerEpi epi;                      // raw pre-BN output: bias only
        const int64_t pre_b = (L.bn == DNE_BN_GPU) ? -1 : L.off_b;   // ModelVirtualBN layers have no pre-normalisation bias
        epi.off_b = pre_b; epi.off_beta = -1; epi.off_gamma = -1;
        epi.act = DNE_ACT_NONE; epi.bn = DNE_BN_NONE; epi.bn_off = 0; epi.vbn_len = 0; epi.vbn = nullptr;
        if (L.kind == DNE_CONV) {
            DNE_CHECK_ARG((int64_t)L.hin * L.hin * L.cin == cur_elems, "conv layer input size mismatch");
            int rc;
            if (s2d) {
                // n_slots * n_ref virtual slots (member = v / n_ref); layer 0 reads frame v % n_ref of the SHARED batch
                const void* in = cur_u8 ? cur : (const void*)cur_img;
                const int64_t in_stride = cur_u8 ? cur_elems : (int64_t)(dne_s2d_image_bytes(L) / sizeof(float));
                DNE_CHECK_ARG(cur_u8 || cur_img, "s2d conv layer without an input image");
                rc = dne_launch_conv_layer_s2d(sa, L, epi, cur_u8, in, in_stride, out, oe, nullptr, n_virtual, ctx->sm_count, st,
                                               nullptr, n_ref, cur_u8 ? n_ref : 0);
            } else {
                // layer 0 reads the SHARED reference batch (slot stride 0); later layers read the member's own buffer
                const int64_t in_slot_stride = cur_u8 ? 0 : (int64_t)n_ref * cur_elems;
                rc = dne_launch_conv_layer(sa, L, epi, cur_u8, cur, in_slot_stride, cur_elems, out, out_slot_stride, oe, n_slots,
                                           n_ref, st);
            }
            if (rc) {
                dne_set_error("dne_vbn_reference_pass: conv layer %d shape not compiled in", l);
                return rc;
            }
        } else {
            DNE_CHECK_ARG(!cur_u8 && L.cin == cur_elems && L.cin % 4 == 0, "dense layer input mismatch");
            // tensor cores (wgmma, 3xTF32: tc_conv.cu member_gemm_tc_kernel) unless conv_tc = 0 selects the fp32 SIMT referee
            if (!(g_dne_conv_tc && dne_launch_member_gemm_tc(sa, L.off_w, pre_b, (const float*)cur, (int64_t)n_ref * cur_elems, n_ref,
                                                             L.cin, L.cout, out, out_slot_stride, n_slots, st) == 0)) {
                dim3 grid((L.cout + MG_BN - 1) / MG_BN, (n_ref + MG_BM - 1) / MG_BM, n_slots);
                member_gemm_kernel<<<grid, MG_THREADS, 0, st>>>(sa, L.off_w, pre_b, (const float*)cur,
                                                               (int64_t)n_ref * cur_elems, n_ref, L.cin, L.cout, out,
                                                               out_slot_stride);
            }
            DNE_LAUNCHED(1);
        }
        DNE_LAUNCH_CHECK();
        const int C = L.cout;
        const int rows = (int)(out_slot_stride / C);
        if (L.bn != DNE_BN_NONE) {
            if (C % 4 == 0 && 256 % (C / 4) == 0 && (out_slot_stride & 3) == 0 && g_dne_conv_tc != 0) {
                double* red = (double*)(ws + vp.red_off);
                vbn_stats_partial_kernel<<<dim3(VS_SPLIT, n_slots), 256, 0, st>>>(sa, out, out_slot_stride, rows, C, red);
                DNE_LAUNCH_CHECK1();
                vbn_stats_final_kernel<<<n_slots, 256, 0, st>>>(sa, red, rows, C, d_vbn, net->vbn_len, L.bn_off);
            } else {                                        // referee (conv_tc = 0) and odd channel counts: two-pass kernel
                vbn_stats_kernel<<<dim3((C + 31) / 32, n_slots), 256, 0, st>>>(sa, out, out_slot_stride, rows, C, d_vbn,
                                                                              net->vbn_len, L.bn_off);
            }
            DNE_LAUNCH_CHECK1();
        }
        cur_img = nullptr;
        if (l < last) {
            const bool to_image = s2d && L.kind == DNE_CONV && vp.img_off[l + 1] != 0 && C % 8 == 0 && C <= 64;
            if (s2d && net->layers[l + 1].kind == DNE_CONV) DNE_CHECK_ARG(to_image, "s2d path: conv layer after a non-conv layer");
            if (to_image) {
                VbnImgGeom g;
                dne_s2d_image_geom(net->layers[l + 1], &g.nS, &g.nPADB, &g.nW, &g.nPIXP, &g.nHP);
                float* img = (float*)(ws + vp.img_off[l + 1]);
                vbn_image_kernel<<<n_virtual, 256, 0, st>>>(sa, out, oe, n_ref, L.hout, C, L.act, L.bn,
                                                           L.bn == DNE_BN_GPU ? L.off_b : L.off_beta,
                                                           L.bn == DNE_BN_GPU ? (int64_t)-1 : L.off_gamma, d_vbn, net->vbn_len,
                                                           L.bn_off, img, (int64_t)(dne_s2d_image_bytes(net->layers[l + 1]) / sizeof(float)), g);
                DNE_LAUNCH_CHECK1();
                cur_img = img;
            } else if (L.bn != DNE_BN_NONE) {
                const int gx = (int)((out_slot_stride + 255) / 256 < 1024 ? (out_slot_stride + 255) / 256 : 1024);
                vbn_apply_kernel<<<dim3(gx, n_slots), 256, 0, st>>>(sa, out, out_slot_stride, out_slot_stride, C,
                                                                   L.act, L.bn == DNE_BN_GPU ? L.off_b : L.off_beta,
                                                                   L.bn == DNE_BN_GPU ? (int64_t)-1 : L.off_gamma, d_vbn,
                                                                   net->vbn_len, L.bn_off);
                DNE_LAUNCH_CHECK1();
            } else if (L.act != DNE_ACT_NONE) {
                const int64_t total = (int64_t)n_slots * out_slot_stride;
                act_inplace_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(out, total, L.act);
                DNE_LAUNCH_CHECK1();
            }
        }
        cur = out;
        cur_elems = oe;
        cur_u8 = false;
    }
    return DNE_OK;
}
