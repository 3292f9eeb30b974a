// dne_api.cu -- C ABI of libdne.so: context, error reporting, forward orchestration (include/dne.h).
#include "common.cuh"
#include "forward.cuh"

static thread_local char g_err[512] = "";
unsigned long long g_dne_launches = 0;
int g_dne_theta_tma = 1;     // TMA-fed shared-theta GEMM when a prepared region is current (dne_set_option("theta_tma", v))
int g_dne_chain_ticks = 0;   // the first conv layer of a tick is a dependent launch too (dne_set_option("chain_ticks", v); see conv_s2d.cu)
int g_dne_pdl = 1;           // programmatic dependent launch of the tick's kernel chain (common.cuh; dne_set_option("pdl", v))
int g_dne_fold_theta = 1;    // fold the theta GEMM's split-K partials into the noise GEMV's output (dne_set_option("fold_theta", v))
int g_dne_fuse_head = 1;     // combine + output head in one kernel (dne_set_option("fuse_head", v))

void dne_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char* dne_last_error(void) { return g_err; }
extern "C" int dne_version(void) { return 100; }
extern "C" int dne_abi_sizes(int* layer_desc_bytes, int* net_desc_bytes) {
    if (layer_desc_bytes) *layer_desc_bytes = (int)sizeof(dne_layer_desc);
    if (net_desc_bytes) *net_desc_bytes = (int)sizeof(dne_net_desc);
    return DNE_OK;
}
extern "C" int dne_abi_maze_size(int* maze_desc_bytes) {
    if (maze_desc_bytes) *maze_desc_bytes = (int)sizeof(dne_maze_desc);
    return DNE_OK;
}

extern "C" int dne_ctx_create(int device, dne_ctx** out) {
    DNE_CHECK_ARG(out, "out is null");
    *out = nullptr;
    int n = 0;
    DNE_CUDA(cudaGetDeviceCount(&n));
    DNE_CHECK_ARG(device >= 0 && device < n, "no such CUDA device");
    DNE_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    DNE_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        dne_set_error("dne_ctx_create: device %d is sm_%d%d; libdne is built for sm_90a (H100) only", device,
                      prop.major, prop.minor);
        return DNE_ERR_CUDA;
    }
    dne_ctx* c = new dne_ctx();
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    c->noise = nullptr;
    c->noise_count = 0;
    c->scratch = nullptr;
    c->ev = nullptr;
    c->ev_cap = c->ev_n = c->prof_on = 0;
    c->ev_wait = c->ev_record = nullptr;
    c->ev_record_done = 0;
    c->ev_mode = 0;
    for (int i = 0; i < DNE_MAX_PREP; ++i) c->prep[i].ws = nullptr, c->prep[i].theta = nullptr;
    cudaError_t e = cudaMalloc(&c->scratch, sizeof(double) * DNE_SCRATCH_DOUBLES);
    if (e != cudaSuccess) {
        delete c;
        dne_set_error("dne_ctx_create: cudaMalloc -> %s", cudaGetErrorString(e));
        return DNE_ERR_CUDA;
    }
    *out = c;
    return DNE_OK;
}

extern "C" int dne_ctx_destroy(dne_ctx* ctx) {
    if (!ctx) return DNE_OK;
    cudaSetDevice(ctx->device);
    if (ctx->scratch) cudaFree(ctx->scratch);
    if (ctx->ev) {
        for (int i = 0; i < 2 * ctx->ev_cap; ++i) cudaEventDestroy(ctx->ev[i]);
        delete[] ctx->ev;
    }
    delete ctx;
    return DNE_OK;
}

// Runtime switches: "conv_tc" (2 = shifted-window wgmma convolutions [default], 1 = im2col-staged wgmma, 0 = fp32 SIMT).
extern "C" int dne_set_option(const char* name, int value) {
    DNE_CHECK_ARG(name, "name is null");
    if (strcmp(name, "conv_tc") == 0 && value >= 0 && value <= 2) { g_dne_conv_tc = value; return DNE_OK; }
    if (strcmp(name, "gemv_bulk") == 0) { g_dne_gemv_bulk = value ? 1 : 0; return DNE_OK; }
    if (strcmp(name, "fuse_head") == 0) { g_dne_fuse_head = value ? 1 : 0; return DNE_OK; }
    if (strcmp(name, "theta_mc") == 0) { extern int g_dne_theta_mc; g_dne_theta_mc = value ? 1 : 0; return DNE_OK; }
    if (strcmp(name, "theta_tma") == 0) { g_dne_theta_tma = value ? 1 : 0; return DNE_OK; }
    if (strcmp(name, "gemv_stages") == 0 && value >= 2 && value <= 8) { extern int g_dne_gemv_stages; g_dne_gemv_stages = value; return DNE_OK; }
    if (strcmp(name, "fold_theta") == 0 && value >= 0 && value <= 1) { g_dne_fold_theta = value; return DNE_OK; }
    if (strcmp(name, "chain_ticks") == 0 && value >= 0 && value <= 1) { g_dne_chain_ticks = value; return DNE_OK; }
    if (strcmp(name, "pdl") == 0 && value >= 0 && value <= 1) { g_dne_pdl = value; return DNE_OK; }
    if (strcmp(name, "gemv_grid") == 0 && value >= 0) { extern int g_dne_gemv_grid; g_dne_gemv_grid = value; return DNE_OK; }
    if (strcmp(name, "gemv_ctas_per_sm") == 0 && value >= 1 && value <= 2) { g_dne_gemv_ctas_per_sm = value; return DNE_OK; }
    dne_set_error("dne_set_option: unknown option '%s'", name);
    return DNE_ERR_ARG;
}

// ---- measurement hooks -------------------------------------------------------------------------------
extern "C" long long dne_launch_count(int reset) {
    const long long v = (long long)g_dne_launches;
    if (reset) g_dne_launches = 0;
    return v;
}

// Time every dense_noise_gemv launch (the HBM-bound kernel) with CUDA events on the launching stream, up to
// `capacity` launches.  on = 0 stops recording; the samples stay readable.
extern "C" int dne_profile_enable(dne_ctx* ctx, int on, int capacity) {
    DNE_CHECK_ARG(ctx, "ctx is null");
    if (on == 2) {                                  // resume after a pause (on = 0): keeps the samples taken so far
        ctx->prof_on = ctx->ev ? 1 : 0;
        return DNE_OK;
    }
    if (on) {
        if (capacity < 1) capacity = 4096;
        if (capacity > ctx->ev_cap) {
            if (ctx->ev) {
                for (int i = 0; i < 2 * ctx->ev_cap; ++i) cudaEventDestroy(ctx->ev[i]);
                delete[] ctx->ev;
            }
            ctx->ev = new cudaEvent_t[2 * (size_t)capacity];
            for (int i = 0; i < 2 * capacity; ++i) DNE_CUDA(cudaEventCreate(&ctx->ev[i]));
            ctx->ev_cap = capacity;
        }
        ctx->ev_n = 0;
    }
    ctx->prof_on = on ? 1 : 0;
    return DNE_OK;
}

// Synchronises the device, then returns the number of timed launches and their summed duration (ms).
extern "C" int dne_profile_read(dne_ctx* ctx, int* n_launches, double* total_ms) {
    DNE_CHECK_ARG(ctx && n_launches && total_ms, "bad arguments");
    DNE_CUDA(cudaDeviceSynchronize());
    double tot = 0.0;
    for (int i = 0; i < ctx->ev_n; ++i) {
        float ms = 0.f;
        DNE_CUDA(cudaEventElapsedTime(&ms, ctx->ev[2 * i], ctx->ev[2 * i + 1]));
        tot += ms;
    }
    *n_launches = ctx->ev_n;
    *total_ms = tot;
    return DNE_OK;
}

extern "C" int dne_noise_bind(dne_ctx* ctx, const float* d_noise, int64_t count) {
    DNE_CHECK_ARG(ctx && d_noise && count > 0, "bad arguments");
    DNE_CHECK_ARG(((uintptr_t)d_noise & 15) == 0, "noise table must be 16-byte aligned");
    ctx->noise = d_noise;
    ctx->noise_count = count;
    return DNE_OK;
}

// ---------------------------------------------------------------------------------------------------
// forward planning: workspace carve-up
// ---------------------------------------------------------------------------------------------------
constexpr int PLAN_SM_COUNT = 132;   // H100 SXM; planning must not depend on a live device (ws query works on CPU)

struct ForwardPlan {
    size_t x0_off;                         // normalised vector observations
    size_t act_off[DNE_MAX_LAYERS];
    int64_t act_elems[DNE_MAX_LAYERS];     // per slot
    DensePlan dense[DNE_MAX_LAYERS];
    size_t part_theta_off, part_noise_off;
    size_t xc_off[DNE_MAX_LAYERS], wc_off[DNE_MAX_LAYERS];   // TMA-fed theta GEMM operands of dense layer l (0 = none)
    size_t total;
};

// dense layer l can take the TMA-fed theta GEMM: it directly follows a shifted-window conv layer (whose epilogue writes Xc)
static bool tgm_candidate(const dne_net_desc* net, int l, const DensePlan& dp) {
    if (l == 0 || net->layers[l].kind != DNE_DENSE || net->layers[l - 1].kind != DNE_CONV || !dp.decomposed) return false;
    if (!dne_s2d_supported(net->layers[l - 1], l - 1 == 0)) return false;
    return dne_tgm_supported(net->layers[l].cin, net->layers[l].cout, dp.k_per_split);
}

static int64_t layer_out_elems(const dne_layer_desc& L) {
    return L.kind == DNE_CONV ? (int64_t)L.hout * L.hout * L.cout : (int64_t)L.cout;
}

static int plan_forward(const dne_net_desc* net, int n_slots, int paired, bool shared_theta, ForwardPlan* fp) {
    DNE_CHECK_ARG(net && net->n_layers >= 1 && net->n_layers <= DNE_MAX_LAYERS, "bad net descriptor");
    size_t off = 0;
    fp->x0_off = off;
    if (net->ob_kind == DNE_OB_VECTOR) off += align_up((size_t)n_slots * net->ob_dim * sizeof(float), 256);
    size_t pt = 0, pn = 0;
    for (int l = 0; l < net->n_layers; ++l) {
        const dne_layer_desc& L = net->layers[l];
        fp->act_elems[l] = layer_out_elems(L);
        // conv -> conv hand-off of the s2d path: the producing epilogue writes the NEXT layer's image (space-to-depth,
        // zero padded, TF32 hi/lo planes: conv_s2d.cu), which is larger than the NHWC activation
        if (L.kind == DNE_CONV && l + 1 < net->n_layers && net->layers[l + 1].kind == DNE_CONV) {
            const int64_t img = (int64_t)(dne_s2d_image_bytes(net->layers[l + 1]) / sizeof(float));
            if (img > fp->act_elems[l]) fp->act_elems[l] = img;
        }
        fp->act_off[l] = off;
        off += align_up((size_t)n_slots * fp->act_elems[l] * sizeof(float), 256);
        if (L.kind == DNE_DENSE) {
            const bool head = (l == net->n_layers - 1);
            fp->dense[l] = dne_plan_dense(L, n_slots, head ? -1 : paired, shared_theta, PLAN_SM_COUNT);
            if (fp->dense[l].part_theta_floats > pt) pt = fp->dense[l].part_theta_floats;
            if (fp->dense[l].part_noise_floats > pn) pn = fp->dense[l].part_noise_floats;
        }
    }
    // operands of the TMA-fed theta GEMM: placed BEFORE the partial buffers so that their offsets do not depend on
    // (paired, shared_theta) -- dne_theta_prepare and every later forward call on the workspace must agree on them
    for (int l = 0; l < net->n_layers; ++l) {
        fp->xc_off[l] = fp->wc_off[l] = 0;
        if (!tgm_candidate(net, l, fp->dense[l])) continue;
        fp->xc_off[l] = off;
        off += align_up(dne_tgm_xc_bytes(n_slots, net->layers[l].cin), 256);
        fp->wc_off[l] = off;
        off += align_up(dne_tgm_wc_bytes(net->layers[l].cin, net->layers[l].cout), 256);
    }
    fp->part_theta_off = off;
    off += align_up(pt * sizeof(float), 256);
    fp->part_noise_off = off;
    off += align_up(pn * sizeof(float), 256);
    fp->total = off;
    return DNE_OK;
}

extern "C" int dne_forward_ws_bytes(const dne_net_desc* net, int n_slots, size_t* out_bytes) {
    DNE_CHECK_ARG(out_bytes && n_slots >= 0, "bad arguments");
    size_t best = 0;
    for (int shared = 0; shared < 2; ++shared)
        for (int paired = 0; paired < 3; ++paired) {
            ForwardPlan a;
            int rc = plan_forward(net, n_slots + (n_slots & 1), paired, shared != 0, &a);
            if (rc) return rc;
            if (a.total > best) best = a.total;
        }
    *out_bytes = best;
    return DNE_OK;
}

static LayerEpi make_layer_epi(const dne_layer_desc& L, const dne_net_desc* net, const float* d_vbn) {
    LayerEpi epi;
    epi.off_b = L.off_b;
    epi.off_beta = L.off_beta;
    epi.off_gamma = L.off_gamma;
    epi.act = L.act;
    epi.bn = L.bn;
    epi.bn_off = L.bn_off;
    epi.vbn_len = net->vbn_len;
    epi.vbn = d_vbn;
    return epi;
}

// ---- prepared theta (TMA-fed theta GEMM) ---------------------------------------------------------------------------------
void dne_prep_invalidate_theta(dne_ctx* ctx, const float* d_theta) {
    for (int i = 0; i < DNE_MAX_PREP; ++i)
        if (ctx->prep[i].theta == d_theta) ctx->prep[i].ws = nullptr, ctx->prep[i].theta = nullptr;
}
static bool prep_current(const dne_ctx* ctx, const void* ws, const float* d_theta, int n_slots) {
    for (int i = 0; i < DNE_MAX_PREP; ++i)
        if (ctx->prep[i].ws == ws && ctx->prep[i].theta == d_theta && ctx->prep[i].n_slots == n_slots) return true;
    return false;
}

// Relays out the shared-theta weight matrices of the net's dense layers into the workspace (theta_prep_kernel) for the
// TMA-fed theta GEMM, and remembers (workspace, theta) as current.  Call again whenever theta changes by any means other
// than dne_adam_step / dne_sgd_step on the same context (those invalidate the entry themselves).  Forward calls on a
// workspace without a current entry use the thread-staged GEMM: always correct, ~20 us slower per 256-slot tick.
extern "C" int dne_theta_prepare(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta, int n_slots, void* d_ws,
                                 size_t ws_bytes, void* stream) {
    DNE_CHECK_ARG(ctx && net && d_theta && d_ws && n_slots > 0, "bad arguments");
    DNE_CHECK_ARG(((uintptr_t)d_ws & 255) == 0 && ((uintptr_t)d_theta & 15) == 0, "workspace / theta alignment");
    ForwardPlan fp;
    int rc = plan_forward(net, n_slots, 1, true, &fp);        // the prepared region's offsets do not depend on `paired`
    if (rc) return rc;
    if (ws_bytes < fp.total) {
        dne_set_error("dne_theta_prepare: workspace too small (%zu < %zu)", ws_bytes, fp.total);
        return DNE_ERR_WS;
    }
    for (int i = 0; i < DNE_MAX_PREP; ++i)                     // drop stale entries of this workspace
        if (ctx->prep[i].ws == d_ws) ctx->prep[i].ws = nullptr, ctx->prep[i].theta = nullptr;
    bool any = false;
    for (int l = 0; l < net->n_layers; ++l) {
        if (!fp.wc_off[l]) continue;
        const dne_layer_desc& L = net->layers[l];
        dne_launch_theta_prep(d_theta + L.off_w, L.cin, L.cout, (float*)((char*)d_ws + fp.wc_off[l]), (cudaStream_t)stream);
        DNE_LAUNCH_CHECK();
        any = true;
    }
    if (any) {
        int slot = 0;
        for (int i = 0; i < DNE_MAX_PREP; ++i)
            if (!ctx->prep[i].ws) { slot = i; break; }
        ctx->prep[slot].ws = d_ws;
        ctx->prep[slot].theta = d_theta;
        ctx->prep[slot].n_slots = n_slots;
    }
    return DNE_OK;
}

// Drops the prepared-theta entries of a workspace (call when a workspace is allocated or freed: entries are keyed by
// ADDRESS, and an allocator may hand a freed workspace's address to a new one).
extern "C" int dne_theta_forget(dne_ctx* ctx, const void* d_ws) {
    DNE_CHECK_ARG(ctx, "ctx is null");
    for (int i = 0; i < DNE_MAX_PREP; ++i)
        if (ctx->prep[i].ws == d_ws || d_ws == nullptr) ctx->prep[i].ws = nullptr, ctx->prep[i].theta = nullptr;
    return DNE_OK;
}

static int forward_impl(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta, const int64_t* d_noise_idx,
                        const float* d_scale, const int32_t* d_theta_idx, const uint8_t* d_active, int n_slots,
                        int paired, const void* d_obs, const float* d_ob_mean, const float* d_ob_std,
                        const float* d_vbn, int32_t* d_actions, float* d_out, void* d_ws, size_t ws_bytes,
                        void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_obs && d_ws, "null pointer");
    DNE_CHECK_ARG(n_slots >= 0, "n_slots < 0");
    DNE_CHECK_ARG(paired >= 0 && paired <= 2, "paired must be 0, 1 (pairs share the noise index) or 2 (pairs share the theta row)");
    DNE_CHECK_ARG(!paired || (n_slots % 2 == 0), "paired modes need an even number of slots");
    DNE_CHECK_ARG(paired != 2 || d_theta_idx, "paired == 2 needs d_theta_idx");
    DNE_CHECK_ARG(net->num_params <= ctx->noise_count, "net larger than the noise table");
    DNE_CHECK_ARG(((uintptr_t)d_ws & 255) == 0, "workspace must be 256-byte aligned");
    // the GEMV / conv kernels derive 16-byte alignment of their vector and bulk loads from element indices relative to
    // the theta BASE pointer (rows of a [n_theta, P] matrix may start anywhere: P % 4 != 0 is handled)
    DNE_CHECK_ARG(((uintptr_t)d_theta & 15) == 0, "d_theta must be 16-byte aligned (pass the base of the parameter matrix, not a row view)");
    if (n_slots == 0) return DNE_OK;
    ForwardPlan fp;
    int rc = plan_forward(net, n_slots, paired, d_theta_idx == nullptr, &fp);
    if (rc) return rc;
    if (ws_bytes < fp.total) {
        dne_set_error("forward: workspace too small (%zu < %zu)", ws_bytes, fp.total);
        return DNE_ERR_WS;
    }
    bool needs_vbn = false;
    for (int l = 0; l < net->n_layers; ++l) needs_vbn = needs_vbn || (net->layers[l].bn != DNE_BN_NONE);
    DNE_CHECK_ARG(!needs_vbn || d_vbn, "net has batch-norm layers: d_vbn (dne_vbn_reference_pass) required");

    // conv path: 2 = shifted-window kernels with TMA-fed images between the conv layers (conv_s2d.cu) when every conv
    // layer of the net has a compiled shape; 1 = per-member im2col staging (tc_conv.cu); 0 = fp32 SIMT
    bool use_s2d = (g_dne_conv_tc >= 2) && net->ob_kind == DNE_OB_ATARI_U8;
    for (int l = 0; l < net->n_layers && use_s2d; ++l)
        if (net->layers[l].kind == DNE_CONV) use_s2d = dne_s2d_supported(net->layers[l], l == 0);
    // TMA-fed theta GEMM: only with a current prepared-theta region in THIS workspace for THIS theta (dne_theta_prepare)
    const bool use_tgm = use_s2d && g_dne_theta_tma && d_theta_idx == nullptr && prep_current(ctx, d_ws, d_theta, n_slots);
    cudaStream_t st = (cudaStream_t)stream;
    // phase events (dne_set_phase_events): consumed by this call
    if (ctx->ev_wait && ctx->ev_mode == 0) {
        DNE_CUDA(cudaStreamWaitEvent(st, (cudaEvent_t)ctx->ev_wait, 0));
        ctx->ev_wait = nullptr;
    }
    ctx->ev_record_done = 0;
    char* ws = (char*)d_ws;
    SlotArgs sa;
    sa.theta = d_theta;
    sa.noise = ctx->noise;
    sa.noise_idx = d_noise_idx;
    sa.scale = d_scale;
    sa.theta_idx = d_theta_idx;
    sa.active = d_active;
    sa.P = net->num_params;

    const void* cur = d_obs;
    int64_t cur_elems = net->ob_dim;           // logical elements per slot of the current activation ...
    int64_t cur_stride = net->ob_dim;          // ... and the slot stride of the buffer that holds it
    bool cur_u8 = (net->ob_kind == DNE_OB_ATARI_U8);
    if (net->ob_kind == DNE_OB_VECTOR) {
        float* x0 = (float*)(ws + fp.x0_off);
        dne_launch_ob_norm((const float*)d_obs, d_ob_mean, d_ob_std, (int64_t)n_slots * net->ob_dim, net->ob_dim,
                           x0, st);
        DNE_LAUNCH_CHECK();
        cur = x0;
    } else {
        cur_elems = cur_stride = 84 * 84 * 4;
    }
    for (int l = 0; l < net->n_layers; ++l) {
        const dne_layer_desc& L = net->layers[l];
        const bool last = (l == net->n_layers - 1);
        float* out = (float*)(ws + fp.act_off[l]);
        int64_t out_stride = fp.act_elems[l];
        if (last && d_out) { out = d_out; out_stride = net->n_out; }
        const LayerEpi epi = make_layer_epi(L, net, d_vbn);
        if (L.kind == DNE_CONV && use_s2d) {
            const dne_layer_desc* next = (!last && net->layers[l + 1].kind == DNE_CONV) ? &net->layers[l + 1] : nullptr;
            float* xc = (use_tgm && !last && fp.xc_off[l + 1]) ? (float*)(ws + fp.xc_off[l + 1]) : nullptr;
            rc = dne_launch_conv_layer_s2d(sa, L, epi, cur_u8, cur, cur_stride, out, out_stride, next, n_slots,
                                           ctx->sm_count, st, xc);
            if (rc) {
                dne_set_error("forward: s2d conv layer %d launch failed (%d)", l, rc);
                return rc;
            }
        } else if (L.kind == DNE_CONV) {
            DNE_CHECK_ARG((int64_t)L.hin * L.hin * L.cin == cur_elems, "conv layer input size mismatch");
            rc = dne_launch_conv_layer(sa, L, epi, cur_u8, cur, cur_stride, 0, out, out_stride, 0, n_slots, 1, st);
            if (rc) {
                dne_set_error("forward: conv layer %d shape not compiled in (cin %d cout %d k %d s %d hin %d)", l,
                              L.cin, L.cout, L.ksize, L.stride, L.hin);
                return rc;
            }
        } else {
            DNE_CHECK_ARG(!cur_u8, "dense layer cannot read uint8 observations");
            DNE_CHECK_ARG(L.cin == cur_elems, "dense layer input size mismatch");
            // the output head rides in the combine kernel of the layer before it (one launch less per tick)
            DenseHead head;
            const bool fuse = g_dne_fuse_head && l + 2 == net->n_layers && net->layers[l + 1].kind == DNE_DENSE &&
                              dne_head_fusable(L, fp.dense[l], net->layers[l + 1], fp.dense[l + 1]);
            if (fuse) {
                head.L = &net->layers[l + 1];
                head.epi = make_layer_epi(net->layers[l + 1], net, d_vbn);
                head.out = d_out ? d_out : (float*)(ws + fp.act_off[l + 1]);
                head.out_slot_stride = d_out ? net->n_out : fp.act_elems[l + 1];
                head.actions = d_actions;
            }
            TgmOperands tgm;
            const bool tg = use_tgm && fp.xc_off[l] && fp.dense[l].Gt == 0;
            if (tg) {
                tgm.Xc = (const float*)(ws + fp.xc_off[l]);
                tgm.Wc = (const float*)(ws + fp.wc_off[l]);
            }
            rc = dne_launch_dense_layer(ctx, sa, L, epi, fp.dense[l], (const float*)cur, cur_stride, out, out_stride,
                                        last ? d_actions : nullptr, (float*)(ws + fp.part_theta_off),
                                        (float*)(ws + fp.part_noise_off), n_slots, st, fuse ? &head : nullptr,
                                        tg ? &tgm : nullptr);
            if (rc == 0 && fuse) {
                DNE_LAUNCH_CHECK();
                break;                                           // the head layer is done
            }
            if (rc) {
                dne_set_error("forward: dense layer %d (%d x %d) not supported", l, L.cin, L.cout);
                return rc;
            }
        }
        DNE_LAUNCH_CHECK();
        cur = out;
        cur_elems = layer_out_elems(L);
        cur_stride = out_stride;
        cur_u8 = false;
    }
    if (ctx->ev_record && !ctx->ev_record_done) DNE_CUDA(cudaEventRecord((cudaEvent_t)ctx->ev_record, st));
    ctx->ev_record = nullptr;
    ctx->ev_wait = nullptr;
    return DNE_OK;
}

// Phase-shifted double buffering of two slot tables on two streams: the NEXT forward call on `ctx` first makes its
// stream wait for `wait_event` (nullable) and records `record_event` (nullable) right before its first HBM-bound noise
// GEMV.  With table A recording eA / waiting eB and table B recording eB / waiting eA, the compute-bound conv phase
// of one table runs under the HBM-bound GEMV of the other instead of both tables doing the same phase in lockstep.
extern "C" int dne_set_phase_events(dne_ctx* ctx, void* wait_event, void* record_event, int mode) {
    DNE_CHECK_ARG(ctx && (mode == 0 || mode == 1), "bad arguments");
    ctx->ev_wait = wait_event;
    ctx->ev_record = record_event;
    ctx->ev_record_done = 0;
    ctx->ev_mode = mode;
    return DNE_OK;
}

extern "C" int dne_perturb_forward_conv(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                                        const int64_t* d_noise_idx, const float* d_scale,
                                        const int32_t* d_theta_idx, const uint8_t* d_active, int n_slots, int paired,
                                        const uint8_t* d_obs, const float* d_vbn, int32_t* d_actions,
                                        float* d_logits, void* d_ws, size_t ws_bytes, void* stream) {
    DNE_CHECK_ARG(net && net->ob_kind == DNE_OB_ATARI_U8, "net must take uint8 Atari observations");
    DNE_CHECK_ARG(net->layers[net->n_layers - 1].kind == DNE_DENSE, "last layer must be dense");
    return forward_impl(ctx, net, d_theta, d_noise_idx, d_scale, d_theta_idx, d_active, n_slots, paired, d_obs,
                        nullptr, nullptr, d_vbn, d_actions, d_logits, d_ws, ws_bytes, stream);
}

// The part of dne_cartpole_episodes / dne_discrete_episodes after their argument checks; errors are prefixed with `fn`.
static int discrete_episodes(const char* fn, dne_ctx* ctx, int env, const dne_net_desc* net, const float* d_theta,
                             const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx, int n_members,
                             const double* d_init_state, int max_steps, float* d_returns, int32_t* d_lengths,
                             double* d_final_state, void* stream) {
    const char* why = "";
    if (!dne_discrete_net_supported(env, net, &why)) {
        dne_set_error("%s: net not supported by the episode kernel: %s", fn, why);
        return DNE_ERR_UNSUP;
    }
    if (net->num_params > ctx->noise_count) {
        dne_set_error("%s: net larger than the noise table", fn);
        return DNE_ERR_ARG;
    }
    if (n_members == 0) return DNE_OK;
    const int rc = dne_launch_discrete_episodes(env, net, d_theta, ctx->noise, d_noise_idx, d_scale, d_theta_idx, n_members,
                                                d_init_state, max_steps, d_returns, d_lengths, d_final_state,
                                                (cudaStream_t)stream);
    if (rc) {
        dne_set_error("%s: launch setup failed (%d)", fn, rc);
        return rc;
    }
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) {
        dne_set_error("%s: kernel launch -> %s", fn, cudaGetErrorString(e));
        return DNE_ERR_CUDA;
    }
    return DNE_OK;
}

extern "C" int dne_cartpole_episodes(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                                     const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                     int n_members, const double* d_init_state, int max_steps, float* d_returns,
                                     int32_t* d_lengths, double* d_final_state, void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_init_state && d_returns && d_lengths, "null pointer");
    DNE_CHECK_ARG(n_members >= 0, "n_members < 0");
    DNE_CHECK_ARG(max_steps >= 1, "max_steps < 1");
    return discrete_episodes("dne_cartpole_episodes", ctx, DNE_EPISODE_CARTPOLE, net, d_theta, d_noise_idx, d_scale,
                             d_theta_idx, n_members, d_init_state, max_steps, d_returns, d_lengths, d_final_state, stream);
}

extern "C" int dne_discrete_episodes(dne_ctx* ctx, int env, const dne_net_desc* net, const float* d_theta,
                                     const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                     int n_members, const double* d_init_state, int max_steps, float* d_returns,
                                     int32_t* d_lengths, double* d_final_state, void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    const int limit = dne_discrete_time_limit(env);
    DNE_CHECK_ARG(limit > 0, "env is not a DNE_EPISODE_* task");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_init_state && d_returns && d_lengths, "null pointer");
    DNE_CHECK_ARG(n_members >= 0, "n_members < 0");
    DNE_CHECK_ARG(max_steps >= 1 && max_steps <= limit, "max_steps outside 1..the task's TimeLimit");
    return discrete_episodes("dne_discrete_episodes", ctx, env, net, d_theta, d_noise_idx, d_scale, d_theta_idx, n_members,
                             d_init_state, max_steps, d_returns, d_lengths, d_final_state, stream);
}

static int pendulum_net_check(const dne_net_desc* net, const char* fn) {
    const char* why = "";
    if (!dne_pendulum_net_supported(net, &why)) {
        dne_set_error("%s: net not supported by the episode kernel: %s", fn, why);
        return DNE_ERR_UNSUP;
    }
    return DNE_OK;
}

extern "C" int dne_pendulum_net_supported(const dne_net_desc* net) {
    DNE_CHECK_ARG(net, "null net");
    return pendulum_net_check(net, "dne_pendulum_net_supported");
}

extern "C" int dne_pendulum_episodes(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                                     const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                     int n_members, const double* d_init_state, int max_steps, const float* d_ob_mean,
                                     const float* d_ob_std, const float* d_ac_noise, float* d_returns,
                                     float* d_signreturns, int32_t* d_lengths, double* d_final_state, double* d_ob_sum,
                                     double* d_ob_sumsq, void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_init_state && d_returns && d_signreturns && d_lengths,
                  "null pointer");
    DNE_CHECK_ARG(n_members >= 0, "n_members < 0");
    DNE_CHECK_ARG(max_steps >= 1 && max_steps <= 200, "max_steps outside 1..200 (Pendulum-v1's TimeLimit)");
    DNE_CHECK_ARG((d_ob_mean == nullptr) == (d_ob_std == nullptr), "pass both d_ob_mean and d_ob_std or neither");
    DNE_CHECK_ARG((d_ob_sum == nullptr) == (d_ob_sumsq == nullptr), "pass both d_ob_sum and d_ob_sumsq or neither");
    const int rc0 = pendulum_net_check(net, "dne_pendulum_episodes");
    if (rc0) return rc0;
    DNE_CHECK_ARG(net->num_params <= ctx->noise_count, "net larger than the noise table");
    if (n_members == 0) return DNE_OK;
    const int rc = dne_launch_pendulum_episodes(net, d_theta, ctx->noise, d_noise_idx, d_scale, d_theta_idx, n_members,
                                                d_init_state, max_steps, d_ob_mean, d_ob_std, d_ac_noise, d_returns,
                                                d_signreturns, d_lengths, d_final_state, d_ob_sum, d_ob_sumsq,
                                                (cudaStream_t)stream);
    if (rc) {
        dne_set_error("dne_pendulum_episodes: launch setup failed (%d)", rc);
        return rc;
    }
    DNE_LAUNCH_CHECK();
    return DNE_OK;
}

static int maze_net_check(const dne_net_desc* net, const char* fn) {
    const char* why = "";
    if (!dne_maze_net_supported(net, &why)) {
        dne_set_error("%s: net not supported by the episode kernel: %s", fn, why);
        return DNE_ERR_UNSUP;
    }
    return DNE_OK;
}

extern "C" int dne_maze_net_supported(const dne_net_desc* net) {
    DNE_CHECK_ARG(net, "null net");
    return maze_net_check(net, "dne_maze_net_supported");
}

extern "C" int dne_maze_episodes(dne_ctx* ctx, const dne_maze_desc* maze, const dne_net_desc* net, const float* d_theta,
                                 const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                 int n_members, const double* d_init_state, int max_steps, const float* d_ob_mean,
                                 const float* d_ob_std, const float* d_ac_noise, float* d_returns, float* d_signreturns,
                                 int32_t* d_lengths, double* d_final_state, double* d_ob_sum, double* d_ob_sumsq,
                                 void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    DNE_CHECK_ARG(maze, "null maze");
    DNE_CHECK_ARG(maze->n_walls >= 0 && maze->n_walls <= DNE_MAZE_MAX_WALLS, "maze n_walls outside 0..64");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_init_state && d_returns && d_signreturns && d_lengths,
                  "null pointer");
    DNE_CHECK_ARG(n_members >= 0, "n_members < 0");
    DNE_CHECK_ARG(max_steps >= 1 && max_steps <= 400, "max_steps outside 1..400 (the maze's episode length)");
    DNE_CHECK_ARG((d_ob_mean == nullptr) == (d_ob_std == nullptr), "pass both d_ob_mean and d_ob_std or neither");
    DNE_CHECK_ARG((d_ob_sum == nullptr) == (d_ob_sumsq == nullptr), "pass both d_ob_sum and d_ob_sumsq or neither");
    const int rc0 = maze_net_check(net, "dne_maze_episodes");
    if (rc0) return rc0;
    DNE_CHECK_ARG(net->num_params <= ctx->noise_count, "net larger than the noise table");
    if (n_members == 0) return DNE_OK;
    const int rc = dne_launch_maze_episodes(maze, net, d_theta, ctx->noise, d_noise_idx, d_scale, d_theta_idx, n_members,
                                            d_init_state, max_steps, d_ob_mean, d_ob_std, d_ac_noise, d_returns,
                                            d_signreturns, d_lengths, d_final_state, d_ob_sum, d_ob_sumsq,
                                            (cudaStream_t)stream);
    if (rc) {
        dne_set_error("dne_maze_episodes: launch setup failed (%d)", rc);
        return rc;
    }
    DNE_LAUNCH_CHECK();
    return DNE_OK;
}

// ---- one member per thread-block cluster (nets too wide for one CTA) ----
static bool cluster_size_ok(int cluster) { return cluster == 0 || cluster == 2 || cluster == 4 || cluster == 8; }

// `rc` from a cluster launch or geometry query with its reason, prefixed with `fn`
static int cluster_fail(const char* fn, int rc, const char* why) {
    if (rc == DNE_ERR_UNSUP)
        dne_set_error("%s: net not supported by the cluster episode kernel: %s", fn, why);
    else
        dne_set_error("%s: launch setup failed (%d): %s", fn, rc, why);
    return rc;
}

static int pendulum_cluster_net_check(const dne_net_desc* net, const char* fn) {
    const char* why = "";
    if (!dne_pendulum_cluster_net_supported(net, &why)) return cluster_fail(fn, DNE_ERR_UNSUP, why);
    return DNE_OK;
}

static int maze_cluster_net_check(const dne_net_desc* net, const char* fn) {
    const char* why = "";
    if (!dne_maze_cluster_net_supported(net, &why)) return cluster_fail(fn, DNE_ERR_UNSUP, why);
    return DNE_OK;
}

extern "C" int dne_pendulum_cluster_net_supported(const dne_net_desc* net) {
    DNE_CHECK_ARG(net, "null net");
    return pendulum_cluster_net_check(net, "dne_pendulum_cluster_net_supported");
}

extern "C" int dne_maze_cluster_net_supported(const dne_net_desc* net) {
    DNE_CHECK_ARG(net, "null net");
    return maze_cluster_net_check(net, "dne_maze_cluster_net_supported");
}

extern "C" int dne_pendulum_cluster_geometry(const dne_net_desc* net, int cluster, int* geometry) {
    DNE_CHECK_ARG(net && geometry, "null pointer");
    DNE_CHECK_ARG(cluster_size_ok(cluster), "cluster must be 0 (automatic), 2, 4 or 8");
    int rc = pendulum_cluster_net_check(net, "dne_pendulum_cluster_geometry");
    if (rc) return rc;
    const char* why = "";
    rc = dne_pendulum_cluster_geometry(net, cluster, geometry, &why);
    return rc ? cluster_fail("dne_pendulum_cluster_geometry", rc, why) : DNE_OK;
}

extern "C" int dne_maze_cluster_geometry(const dne_net_desc* net, int cluster, int* geometry) {
    DNE_CHECK_ARG(net && geometry, "null pointer");
    DNE_CHECK_ARG(cluster_size_ok(cluster), "cluster must be 0 (automatic), 2, 4 or 8");
    int rc = maze_cluster_net_check(net, "dne_maze_cluster_geometry");
    if (rc) return rc;
    const char* why = "";
    rc = dne_maze_cluster_geometry(net, cluster, geometry, &why);
    return rc ? cluster_fail("dne_maze_cluster_geometry", rc, why) : DNE_OK;
}

extern "C" int dne_pendulum_cluster_episodes(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                                             const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                             int n_members, const double* d_init_state, int max_steps,
                                             const float* d_ob_mean, const float* d_ob_std, const float* d_ac_noise,
                                             float* d_returns, float* d_signreturns, int32_t* d_lengths,
                                             double* d_final_state, double* d_ob_sum, double* d_ob_sumsq, int cluster,
                                             void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_init_state && d_returns && d_signreturns && d_lengths,
                  "null pointer");
    DNE_CHECK_ARG(n_members >= 0, "n_members < 0");
    DNE_CHECK_ARG(max_steps >= 1 && max_steps <= 200, "max_steps outside 1..200 (Pendulum-v1's TimeLimit)");
    DNE_CHECK_ARG((d_ob_mean == nullptr) == (d_ob_std == nullptr), "pass both d_ob_mean and d_ob_std or neither");
    DNE_CHECK_ARG((d_ob_sum == nullptr) == (d_ob_sumsq == nullptr), "pass both d_ob_sum and d_ob_sumsq or neither");
    DNE_CHECK_ARG(cluster_size_ok(cluster), "cluster must be 0 (automatic), 2, 4 or 8");
    const int rc0 = pendulum_cluster_net_check(net, "dne_pendulum_cluster_episodes");
    if (rc0) return rc0;
    DNE_CHECK_ARG(net->num_params <= ctx->noise_count, "net larger than the noise table");
    if (n_members == 0) return DNE_OK;
    const char* why = "";
    const int rc = dne_launch_pendulum_cluster_episodes(net, d_theta, ctx->noise, d_noise_idx, d_scale, d_theta_idx,
                                                        n_members, d_init_state, max_steps, d_ob_mean, d_ob_std,
                                                        d_ac_noise, d_returns, d_signreturns, d_lengths, d_final_state,
                                                        d_ob_sum, d_ob_sumsq, cluster, &why, (cudaStream_t)stream);
    if (rc) return cluster_fail("dne_pendulum_cluster_episodes", rc, why);
    DNE_LAUNCH_CHECK();
    return DNE_OK;
}

extern "C" int dne_maze_cluster_episodes(dne_ctx* ctx, const dne_maze_desc* maze, const dne_net_desc* net,
                                         const float* d_theta, const int64_t* d_noise_idx, const float* d_scale,
                                         const int32_t* d_theta_idx, int n_members, const double* d_init_state,
                                         int max_steps, const float* d_ob_mean, const float* d_ob_std,
                                         const float* d_ac_noise, float* d_returns, float* d_signreturns,
                                         int32_t* d_lengths, double* d_final_state, double* d_ob_sum,
                                         double* d_ob_sumsq, int cluster, void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    DNE_CHECK_ARG(maze, "null maze");
    DNE_CHECK_ARG(maze->n_walls >= 0 && maze->n_walls <= DNE_MAZE_MAX_WALLS, "maze n_walls outside 0..64");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_init_state && d_returns && d_signreturns && d_lengths,
                  "null pointer");
    DNE_CHECK_ARG(n_members >= 0, "n_members < 0");
    DNE_CHECK_ARG(max_steps >= 1 && max_steps <= 400, "max_steps outside 1..400 (the maze's episode length)");
    DNE_CHECK_ARG((d_ob_mean == nullptr) == (d_ob_std == nullptr), "pass both d_ob_mean and d_ob_std or neither");
    DNE_CHECK_ARG((d_ob_sum == nullptr) == (d_ob_sumsq == nullptr), "pass both d_ob_sum and d_ob_sumsq or neither");
    DNE_CHECK_ARG(cluster_size_ok(cluster), "cluster must be 0 (automatic), 2, 4 or 8");
    const int rc0 = maze_cluster_net_check(net, "dne_maze_cluster_episodes");
    if (rc0) return rc0;
    DNE_CHECK_ARG(net->num_params <= ctx->noise_count, "net larger than the noise table");
    if (n_members == 0) return DNE_OK;
    const char* why = "";
    const int rc = dne_launch_maze_cluster_episodes(maze, net, d_theta, ctx->noise, d_noise_idx, d_scale, d_theta_idx,
                                                    n_members, d_init_state, max_steps, d_ob_mean, d_ob_std, d_ac_noise,
                                                    d_returns, d_signreturns, d_lengths, d_final_state, d_ob_sum,
                                                    d_ob_sumsq, cluster, &why, (cudaStream_t)stream);
    if (rc) return cluster_fail("dne_maze_cluster_episodes", rc, why);
    DNE_LAUNCH_CHECK();
    return DNE_OK;
}

// ---- discretised heads ----
static int pendulum_binned_net_check(const dne_net_desc* net, int n_bins, const char* fn) {
    const char* why = "";
    if (!dne_pendulum_binned_net_supported(net, n_bins, &why)) {
        dne_set_error("%s: net not supported by the binned episode kernels: %s", fn, why);
        return DNE_ERR_UNSUP;
    }
    return DNE_OK;
}

static int maze_binned_net_check(const dne_net_desc* net, int n_bins, const char* fn) {
    const char* why = "";
    if (!dne_maze_binned_net_supported(net, n_bins, &why)) {
        dne_set_error("%s: net not supported by the binned episode kernels: %s", fn, why);
        return DNE_ERR_UNSUP;
    }
    return DNE_OK;
}

extern "C" int dne_pendulum_binned_net_supported(const dne_net_desc* net, int n_bins) {
    DNE_CHECK_ARG(net, "null net");
    return pendulum_binned_net_check(net, n_bins, "dne_pendulum_binned_net_supported");
}

extern "C" int dne_maze_binned_net_supported(const dne_net_desc* net, int n_bins) {
    DNE_CHECK_ARG(net, "null net");
    return maze_binned_net_check(net, n_bins, "dne_maze_binned_net_supported");
}

extern "C" int dne_pendulum_binned_episodes(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                                            const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                            int n_members, const double* d_init_state, int max_steps,
                                            const float* d_ob_mean, const float* d_ob_std, const float* d_ac_noise,
                                            float* d_returns, float* d_signreturns, int32_t* d_lengths,
                                            double* d_final_state, double* d_ob_sum, double* d_ob_sumsq,
                                            const float* bin_values_host, int n_bins, int cluster, void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_init_state && d_returns && d_signreturns && d_lengths,
                  "null pointer");
    DNE_CHECK_ARG(bin_values_host, "null bin_values_host (the [1][n_bins] table of bin values)");
    DNE_CHECK_ARG(n_members >= 0, "n_members < 0");
    DNE_CHECK_ARG(max_steps >= 1 && max_steps <= 200, "max_steps outside 1..200 (Pendulum-v1's TimeLimit)");
    DNE_CHECK_ARG((d_ob_mean == nullptr) == (d_ob_std == nullptr), "pass both d_ob_mean and d_ob_std or neither");
    DNE_CHECK_ARG((d_ob_sum == nullptr) == (d_ob_sumsq == nullptr), "pass both d_ob_sum and d_ob_sumsq or neither");
    DNE_CHECK_ARG(cluster_size_ok(cluster), "cluster must be 0 (automatic), 2, 4 or 8");
    const int rc0 = pendulum_binned_net_check(net, n_bins, "dne_pendulum_binned_episodes");
    if (rc0) return rc0;
    DNE_CHECK_ARG(net->num_params <= ctx->noise_count, "net larger than the noise table");
    if (n_members == 0) return DNE_OK;
    const char* why = "";
    const int rc = dne_launch_pendulum_binned_episodes(net, d_theta, ctx->noise, d_noise_idx, d_scale, d_theta_idx,
                                                       n_members, d_init_state, max_steps, d_ob_mean, d_ob_std, d_ac_noise,
                                                       d_returns, d_signreturns, d_lengths, d_final_state, d_ob_sum,
                                                       d_ob_sumsq, bin_values_host, n_bins, cluster, &why,
                                                       (cudaStream_t)stream);
    if (rc) return cluster_fail("dne_pendulum_binned_episodes", rc, why);
    DNE_LAUNCH_CHECK();
    return DNE_OK;
}

extern "C" int dne_maze_binned_episodes(dne_ctx* ctx, const dne_maze_desc* maze, const dne_net_desc* net,
                                        const float* d_theta, const int64_t* d_noise_idx, const float* d_scale,
                                        const int32_t* d_theta_idx, int n_members, const double* d_init_state,
                                        int max_steps, const float* d_ob_mean, const float* d_ob_std,
                                        const float* d_ac_noise, float* d_returns, float* d_signreturns,
                                        int32_t* d_lengths, double* d_final_state, double* d_ob_sum, double* d_ob_sumsq,
                                        const float* bin_values_host, int n_bins, int cluster, void* stream) {
    DNE_CHECK_ARG(ctx && ctx->noise, "noise table not bound (dne_noise_bind)");
    DNE_CHECK_ARG(maze, "null maze");
    DNE_CHECK_ARG(maze->n_walls >= 0 && maze->n_walls <= DNE_MAZE_MAX_WALLS, "maze n_walls outside 0..64");
    DNE_CHECK_ARG(net && d_theta && d_noise_idx && d_scale && d_init_state && d_returns && d_signreturns && d_lengths,
                  "null pointer");
    DNE_CHECK_ARG(bin_values_host, "null bin_values_host (the [2][n_bins] table of bin values)");
    DNE_CHECK_ARG(n_members >= 0, "n_members < 0");
    DNE_CHECK_ARG(max_steps >= 1 && max_steps <= 400, "max_steps outside 1..400 (the maze's episode length)");
    DNE_CHECK_ARG((d_ob_mean == nullptr) == (d_ob_std == nullptr), "pass both d_ob_mean and d_ob_std or neither");
    DNE_CHECK_ARG((d_ob_sum == nullptr) == (d_ob_sumsq == nullptr), "pass both d_ob_sum and d_ob_sumsq or neither");
    DNE_CHECK_ARG(cluster_size_ok(cluster), "cluster must be 0 (automatic), 2, 4 or 8");
    const int rc0 = maze_binned_net_check(net, n_bins, "dne_maze_binned_episodes");
    if (rc0) return rc0;
    DNE_CHECK_ARG(net->num_params <= ctx->noise_count, "net larger than the noise table");
    if (n_members == 0) return DNE_OK;
    const char* why = "";
    const int rc = dne_launch_maze_binned_episodes(maze, net, d_theta, ctx->noise, d_noise_idx, d_scale, d_theta_idx,
                                                   n_members, d_init_state, max_steps, d_ob_mean, d_ob_std, d_ac_noise,
                                                   d_returns, d_signreturns, d_lengths, d_final_state, d_ob_sum,
                                                   d_ob_sumsq, bin_values_host, n_bins, cluster, &why,
                                                   (cudaStream_t)stream);
    if (rc) return cluster_fail("dne_maze_binned_episodes", rc, why);
    DNE_LAUNCH_CHECK();
    return DNE_OK;
}

extern "C" int dne_perturb_forward_mlp(dne_ctx* ctx, const dne_net_desc* net, const float* d_theta,
                                       const int64_t* d_noise_idx, const float* d_scale, const int32_t* d_theta_idx,
                                       const uint8_t* d_active, int n_slots, int paired, const float* d_obs,
                                       const float* d_ob_mean, const float* d_ob_std, float* d_actions_out,
                                       void* d_ws, size_t ws_bytes, void* stream) {
    DNE_CHECK_ARG(net && net->ob_kind == DNE_OB_VECTOR, "net must take float vector observations");
    DNE_CHECK_ARG(d_actions_out, "d_actions_out is null");
    DNE_CHECK_ARG((d_ob_mean == nullptr) == (d_ob_std == nullptr), "ob_mean / ob_std must both be given or both null");
    return forward_impl(ctx, net, d_theta, d_noise_idx, d_scale, d_theta_idx, d_active, n_slots, paired, d_obs,
                        d_ob_mean, d_ob_std, nullptr, nullptr, d_actions_out, d_ws, ws_bytes, stream);
}
