// common.cuh -- shared helpers for libdne.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <string.h>

#include "../../include/dne.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libdne is written for sm_90a (H100) only"
#endif

#define DNE_MAX_PREP 16
struct dne_ctx {
    int device;
    int sm_count;
    const float* noise;     // borrowed
    int64_t noise_count;
    double* scratch;        // owned: DNE_SCRATCH_DOUBLES doubles
    // optional CUDA-event timing of the dominant kernel (dense_noise_gemv) on the launching stream
    cudaEvent_t* ev;        // 2 * ev_cap events
    int ev_cap, ev_n, prof_on;
    // optional phase events of the NEXT forward call (two half-tables on two streams, phase-shifted by half a tick)
    void* ev_wait;          // the forward's stream waits for this event before its first kernel
    void* ev_record;        // recorded right before the first HBM-bound noise GEMV of the call
    int ev_record_done;
    int ev_mode;            // 0: wait before the first kernel, record before the GEMV; 1: wait before / record after the GEMV
    // workspaces whose prepared-theta region (dne_theta_prepare) is current: (workspace, theta it was made from)
    struct { const void* ws; const float* theta; int n_slots; } prep[DNE_MAX_PREP];
};
void dne_prep_invalidate_theta(dne_ctx* ctx, const float* d_theta);   // a kernel of this library is about to rewrite theta
extern unsigned long long g_dne_launches;   // kernels launched by this library (process-wide)
#define DNE_LAUNCHED(n) (g_dne_launches += (unsigned long long)(n))
#define DNE_SCRATCH_DOUBLES 16384

void dne_set_error(const char* fmt, ...);

#define DNE_CHECK_ARG(cond, msg)                                   \
    do {                                                           \
        if (!(cond)) {                                             \
            dne_set_error("%s: %s", __func__, msg);                \
            return DNE_ERR_ARG;                                    \
        }                                                          \
    } while (0)

#define DNE_CUDA(call)                                                                 \
    do {                                                                               \
        cudaError_t e__ = (call);                                                      \
        if (e__ != cudaSuccess) {                                                      \
            dne_set_error("%s: %s -> %s", __func__, #call, cudaGetErrorString(e__));   \
            return DNE_ERR_CUDA;                                                       \
        }                                                                              \
    } while (0)

#define DNE_LAUNCH_CHECK1() do { DNE_LAUNCHED(1); DNE_LAUNCH_CHECK(); } while (0)
#define DNE_LAUNCH_CHECK()                                                             \
    do {                                                                               \
        cudaError_t e__ = cudaGetLastError();                                          \
        if (e__ != cudaSuccess) {                                                      \
            dne_set_error("%s: kernel launch -> %s", __func__, cudaGetErrorString(e__)); \
            return DNE_ERR_CUDA;                                                       \
        }                                                                              \
    } while (0)

// ---- programmatic dependent launch (PDL) of the tick's kernel chain -----------------------------------------------
// conv1 -> conv2 -> conv3 -> theta GEMM -> noise GEMV -> combine+head run back to back on one stream.  Kernels 2..6 are
// launched with cudaLaunchAttributeProgrammaticStreamSerialization: every kernel of the chain calls pdl_trigger() first
// thing (the NEXT launch may be scheduled as soon as all CTAs of this grid have started), sets itself up (barriers,
// weight prefetch: nothing that an upstream kernel of the tick writes) and calls pdl_wait() before the first access to
// upstream data or to any global buffer it writes.  pdl_wait() returns when the previous grid has completed and flushed --
// which itself waited for ITS predecessor, so completion is transitive along the chain.  The launch latency and the
// prologue of kernel i+1 overlap the tail of kernel i.  dne_set_option("pdl", 0) launches the chain fully serialized.
extern int g_dne_pdl;
extern int g_dne_chain_ticks;
template <typename... KArgs, typename... Args>
static inline cudaError_t dne_launch_chain(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool dependent,
                                           Args... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = (dependent && g_dne_pdl) ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, args...);
}
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

static inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- device helpers --------------------------------------------------------------------------------
__device__ __forceinline__ float4 ldg_stream_f4(const float* p) {
    // streaming 128-bit load: read-only path, do not allocate in L1 (data is touched once)
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
// Eight independent streaming 128-bit loads issued back to back from ONE asm statement, so the compiler cannot
// interleave them with their consumers: 8 x 16 B per thread are guaranteed to be in flight together (memory-level
// parallelism is what an HBM-bound kernel lives on; ptxas otherwise serialises to ~3 loads in flight).
__device__ __forceinline__ void ldg_stream_f4x8(const float* p, int64_t stride, float4 (&v)[8]) {
    const float* p0 = p;
    const float* p1 = p + stride;
    const float* p2 = p + 2 * stride;
    const float* p3 = p + 3 * stride;
    const float* p4 = p + 4 * stride;
    const float* p5 = p + 5 * stride;
    const float* p6 = p + 6 * stride;
    const float* p7 = p + 7 * stride;
    asm volatile(
        "ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%32];\n\t"
        "ld.global.nc.L1::no_allocate.v4.f32 {%4,%5,%6,%7}, [%33];\n\t"
        "ld.global.nc.L1::no_allocate.v4.f32 {%8,%9,%10,%11}, [%34];\n\t"
        "ld.global.nc.L1::no_allocate.v4.f32 {%12,%13,%14,%15}, [%35];\n\t"
        "ld.global.nc.L1::no_allocate.v4.f32 {%16,%17,%18,%19}, [%36];\n\t"
        "ld.global.nc.L1::no_allocate.v4.f32 {%20,%21,%22,%23}, [%37];\n\t"
        "ld.global.nc.L1::no_allocate.v4.f32 {%24,%25,%26,%27}, [%38];\n\t"
        "ld.global.nc.L1::no_allocate.v4.f32 {%28,%29,%30,%31}, [%39];"
        : "=f"(v[0].x), "=f"(v[0].y), "=f"(v[0].z), "=f"(v[0].w), "=f"(v[1].x), "=f"(v[1].y), "=f"(v[1].z), "=f"(v[1].w),
          "=f"(v[2].x), "=f"(v[2].y), "=f"(v[2].z), "=f"(v[2].w), "=f"(v[3].x), "=f"(v[3].y), "=f"(v[3].z), "=f"(v[3].w),
          "=f"(v[4].x), "=f"(v[4].y), "=f"(v[4].z), "=f"(v[4].w), "=f"(v[5].x), "=f"(v[5].y), "=f"(v[5].z), "=f"(v[5].w),
          "=f"(v[6].x), "=f"(v[6].y), "=f"(v[6].z), "=f"(v[6].w), "=f"(v[7].x), "=f"(v[7].y), "=f"(v[7].z), "=f"(v[7].w)
        : "l"(p0), "l"(p1), "l"(p2), "l"(p3), "l"(p4), "l"(p5), "l"(p6), "l"(p7));
}
__device__ __forceinline__ float ldg_stream_f1(const float* p) {
    float r;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
    return r;
}

__device__ __forceinline__ float apply_act(float x, int act) {
    if (act == DNE_ACT_RELU) return fmaxf(x, 0.0f);
    if (act == DNE_ACT_TANH) return tanhf(x);
    return x;
}

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
