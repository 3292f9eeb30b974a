// wgmma.cuh -- Hopper warpgroup-MMA (wgmma) wrappers for sm_90a; the operand layout is described in ptx.cuh.
#pragma once
#include "ptx.cuh"

namespace wg {

// ---- warpgroup MMA -----------------------------------------------------------------------------------
// D[m64 x N] (+)= A[smem, 64 x K] * B[smem, N x K]^T, issued by all 128 threads of a warpgroup (warp-uniform operands).
// d points at the N/2 accumulator registers of this thread; scale_d = 0 overwrites D, 1 accumulates.
// wgmma_f16: K = 16 fp16 (two k-octets), wgmma_tf32: K = 8 tf32 (two k-quads; the hardware truncates fp32 to tf32).
template <int N> __device__ __forceinline__ void wgmma_f16(float* d, uint64_t da, uint64_t db, uint32_t scale_d);
#define WG_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
template <int N> __device__ __forceinline__ void wgmma_tf32(float* d, uint64_t da, uint64_t db, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_f16<16>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %8, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %9, %10, p, 1, 1, 0, 0;\n\t}\n"
        : WG_ACC8(0)
        : "r"(scale_d), "l"(da), "l"(db)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_f16<32>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %16, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %17, %18, p, 1, 1, 0, 0;\n\t}\n"
        : WG_ACC8(0), WG_ACC8(8)
        : "r"(scale_d), "l"(da), "l"(db)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_f16<64>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %32, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %33, %34, p, 1, 1, 0, 0;\n\t}\n"
        : WG_ACC8(0), WG_ACC8(8), WG_ACC8(16), WG_ACC8(24)
        : "r"(scale_d), "l"(da), "l"(db)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_f16<128>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %64, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %65, %66, p, 1, 1, 0, 0;\n\t}\n"
        : WG_ACC8(0), WG_ACC8(8), WG_ACC8(16), WG_ACC8(24), WG_ACC8(32), WG_ACC8(40), WG_ACC8(48), WG_ACC8(56)
        : "r"(scale_d), "l"(da), "l"(db)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<16>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %8, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %9, %10, p, 1, 1;\n\t}\n"
        : WG_ACC8(0)
        : "r"(scale_d), "l"(da), "l"(db)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<32>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %16, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %17, %18, p, 1, 1;\n\t}\n"
        : WG_ACC8(0), WG_ACC8(8)
        : "r"(scale_d), "l"(da), "l"(db)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<64>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %32, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %33, %34, p, 1, 1;\n\t}\n"
        : WG_ACC8(0), WG_ACC8(8), WG_ACC8(16), WG_ACC8(24)
        : "r"(scale_d), "l"(da), "l"(db)
        : "memory");
}
template <> __device__ __forceinline__ void wgmma_tf32<128>(float* d, uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %64, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %65, %66, p, 1, 1;\n\t}\n"
        : WG_ACC8(0), WG_ACC8(8), WG_ACC8(16), WG_ACC8(24), WG_ACC8(32), WG_ACC8(40), WG_ACC8(48), WG_ACC8(56)
        : "r"(scale_d), "l"(da), "l"(db)
        : "memory");
}
// orders register accesses of the accumulators against the asynchronous MMAs (before the first wgmma of a batch)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// returns when at most N committed groups of this warp are still in flight
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the compiler must not move reads / writes of the accumulators across wgmma_wait / wgmma_fence
template <int N> __device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// register budget of a warpgroup-specialised kernel: producer warpgroups give registers back, MMA warpgroups take them
template <int R> __device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R> __device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }

}  // namespace wg
