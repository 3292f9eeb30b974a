// ptx.cuh -- minimal mbarrier / bulk-copy / operand-split PTX helpers for sm_90a (hand-written; no CUTLASS dependency).
//
// Operand layout used throughout (wgmma "K-major, no swizzle" canonical layout, 32-bit elements shown):
// a tile of R rows x KC k-elements is stored as float4 T[KC/4][R]:  element (r, k) lives at byte
//     (k/4) * (R*16)  +  r*16  +  (k%4)*4
// i.e. core matrices of 8 rows x 16 bytes are contiguous (128 B), the next 8-row group follows at SBO = 128 B and the
// next 4 k-elements at LBO = R*16 B.  One wgmma kind tf32 consumes K = 8 elements = two such k-quads; with fp16 elements a
// 16-byte row holds 8 k values and one kind f16 wgmma consumes K = 16 = two k-octets.
// Consecutive rows are consecutive 16-byte chunks, so staging threads that own consecutive rows write conflict-free.
//
// Accumulators live in the registers of the issuing warpgroup (128 threads, warps 4i..4i+3).  For an m64nN tile, thread
// t = 32*w + l of the warpgroup holds N/2 floats: d[4*j + 2*h + e] is row 16*w + l/4 + 8*h, column 8*j + 2*(l%4) + e.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ----------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t a = smem_u32(bar);
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
        "@P1 bra DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "DONE:\n\t"
        "}\n" ::"r"(a), "r"(parity)
        : "memory");
}

// ---- fences ------------------------------------------------------------------------------------------
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads, bulk copies)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- descriptors -------------------------------------------------------------------------------------
// shared-memory matrix descriptor (sm_90), K-major, no swizzle (layout type 0), base offset 0
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}

// Explicit shared-window accesses with 32-bit addresses.  Stores through a C++ pointer derived from the (re-aligned)
// dynamic shared-memory base compile to GENERIC ST.E / LD.E (the cast hides the address space from ptxas).
__device__ __forceinline__ void sts128(uint32_t saddr, const float4& v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t saddr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr));
    return v;
}
__device__ __forceinline__ float lds32(uint32_t saddr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr));
    return v;
}

// ---- 3xTF32 operand split ---------------------------------------------------------------------------
// hi = rna_tf32(x), lo = rna_tf32(x - hi): both have their low 13 mantissa bits clear, so the tensor core's fp32->tf32
// input truncation is exact.  a*b ~= hi_a*hi_b + lo_a*hi_b + hi_a*lo_b  (dropped lo*lo term ~2^-24 relative).
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    uint32_t h;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
    hi = __uint_as_float(h);
    uint32_t l;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(x - hi));
    lo = __uint_as_float(l);
}

// Cheap variant used by the staging loops (4 integer/float ops instead of two cvt.rna sequences):
// hi = x rounded to TF32 by adding half an ulp to the magnitude bits and masking, lo = (x - hi) truncated to TF32.
// |lo| <= 2^-11 |x| and its truncation loses <= 2^-11 of it, so the dropped part is <= 2^-22 |x| per operand.
__device__ __forceinline__ void split_tf32_fast(float x, float& hi, float& lo) {
    const uint32_t hb = (__float_as_uint(x) + 0x1000u) & 0xFFFFE000u;
    hi = __uint_as_float(hb);
    lo = __uint_as_float(__float_as_uint(x - hi) & 0xFFFFE000u);
}

// ---- 2 x fp16 operand split (f16 wgmma runs at twice the MAC rate of tf32) ----------------------------------------
// x = h0 + h1 * 2^-11 with h0 = rn_fp16(x), h1 = rn_fp16((x - h0) * 2^11): 22 significand bits, |error| <= 2^-24 |x| (fp16
// subnormals are exact to 2^-25 absolute and h1 picks up the rest).  The lo part is carried SCALED by 2^11 so that it never
// falls into fp16's subnormal range before x itself does; products with it go to a separate accumulator that the epilogue
// folds back with 2^-11:  a*b ~= h0a*h0b + 2^-11 * (h0a*h1b + h1a*h0b)   (dropped h1a*h1b term: 2^-24 relative).
// fp16 products are exact in the fp32 accumulator.  Range: |x| <= 65504 (fp16 max); larger magnitudes saturate.
constexpr float F16_LO_SCALE = 2048.0f, F16_LO_INV = 1.0f / 2048.0f;
__device__ __forceinline__ void split_f16(float x, __half& h0, __half& h1) {
    h0 = __float2half_rn(fminf(fmaxf(x, -65504.0f), 65504.0f));
    h1 = __float2half_rn((x - __half2float(h0)) * F16_LO_SCALE);
}
// two values at a time with the packed conversions (cvt.rn.satfinite.f16x2.f32: saturating, one instruction per pair)
__device__ __forceinline__ void split_f16x2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(x1), "f"(x0));      // d = {hi half: a, lo half: b}
    const __half2 h = *reinterpret_cast<const __half2*>(&hi);
    const float2 hf = __half22float2(h);
    const float r0 = (x0 - hf.x) * F16_LO_SCALE, r1 = (x1 - hf.y) * F16_LO_SCALE;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(r1), "f"(r0));
}
// eight values -> one 16-byte row of the hi plane and one of the (scaled) lo plane
__device__ __forceinline__ void split_f16x8(const float (&x)[8], uint4& hi, uint4& lo) {
    split_f16x2(x[0], x[1], hi.x, lo.x);
    split_f16x2(x[2], x[3], hi.y, lo.y);
    split_f16x2(x[4], x[5], hi.z, lo.z);
    split_f16x2(x[6], x[7], hi.w, lo.w);
}
__device__ __forceinline__ void sts128u(uint32_t saddr, const uint4& v) {
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

}  // namespace wg

// ---- 1-D bulk async copy (TMA engine, no tensor map): global -> shared, completion on an mbarrier ---------------
namespace wg {
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// src and dst 16-byte aligned, bytes a multiple of 16
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// L2-only prefetch of a contiguous global range (16-byte aligned, size % 16 == 0): no shared-memory destination
__device__ __forceinline__ void bulk_prefetch_l2(const void* gptr, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(gptr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
}  // namespace wg
