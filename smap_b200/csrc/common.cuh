// Shared device helpers for the smap_b200 kernels (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#ifndef __CUDA_ARCH_FEAT_SM90_ALL
#if defined(__CUDA_ARCH__)
#error "smap_b200 kernels must be compiled with -gencode arch=compute_90a,code=sm_90a"
#endif
#endif

namespace smapb {

// ---------------------------------------------------------------------------------------------
// shared-memory addressing + mbarrier + bulk-async (TMA) primitives, raw PTX.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
// make mbarrier.init visible to the async proxy (TMA)
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok;
}
// Out of line: a trap inlined after setmaxnreg.inc makes ptxas hold that role to the launch-time register budget
// (spills in the 232-register consumers of conv_tc_kernel); behind a call it does not.
static __device__ __noinline__ void mbar_timeout() { __trap(); }
// Bounded wait: a protocol bug traps (kernel error) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > 4000000000LL) {  // ~2 s at 2 GHz
            mbar_timeout();
        }
    }
}

// 1-D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP).
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// Programmatic dependent launch hooks (no-ops when the launch has no PDL attribute).
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// split-bf16 helpers: v ~= hi + lo with |v - hi - lo| <= 2^-17 |v|
__device__ __forceinline__ void split_bf16(float v, __nv_bfloat16& hi, __nv_bfloat16& lo) {
    hi = __float2bfloat16_rn(v);
    lo = __float2bfloat16_rn(v - __bfloat162float(hi));
}
__device__ __forceinline__ uint32_t pack_bf16x2(__nv_bfloat16 a, __nv_bfloat16 b) {
    return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}
__device__ __forceinline__ float bf16lo_to_f(uint32_t packed) { return __uint_as_float(packed << 16); }
__device__ __forceinline__ float bf16hi_to_f(uint32_t packed) { return __uint_as_float(packed & 0xffff0000u); }

// ---------------------------------------------------------------------------------------------
// Activation / weight element format.  Every 2-byte format the kernels store is described here: the wgmma operand type,
// the TMA data type, pack (fp32 -> 2 elements, round to nearest even) and unpack (exact widening).
//   ElemBF16 : bf16, fp32's exponent range (the bf16x3 and bf16 precisions)
//   ElemF16  : fp16, 10-bit mantissa, finite range +-65504: stores clamp to it and count the clamped elements
// ---------------------------------------------------------------------------------------------
struct ElemBF16 {
    static constexpr bool F16 = false;
    static constexpr CUtensorMapDataType TMA_DTYPE = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    // low half = a, high half = b
    static __device__ __forceinline__ uint32_t pack2(float a, float b) {
        uint32_t w;
        asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(w) : "f"(b), "f"(a));
        return w;
    }
    static __device__ __forceinline__ float lo(uint32_t w) { return bf16lo_to_f(w); }
    static __device__ __forceinline__ float hi(uint32_t w) { return bf16hi_to_f(w); }
};
struct ElemF16 {
    static constexpr bool F16 = true;
    static constexpr CUtensorMapDataType TMA_DTYPE = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    static constexpr float MAX = 65504.f;
    static __device__ __forceinline__ uint32_t pack2(float a, float b) {
        uint32_t w;
        asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(w) : "f"(b), "f"(a));
        return w;
    }
    static __device__ __forceinline__ float lo(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w & 0xffffu))); }
    static __device__ __forceinline__ float hi(uint32_t w) { return __half2float(__ushort_as_half((unsigned short)(w >> 16))); }
    // max(m, |v|), NaN if either is NaN
    static __device__ __forceinline__ float absmax(float m, float v) {
        float r;
        asm("{\n\t.reg .f32 t;\n\tabs.f32 t, %2;\n\tmax.NaN.f32 %0, %1, t;\n\t}" : "=f"(r) : "f"(m), "f"(v));
        return r;
    }
    // v limited to the finite fp16 range (NaN -> -MAX); n counts the values that were outside it
    static __device__ __forceinline__ float clamp(float v, int& n) {
        n += !(fabsf(v) <= MAX);
        return fminf(fmaxf(v, -MAX), MAX);
    }
};
// Adds a warp's clamp count to the saturation counter: one atomic per warp, and none when nothing was clamped.  Every lane
// of the warp must call it.
__device__ __forceinline__ void saturation_add(unsigned long long* counter, int n) {
    const unsigned total = __reduce_add_sync(0xffffffffu, (unsigned)n);
    if (total != 0 && (threadIdx.x & 31) == 0 && counter) atomicAdd(counter, (unsigned long long)total);
}

}  // namespace smapb
