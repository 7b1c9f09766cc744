// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor); the wgmma wrappers are in wgmma.cuh.
// Everything here is device-only and header-only.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace vita {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (kernel aborts with an error) instead of hanging the GPU.
// The timeout message is a debug-build aid (-DVITA_MBAR_PRINT=1): a printf call anywhere in a kernel makes ptxas
// serialise its wgmma.mma_async instructions.
#ifndef VITA_MBAR_PRINT
#define VITA_MBAR_PRINT 0
#endif
#ifndef VITA_MBAR_TIMEOUT_CYCLES
#define VITA_MBAR_TIMEOUT_CYCLES (4000000000ll)  // ~2 s at the H100 boost clock
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, int tag = 0) {
    if (mbar_try_wait(bar, parity)) return;
    long long t0 = clock64();
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0x3ff) == 0 && clock64() - t0 > VITA_MBAR_TIMEOUT_CYCLES) {
            if (VITA_MBAR_PRINT) printf("[vita] mbarrier timeout: block %d thread %d tag %d parity %u\n", blockIdx.x, threadIdx.x, tag,
                   parity);
            __trap();
        }
    }
}
// ---------------------------------------------------------------- TMA
// L2-only prefetch of one 2-D tile (no shared-memory destination, no barrier)
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* m, int c0, int c1) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(reinterpret_cast<uint64_t>(m)),
                 "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
        "[%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
        "[%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// ---------------------------------------------------------------- programmatic dependent launch
// No-ops unless the kernel was launched with cudaLaunchAttributeProgrammaticStreamSerialization.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- decode-chain completion counters (see common.h)
struct ChainArgsDev {
    const unsigned long long* serial;
    const unsigned long long* wait_cnt;
    unsigned long long* done_cnt;
    int wait_arrivals;
};
// one thread: returns once the predecessor's stores are visible (acquire); other threads follow through a CTA barrier
__device__ __forceinline__ void chain_wait(const ChainArgsDev& c) {
    if (c.wait_cnt != nullptr) {
        const unsigned long long target = *reinterpret_cast<const volatile unsigned long long*>(c.serial) *
                                          static_cast<unsigned long long>(c.wait_arrivals);
        for (int i = 0; i < 4096; ++i) {
            unsigned long long v;
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(c.wait_cnt) : "memory");
            if (v >= target) return;
        }
    }
    pdl_wait();   // chain start, protocol off, or a counter that never arrived: the hardware dependency always holds
}
// one thread, after a CTA-level barrier that orders the CTA's last global stores before it
__device__ __forceinline__ void chain_arrive(const ChainArgsDev& c) {
    if (c.done_cnt != nullptr) {
        __threadfence();
        asm volatile("red.release.gpu.global.add.u64 [%0], 1;" ::"l"(c.done_cnt) : "memory");
    }
}

// ---------------------------------------------------------------- misc
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
    __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint4 ldg_nc_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
// 2^x on the FMA / ALU pipes (no MUFU): round-to-nearest split x = n + f with the 1.5 * 2^23 trick, cubic minimax of
// 2^f on [-0.5, 0.5] (relative error 7.5e-5, far below the bf16 rounding of the result), exponent insertion by integer
// add.  x is clamped at -126 (anything smaller is 0 after the bf16 conversion anyway).
__device__ __forceinline__ float ex2_poly(float x) {
    x = fmaxf(x, -126.0f);
    const float xr = x + 12582912.0f;
    const float f = x - (xr - 12582912.0f);
    float p = fmaf(0.05517162f, f, 0.24261113f);
    p = fmaf(p, f, 0.69326097f);
    p = fmaf(p, f, 0.99992806f);
    return __int_as_float(__float_as_int(p) + (__float_as_int(xr) << 23));
}
// rotate-half RoPE of one (x[j], x[j + D/2]) pair (transformers apply_rotary_pos_emb, modeling_mixtral.py:232-254).  One
// definition for the stand-alone pass and the qkv GEMM epilogue, so both round identically.
__device__ __forceinline__ void rope_rotate(float x1, float x2, float c, float s, float& o1, float& o2) {
    o1 = x1 * c - x2 * s;
    o2 = x2 * c + x1 * s;
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float silu(float x) { return x / (1.0f + __expf(-x)); }

#ifdef VITA_TRACE
__device__ __forceinline__ unsigned long long global_timer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
#define VITA_STAMP(i) do { if (trace) trace[i] = global_timer_ns(); } while (0)
#define VITA_STAMP_SET(i, v) do { if (trace) trace[i] = (v); } while (0)
#else
#define VITA_STAMP(i) do { } while (0)
#define VITA_STAMP_SET(i, v) do { } while (0)
#endif

}  // namespace vita
