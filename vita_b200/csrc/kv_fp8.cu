// Paged FlashAttention over e4m3 pages: the pages a prompt-continuation plan references are gathered and dequantized
// into a bf16 scratch (kv_fp8.cuh's read definition), which flash_tc_kernel<..., PAGED = true> then reads through a
// remapped block table, unchanged.  So its output is bit for bit the bf16 kernel's on the dequantized pages.
#include "common.h"
#include "kv_fp8.cuh"

namespace vita {

constexpr int kStageThreads = 256;

// One CTA per work item (sequence, page index, scratch page): the page block_table[seq][p] of K and of V, every row
// dequantized; rows at or past the sequence's context are written as zeros (never attended, kept finite).
__global__ void __launch_bounds__(kStageThreads)
kv_fp8_stage_pages_kernel(const uint8_t* __restrict__ k8, const uint8_t* __restrict__ v8, const int* __restrict__ bt,
                          int bt_stride, const int* __restrict__ ctx, const int* __restrict__ work,
                          __nv_bfloat16* __restrict__ k16, __nv_bfloat16* __restrict__ v16, int row_elems,
                          int page_size, float k_scale, float v_scale) {
    const int seq = work[3 * blockIdx.x], pi = work[3 * blockIdx.x + 1], dst = work[3 * blockIdx.x + 2];
    const int src = bt[static_cast<long long>(seq) * bt_stride + pi];
    const int valid_rows = min(page_size, max(ctx[seq] - pi * page_size, 0));
    const int vecs_per_row = row_elems / 16;               // 16 elements: 16 bytes in, 32 bytes out
    const int n_vecs = page_size * vecs_per_row;
    const long long src0 = static_cast<long long>(src) * page_size * row_elems;
    const long long dst0 = static_cast<long long>(dst) * page_size * row_elems;
    for (int i = threadIdx.x; i < 2 * n_vecs; i += kStageThreads) {
        const bool is_v = i >= n_vecs;
        const int vi = is_v ? i - n_vecs : i;
        const long long e = static_cast<long long>(vi) * 16;
        uint4 o[2] = {make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0)};
        if (vi / vecs_per_row < valid_rows) {
            const uint4 w = __ldg(reinterpret_cast<const uint4*>((is_v ? v8 : k8) + src0 + e));
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
            const float sc = is_v ? v_scale : k_scale;
            uint32_t packed[8];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float f[4];
                kv_fp8_dequant4(ws[q], sc, f);
                packed[2 * q] = (__float_as_uint(f[0]) >> 16) | (__float_as_uint(f[1]) & 0xffff0000u);
                packed[2 * q + 1] = (__float_as_uint(f[2]) >> 16) | (__float_as_uint(f[3]) & 0xffff0000u);
            }
            o[0] = make_uint4(packed[0], packed[1], packed[2], packed[3]);
            o[1] = make_uint4(packed[4], packed[5], packed[6], packed[7]);
        }
        uint4* d = reinterpret_cast<uint4*>((is_v ? v16 : k16) + dst0 + e);
        d[0] = o[0];
        d[1] = o[1];
    }
}

}  // namespace vita

using namespace vita;

extern "C" int vita_kv_fp8_stage_pages(const void* k_cache, const void* v_cache, const int32_t* block_table,
                                       int64_t bt_stride, const int32_t* ctx_lens, const int32_t* work,
                                       int64_t n_work, void* k_out, void* v_out, int64_t n_kv_heads,
                                       int64_t head_dim, int64_t page_size, float k_scale, float v_scale,
                                       void* stream) {
    VITA_REQUIRE(head_dim == 128 && n_kv_heads > 0, "head_dim must be 128");
    VITA_REQUIRE(page_size > 0 && page_size <= 1024, "bad page_size");
    VITA_REQUIRE(kv_fp8_scales_ok(k_scale, v_scale), "k_scale / v_scale must be finite and positive");
    VITA_REQUIRE(n_work >= 0 && n_work <= 0x7fffffff && bt_stride > 0, "bad work count or block-table stride");
    if (n_work == 0) return VITA_OK;
    VITA_REQUIRE(k_cache && v_cache && block_table && ctx_lens && work && k_out && v_out, "null pointer");
    VITA_REQUIRE(aligned16(k_cache) && aligned16(v_cache) && aligned16(k_out) && aligned16(v_out),
                 "caches and scratch must be 16-byte aligned");
    kv_fp8_stage_pages_kernel<<<static_cast<unsigned>(n_work), kStageThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const uint8_t*>(k_cache), static_cast<const uint8_t*>(v_cache), block_table, (int)bt_stride,
        ctx_lens, work, static_cast<__nv_bfloat16*>(k_out), static_cast<__nv_bfloat16*>(v_out),
        (int)(n_kv_heads * head_dim), (int)page_size, k_scale, v_scale);
    return check_launch("kv_fp8_stage_pages");
}
