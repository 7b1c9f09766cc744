// Copy-on-write for the paged KV cache: whole pages copied from src to dst in the K and the V cache of every layer
// (vLLM's cache_ops.copy_blocks role).  Beam search forks a sequence's cache and gives each child beam a private copy
// of the page its next row lands in; one launch per step covers every (src, dst) pair and every layer.
//
// layer_base[n_bases]: device pointers of the per-layer caches (K of layer 0 .. L-1, then V, or any order); every
// cache holds n_pages pages of page_bytes bytes.  pairs[n_pairs][2] (device, i32): (src page, dst page).  A pair with
// an index outside [0, n_pages) is skipped.  16-byte vector copies, bit-exact; the kernel only streams HBM.
// Precondition: the pairs are copied concurrently, so no dst page is also a src page of the launch and no two pairs
// share a dst page (PagePool takes every dst fresh from its free list and copies only pages still referenced).
#include "common.h"

namespace vita {

constexpr int kCopyThreads = 256;
constexpr int kCopyUnroll = 4;          // 16-byte vectors in flight per thread

__global__ void __launch_bounds__(kCopyThreads)
kv_copy_pages_kernel(const unsigned long long* __restrict__ layer_base, const int* __restrict__ pairs, int n_pages,
                     long long page_vecs) {
    const int src = pairs[2 * blockIdx.y], dst = pairs[2 * blockIdx.y + 1];
    if (src < 0 || dst < 0 || src >= n_pages || dst >= n_pages || src == dst) return;
    const uint4* s = reinterpret_cast<const uint4*>(layer_base[blockIdx.z]) + static_cast<long long>(src) * page_vecs;
    uint4* d = reinterpret_cast<uint4*>(layer_base[blockIdx.z]) + static_cast<long long>(dst) * page_vecs;
    const long long stride = static_cast<long long>(gridDim.x) * kCopyThreads * kCopyUnroll;
    for (long long i0 = static_cast<long long>(blockIdx.x) * kCopyThreads * kCopyUnroll + threadIdx.x; i0 < page_vecs;
         i0 += stride) {
        uint4 v[kCopyUnroll];
#pragma unroll
        for (int u = 0; u < kCopyUnroll; ++u) {
            const long long i = i0 + u * kCopyThreads;
            if (i < page_vecs) v[u] = __ldg(s + i);
        }
#pragma unroll
        for (int u = 0; u < kCopyUnroll; ++u) {
            const long long i = i0 + u * kCopyThreads;
            if (i < page_vecs) d[i] = v[u];
        }
    }
}

}  // namespace vita

using namespace vita;

extern "C" int vita_kv_copy_pages(const uint64_t* layer_base, int64_t n_bases, const int32_t* pairs, int64_t n_pairs,
                                  int64_t n_pages, int64_t page_bytes, void* stream) {
    VITA_REQUIRE(page_bytes > 0 && page_bytes % 16 == 0, "page_bytes must be a positive multiple of 16");
    VITA_REQUIRE(n_bases >= 0 && n_bases <= 65535, "n_bases must be in [0, 65535]");
    VITA_REQUIRE(n_pairs >= 0 && n_pairs <= 65535, "n_pairs must be in [0, 65535]");
    VITA_REQUIRE(n_pages > 0 && n_pages <= 0x7fffffff, "n_pages must be positive");
    if (n_bases == 0 || n_pairs == 0) return VITA_OK;
    VITA_REQUIRE(layer_base && pairs, "layer_base and pairs are required");
    const long long page_vecs = page_bytes / 16;
    const long long per_cta = static_cast<long long>(kCopyThreads) * kCopyUnroll;
    const unsigned gx = static_cast<unsigned>((page_vecs + per_cta - 1) / per_cta);
    kv_copy_pages_kernel<<<dim3(gx, static_cast<unsigned>(n_pairs), static_cast<unsigned>(n_bases)), kCopyThreads, 0,
                           static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const unsigned long long*>(layer_base),
                                                                pairs, (int)n_pages, page_vecs);
    return check_launch("kv_copy_pages");
}
