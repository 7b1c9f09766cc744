// Page digests of the prompt rows for prefix caching in the continuous batcher: one 128-bit digest per full KV page
// of the spliced bf16 prompt rows (text, image and audio rows alike), so two requests share a page only when the model
// saw the same rows there.  The host chains the digests into per-page keys (vita_b200/model/mixtral.py, prefix_keys).
//
// The function (include/vita_b200.h, vita_page_digest), reproduced bit for bit by the numpy reference of the tests:
// the rows of page p, each row's first H bf16 values read as H / 4 little-endian u64 words, are concatenated row by
// row into the words w_0 .. w_{n-1} (n = page_size * H / 4), and lane l in {0, 1} is
//     d_l = sum_j mix64(w_j + j * kGamma + kSeed[l])   (mod 2^64)
// with mix64 = splitmix64's finalizer.  A sum is order free, so the CTA's reduction order does not matter.
#include "common.h"

namespace vita {

constexpr int kDigestThreads = 256;
constexpr unsigned long long kGamma = 0x9E3779B97F4A7C15ull;
constexpr unsigned long long kSeed0 = 0x243F6A8885A308D3ull;
constexpr unsigned long long kSeed1 = 0x13198A2E03707344ull;

__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// One CTA per page; 16-byte loads (two words) of the page's rows, row stride `ld` bf16 values.
__global__ void __launch_bounds__(kDigestThreads)
page_digest_kernel(const __nv_bfloat16* __restrict__ rows, long long ld, int H, int page_size,
                   unsigned long long* __restrict__ out) {
    const int vec_per_row = H / 8;                       // uint4 = 8 bf16 = 2 words
    const int n_vec = page_size * vec_per_row;
    const long long row0 = static_cast<long long>(blockIdx.x) * page_size;
    unsigned long long a0 = 0, a1 = 0;
    for (int i = threadIdx.x; i < n_vec; i += kDigestThreads) {
        const int r = i / vec_per_row, c = i - r * vec_per_row;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(rows + (row0 + r) * ld) + c);
        const unsigned long long j = 2ull * static_cast<unsigned long long>(i);    // word index within the page
        const unsigned long long w0 = (static_cast<unsigned long long>(v.y) << 32) | v.x;
        const unsigned long long w1 = (static_cast<unsigned long long>(v.w) << 32) | v.z;
        a0 += mix64(w0 + j * kGamma + kSeed0) + mix64(w1 + (j + 1) * kGamma + kSeed0);
        a1 += mix64(w0 + j * kGamma + kSeed1) + mix64(w1 + (j + 1) * kGamma + kSeed1);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a0 += __shfl_xor_sync(0xffffffffu, a0, o);
        a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    __shared__ unsigned long long part[2][kDigestThreads / 32];
    const int warp = threadIdx.x / 32, lane = threadIdx.x % 32;
    if (lane == 0) {
        part[0][warp] = a0;
        part[1][warp] = a1;
    }
    __syncthreads();
    if (threadIdx.x < 2) {
        unsigned long long s = 0;
        for (int w = 0; w < kDigestThreads / 32; ++w) s += part[threadIdx.x][w];
        out[2 * blockIdx.x + threadIdx.x] = s;
    }
}

}  // namespace vita

using namespace vita;

extern "C" int vita_page_digest(const void* rows, int64_t ld, int64_t n_rows, int64_t H, int64_t page_size,
                                uint64_t* out, void* stream) {
    VITA_REQUIRE(H > 0 && H % 8 == 0, "H must be a positive multiple of 8");
    VITA_REQUIRE(ld >= H && ld % 8 == 0, "ld must be >= H and a multiple of 8");
    VITA_REQUIRE(page_size > 0 && page_size * H / 8 <= 0x7fffffff, "page_size must be positive");
    VITA_REQUIRE(n_rows >= 0, "n_rows must be non-negative");
    const int64_t n_pages = n_rows / page_size;          // a partial last page gets no digest
    if (n_pages == 0) return VITA_OK;
    VITA_REQUIRE(n_pages <= 0x7fffffff, "too many pages");
    VITA_REQUIRE(rows && out, "rows and out are required");
    VITA_REQUIRE(reinterpret_cast<uintptr_t>(rows) % 16 == 0, "rows must be 16-byte aligned");
    page_digest_kernel<<<static_cast<unsigned>(n_pages), kDigestThreads, 0, static_cast<cudaStream_t>(stream)>>>(
        static_cast<const __nv_bfloat16*>(rows), ld, (int)H, (int)page_size, reinterpret_cast<unsigned long long*>(out));
    return check_launch("page_digest");
}
