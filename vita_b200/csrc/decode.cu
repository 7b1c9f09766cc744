// Small kernels of the greedy-decode step (the linears are the wgmma GEMVs of decode_tc.cu):
//   decode_embed   start of a step: consume the previous arg-max, log it, advance the cache length (saturating at the
//                  KV capacity), bump the completion-counter serial, gather the embedding row
//   decode_router  post-attention RMSNorm + router of one token per CTA (stand-alone form; the decode chain uses the
//                  router fused into the gate/up GEMV)
//   argmax_rows / decode_slots   batched decode step (several sequences through the GEMM path)
//
// Reference: the decode step of HF generate() over transformers MixtralDecoderLayer (vita_mixtral.py:158-173,
// video_audio_demo.py:257-270); vLLM twin web_demo/vllm_tools/vllm_file/mixtral.py:491-566.
#include "common.h"
#include "ptx.cuh"

namespace vita {

// (logit, ~index) as one ordered 64-bit key: atomicMax / max picks the largest logit, the lowest index on ties.
// -0.0 is packed as +0.0: the two are equal logits, so the lower index wins between them too (as in torch.argmax).
// (NaN logits are not ordered like torch.argmax does.)
__device__ __forceinline__ unsigned long long pack_argmax(float v, int idx) {
    uint32_t u = __float_as_uint(v);
    if (u == 0x80000000u) u = 0u;
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return (static_cast<unsigned long long>(u) << 32) | static_cast<unsigned long long>(0xFFFFFFFFu - static_cast<uint32_t>(idx));
}

// ------------------------------------------------------------------------------------------------ small kernels
// Start of a decode step: consume the previous arg-max, log it, advance the cache length, gather the embedding.
__global__ void __launch_bounds__(256)
decode_embed_kernel(unsigned long long* best, int* token_log, int* gen_count, int max_log, int* cache_len,
                    int* cur_pos, const __nv_bfloat16* embed, __nv_bfloat16* h, int H, int vocab, int max_ctx,
                    unsigned long long* chain_serial) {
    const int b = blockIdx.x;
    __shared__ int s_tok;
    pdl_launch_dependents();
    pdl_wait();
    if (threadIdx.x == 0) {
        if (b == 0 && chain_serial != nullptr) *chain_serial += 1;   // the step's kernels poll serial x arrivals
        const unsigned long long key = best[b];
        int tok = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(key & 0xFFFFFFFFull));
        if (tok < 0 || tok >= vocab) tok = 0;
        s_tok = tok;
        const int n = gen_count[b];
        if (n < max_log) token_log[static_cast<long long>(b) * max_log + n] = tok;
        gen_count[b] = n + 1;
        // a full cache stays full: the position saturates on the last slot instead of running into the next
        // sequence's block-table row / beyond the rope table (the host refuses such requests up front)
        const int len = cache_len[b];
        cur_pos[b] = len < max_ctx ? len : max_ctx - 1;
        cache_len[b] = len < max_ctx ? len + 1 : max_ctx;
        best[b] = 0ull;
    }
    __syncthreads();
    const uint4* src = reinterpret_cast<const uint4*>(embed + static_cast<long long>(s_tok) * H);
    uint4* dst = reinterpret_cast<uint4*>(h + static_cast<long long>(b) * H);
    for (int i = threadIdx.x; i < (H >> 3); i += blockDim.x) dst[i] = src[i];
}

// post_attention_layernorm + router for one token per block (E = 8 warps).
__global__ void __launch_bounds__(256)
decode_router_kernel(const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ norm_w,
                     const __nv_bfloat16* __restrict__ gate_w, __nv_bfloat16* __restrict__ xn,
                     int* __restrict__ topk_ids, float* __restrict__ topk_w, int H, float eps) {
    extern __shared__ __align__(16) uint8_t smem_r[];
    __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(smem_r);
    __shared__ float red[8];
    __shared__ float logits[8];
    const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const __nv_bfloat16* hr = h + static_cast<long long>(b) * H;
    float ss = 0.0f;
    for (int i = threadIdx.x; i < H; i += 256) { const float v = __bfloat162float(hr[i]); ss += v * v; }
    ss = warp_sum(ss);
    if (lane == 0) red[warp] = ss;
    __syncthreads();
    float tot = 0.0f;
#pragma unroll
    for (int i = 0; i < 8; ++i) tot += red[i];
    const float inv = rsqrtf(tot / static_cast<float>(H) + eps);
    for (int i = threadIdx.x; i < H; i += 256) {
        const __nv_bfloat16 v = __float2bfloat16(__bfloat162float(hr[i]) * inv * __bfloat162float(norm_w[i]));
        xs[i] = v;
        xn[static_cast<long long>(b) * H + i] = v;
    }
    __syncthreads();
    float acc = 0.0f;
    const __nv_bfloat16* gw = gate_w + static_cast<long long>(warp) * H;
    for (int i = lane * 8; i < H; i += 256) {
        const uint4 w = *reinterpret_cast<const uint4*>(gw + i);
        const uint4 x = *reinterpret_cast<const uint4*>(xs + i);
        const uint32_t wa[4] = {w.x, w.y, w.z, w.w}, xa[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) acc += bf16_lo(wa[e]) * bf16_lo(xa[e]) + bf16_hi(wa[e]) * bf16_hi(xa[e]);
    }
    acc = warp_sum(acc);
    if (lane == 0) logits[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = -INFINITY;
        for (int e = 0; e < 8; ++e) m = fmaxf(m, logits[e]);
        float p[8], sum = 0.0f;
        for (int e = 0; e < 8; ++e) { p[e] = expf(logits[e] - m); sum += p[e]; }
        int i0 = 0;
        for (int e = 1; e < 8; ++e) if (p[e] > p[i0]) i0 = e;
        int i1 = (i0 == 0) ? 1 : 0;
        for (int e = 0; e < 8; ++e) if (e != i0 && p[e] > p[i1]) i1 = e;
        const float p0 = p[i0] / sum, p1 = p[i1] / sum, den = p0 + p1;
        topk_ids[b * 2] = i0;
        topk_ids[b * 2 + 1] = i1;
        topk_w[b * 2] = p0 / den;
        topk_w[b * 2 + 1] = p1 / den;
    }
}

// Row-wise arg-max of bf16 logits (first index on ties, like torch.argmax), packed like the GEMV kernels do.
__global__ void __launch_bounds__(256)
argmax_rows_kernel(const __nv_bfloat16* __restrict__ logits, unsigned long long* __restrict__ best, int V) {
    __shared__ unsigned long long red[8];
    const __nv_bfloat16* row = logits + static_cast<long long>(blockIdx.x) * V;
    unsigned long long loc = 0ull;
    for (int i = threadIdx.x; i < V; i += 256) {
        const unsigned long long k = pack_argmax(__bfloat162float(row[i]), i);
        loc = k > loc ? k : loc;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, loc, o);
        loc = other > loc ? other : loc;
    }
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = loc;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long m = red[0];
        for (int i = 1; i < 8; ++i) m = red[i] > m ? red[i] : m;
        best[blockIdx.x] = m;
    }
}

// slots[b] = paged-KV slot of position cur_pos[b] of sequence b (batched decode through the GEMM path)
__global__ void decode_slots_kernel(const int* __restrict__ cur_pos, const int* __restrict__ block_table,
                                    int* __restrict__ slots, int B, int page_size, int max_pages) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const int pos = cur_pos[b];
    slots[b] = block_table[static_cast<long long>(b) * max_pages + pos / page_size] * page_size + pos % page_size;
}

}  // namespace vita

using namespace vita;


extern "C" int vita_argmax_rows(const void* logits, uint64_t* best, int64_t B, int64_t V, void* stream) {
    if (B == 0) return VITA_OK;
    argmax_rows_kernel<<<static_cast<unsigned>(B), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        BF16C(logits), reinterpret_cast<unsigned long long*>(best), (int)V);
    return check_launch("argmax_rows");
}

extern "C" int vita_decode_slots(const int32_t* cur_pos, const int32_t* block_table, int32_t* slots, int64_t B,
                                 int64_t page_size, int64_t max_pages, void* stream) {
    if (B == 0) return VITA_OK;
    decode_slots_kernel<<<static_cast<unsigned>((B + 63) / 64), 64, 0, static_cast<cudaStream_t>(stream)>>>(
        cur_pos, block_table, slots, (int)B, (int)page_size, (int)max_pages);
    return check_launch("decode_slots");
}

extern "C" int vita_decode_embed(uint64_t* best, int32_t* token_log, int32_t* gen_count, int64_t max_log,
                                 int32_t* cache_len, int32_t* cur_pos, const void* embed, void* h, int64_t B,
                                 int64_t H, int64_t vocab, int64_t max_ctx, uint64_t* chain_serial, void* stream) {
    VITA_REQUIRE(H % 8 == 0, "H must be a multiple of 8");
    VITA_REQUIRE(max_ctx > 0 && max_ctx <= 0x7fffffff, "max_ctx (KV capacity per sequence) must be positive");
    if (B == 0) return VITA_OK;
    cudaError_t e = launch_chain(decode_embed_kernel, dim3(static_cast<unsigned>(B)), dim3(256), 0,
                                 static_cast<cudaStream_t>(stream), reinterpret_cast<unsigned long long*>(best),
                                 token_log, gen_count, (int)max_log, cache_len, cur_pos, BF16C(embed),
                                 static_cast<__nv_bfloat16*>(h), (int)H, (int)vocab, (int)max_ctx,
                                 reinterpret_cast<unsigned long long*>(chain_serial));
    if (e != cudaSuccess) return check_cuda(e, "decode_embed");
    return check_launch("decode_embed");
}



extern "C" int vita_decode_router(const void* h, const void* norm_w, const void* gate_w, void* xn, int32_t* topk_ids,
                                  float* topk_w, int64_t B, int64_t H, int64_t E, float eps, void* stream) {
    VITA_REQUIRE(E == 8, "router is specialised for 8 experts (Mixtral-8x7B)");
    VITA_REQUIRE(H % 8 == 0 && H * 2 <= 48 * 1024, "H must be a multiple of 8 and fit 48 KB of shared memory");
    if (B == 0) return VITA_OK;
    decode_router_kernel<<<static_cast<unsigned>(B), 256, H * 2, static_cast<cudaStream_t>(stream)>>>(
        BF16C(h), BF16C(norm_w), BF16C(gate_w), static_cast<__nv_bfloat16*>(xn), topk_ids, topk_w, (int)H, eps);
    return check_launch("decode_router");
}



