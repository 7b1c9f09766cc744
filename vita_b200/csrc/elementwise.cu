// HBM-bound row kernels of the omni forward path: norms, embedding gather / splice scatter, RoPE + paged-KV write,
// MoE router / align / gather / combine, and the im2col / layout kernels that feed the wgmma GEMM for the
// convolutional front-ends.  All of them are one-pass, 16-byte vectorised, fp32 math, bf16 storage.
#include "common.h"
#include "ptx.cuh"

namespace vita {

// ------------------------------------------------------------------------------------------------ helpers
template <int THREADS>
__device__ __forceinline__ float block_sum(float v, float* red) {
    v = warp_sum(v);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) red[w] = v;
    __syncthreads();
    float t = (l < THREADS / 32) ? red[l] : 0.0f;
    t = warp_sum(t);
    __syncthreads();
    return t;
}

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
    f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
    f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
    uint4 o;
    o.x = pack_bf16(f[0], f[1]); o.y = pack_bf16(f[2], f[3]); o.z = pack_bf16(f[4], f[5]); o.w = pack_bf16(f[6], f[7]);
    return o;
}

// ------------------------------------------------------------------------------------------------ RMSNorm
// transformers MixtralRMSNorm.forward (modeling_mixtral.py:148-153): fp32 variance, eps inside rsqrt.
// One block per row; the row is kept in registers between the two passes (H <= 8 * 8 * THREADS).
template <int THREADS, int VPT>
__global__ void __launch_bounds__(THREADS)
rmsnorm_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w, __nv_bfloat16* __restrict__ y,
               int H, float eps) {
    __shared__ float red[32];
    const long long row = blockIdx.x;
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * H);
    const int nvec = H >> 3;
    uint4 v[VPT];
    float ss = 0.0f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        if (idx < nvec) {
            v[i] = xr[idx];
            float f[8];
            unpack8(v[i], f);
#pragma unroll
            for (int j = 0; j < 8; ++j) ss += f[j] * f[j];
        }
    }
    const float tot = block_sum<THREADS>(ss, red);
    const float inv = rsqrtf(tot / static_cast<float>(H) + eps);
    const uint4* wr = reinterpret_cast<const uint4*>(w);
    uint4* yr = reinterpret_cast<uint4*>(y + row * H);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        if (idx < nvec) {
            float f[8], g[8];
            unpack8(v[i], f);
            unpack8(__ldg(wr + idx), g);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] = f[j] * inv * g[j];
            yr[idx] = pack8(f);
        }
    }
}

// ------------------------------------------------------------------------------------------------ LayerNorm
// torch.nn.LayerNorm (biased variance), optional activation and output scale.  Used by InternViT norm1/norm2
// (modeling_intern_vit.py:229-230), Whale norm1/norm2/after_norm/embed LayerNorm (transformer.py:88-89,313-318,371)
// and the adapter LayerNorm(eps=1e-3)+GELU (adapter.py:98-104).
template <int THREADS, int VPT>
__global__ void __launch_bounds__(THREADS)
layernorm_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ w,
                 const __nv_bfloat16* __restrict__ b, __nv_bfloat16* __restrict__ y, int H, float eps, int act,
                 float out_scale) {
    __shared__ float red[32];
    const long long row = blockIdx.x;
    const uint4* xr = reinterpret_cast<const uint4*>(x + row * H);
    const int nvec = H >> 3;
    uint4 v[VPT];
    float s = 0.0f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        if (idx < nvec) {
            v[i] = xr[idx];
            float f[8];
            unpack8(v[i], f);
#pragma unroll
            for (int j = 0; j < 8; ++j) s += f[j];
        }
    }
    const float mean = block_sum<THREADS>(s, red) / static_cast<float>(H);
    float ss = 0.0f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        if (idx < nvec) {
            float f[8];
            unpack8(v[i], f);
#pragma unroll
            for (int j = 0; j < 8; ++j) { const float d = f[j] - mean; ss += d * d; }
        }
    }
    const float var = block_sum<THREADS>(ss, red) / static_cast<float>(H);
    const float inv = rsqrtf(var + eps);
    const uint4* wr = reinterpret_cast<const uint4*>(w);
    const uint4* br = reinterpret_cast<const uint4*>(b);
    uint4* yr = reinterpret_cast<uint4*>(y + row * H);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        if (idx < nvec) {
            float f[8], g[8], c[8];
            unpack8(v[i], f);
            unpack8(__ldg(wr + idx), g);
            unpack8(__ldg(br + idx), c);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                float o = (f[j] - mean) * inv * g[j] + c[j];
                if (act == VITA_ACT_RELU) o = fmaxf(o, 0.0f);
                else if (act == VITA_ACT_GELU) o = gelu_erf(o);
                f[j] = o * out_scale;
            }
            yr[idx] = pack8(f);
        }
    }
}

// ------------------------------------------------------------------------------------------------ row gather / scatter
// out[dst_index ? dst_index[i] : i] = table[src_index ? src_index[i] : i]; rows with a negative index are skipped.
// Covers embed_tokens lookup (vita_arch.py:274), the placeholder splice (vita_arch.py:277-303; vLLM twin
// mixtral.py:1116,1126) and the MoE token permute.
__global__ void __launch_bounds__(256)
row_copy_kernel(const __nv_bfloat16* __restrict__ table, const int* __restrict__ src_index,
                const int* __restrict__ dst_index, __nv_bfloat16* __restrict__ out, int n_rows, int H) {
    const int nvec = H >> 3;
    for (long long row = blockIdx.x; row < n_rows; row += gridDim.x) {
        const int s = src_index ? src_index[row] : static_cast<int>(row);
        const int d = dst_index ? dst_index[row] : static_cast<int>(row);
        if (s < 0 || d < 0) continue;
        const uint4* sp = reinterpret_cast<const uint4*>(table + static_cast<long long>(s) * H);
        uint4* dp = reinterpret_cast<uint4*>(out + static_cast<long long>(d) * H);
        for (int i = threadIdx.x; i < nvec; i += blockDim.x) dp[i] = sp[i];
    }
}

// ------------------------------------------------------------------------------------------------ RoPE + paged KV write
// transformers apply_rotary_pos_emb / rotate_half (modeling_mixtral.py:224-254): out = x*cos + rotate_half(x)*sin with
// cos/sin = [f0..f63, f0..f63].  cos_sin: fp32 [max_pos, 2, D/2].  qkv rows: [q heads | k heads | v heads] x D.
// K (rotated) and V are additionally written into the paged cache: cache[slot][kv_head][D], slot = slot_mapping[tok].
template <int D>
__global__ void __launch_bounds__(256)
rope_kv_write_kernel(__nv_bfloat16* __restrict__ qkv, const int* __restrict__ positions,
                     const int* __restrict__ slot_mapping, const float* __restrict__ cos_sin,
                     __nv_bfloat16* __restrict__ k_cache, __nv_bfloat16* __restrict__ v_cache, int n_tok, int n_q,
                     int n_kv) {
    constexpr int HALF = D / 2;
    const int tok = blockIdx.x;
    const int pos = positions[tok];
    const int slot = slot_mapping ? slot_mapping[tok] : -1;
    const float* cs = cos_sin + static_cast<long long>(pos) * D;
    __nv_bfloat16* row = qkv + static_cast<long long>(tok) * (n_q + 2 * n_kv) * D;
    const int n_rot = (n_q + n_kv) * HALF;  // rotated pairs
    for (int i = threadIdx.x; i < n_rot; i += blockDim.x) {
        const int head = i / HALF, j = i % HALF;
        __nv_bfloat16* h = row + head * D;
        const float x1 = __bfloat162float(h[j]), x2 = __bfloat162float(h[j + HALF]);
        const float c = cs[j], s = cs[HALF + j];
        float r1, r2;
        rope_rotate(x1, x2, c, s, r1, r2);
        const __nv_bfloat16 o1 = __float2bfloat16(r1);
        const __nv_bfloat16 o2 = __float2bfloat16(r2);
        h[j] = o1;
        h[j + HALF] = o2;
        if (head >= n_q && slot >= 0) {
            __nv_bfloat16* kc = k_cache + (static_cast<long long>(slot) * n_kv + (head - n_q)) * D;
            kc[j] = o1;
            kc[j + HALF] = o2;
        }
    }
    if (slot >= 0) {
        const __nv_bfloat16* vsrc = row + (n_q + n_kv) * D;
        __nv_bfloat16* vdst = v_cache + static_cast<long long>(slot) * n_kv * D;
        const int nvec = n_kv * D / 8;
        for (int i = threadIdx.x; i < nvec; i += blockDim.x)
            reinterpret_cast<uint4*>(vdst)[i] = reinterpret_cast<const uint4*>(vsrc)[i];
    }
}

// ------------------------------------------------------------------------------------------------ MoE router
// post_attention_layernorm + MixtralTopKRouter (modeling_mixtral.py:109-116): logits = xn . Wg^T on the bf16-rounded
// normed activations, fp32 softmax over E, top-2 (first index wins ties, as torch.topk), renormalise by the pair sum.
// One 128-thread CTA per token (the row stays in registers between the two passes), whatever the token count: the
// bits of a token's routing do not depend on how many tokens share the launch.  Also writes xn (the expert GEMM input).
template <int E>
__global__ void __launch_bounds__(128)
rmsnorm_router_kernel(const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ norm_w,
                      const __nv_bfloat16* __restrict__ gate_w, __nv_bfloat16* __restrict__ xn,
                      int* __restrict__ topk_ids, float* __restrict__ topk_w, int n_tok, int H, float eps) {
    constexpr int MAXV = 4;                      // 128 threads x 4 x 8 elements = H <= 4096
    __shared__ float red[4][E + 1];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tok = blockIdx.x;
    const uint4* hr = reinterpret_cast<const uint4*>(h + static_cast<long long>(tok) * H);
    const int nvec = H >> 3;
    uint4 hv[MAXV];
    float ss = 0.0f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int i = threadIdx.x + j * 128;
        if (i < nvec) {
            hv[j] = hr[i];
            float f[8];
            unpack8(hv[j], f);
#pragma unroll
            for (int q = 0; q < 8; ++q) ss += f[q] * f[q];
        }
    }
    ss = warp_sum(ss);
    if (lane == 0) red[warp][E] = ss;
    __syncthreads();
    const float inv = rsqrtf((red[0][E] + red[1][E] + red[2][E] + red[3][E]) / static_cast<float>(H) + eps);
    float logit[E];
#pragma unroll
    for (int e = 0; e < E; ++e) logit[e] = 0.0f;
    uint4* xr = reinterpret_cast<uint4*>(xn + static_cast<long long>(tok) * H);
    const uint4* nw = reinterpret_cast<const uint4*>(norm_w);
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int i = threadIdx.x + j * 128;
        if (i < nvec) {
            float f[8], g[8];
            unpack8(hv[j], f);
            unpack8(__ldg(nw + i), g);
#pragma unroll
            for (int q = 0; q < 8; ++q) f[q] = f[q] * inv * g[q];
            const uint4 packed = pack8(f);
            xr[i] = packed;
            unpack8(packed, f);  // router sees the bf16-rounded activations
#pragma unroll
            for (int e = 0; e < E; ++e) {
                float wv[8];
                unpack8(__ldg(reinterpret_cast<const uint4*>(gate_w + static_cast<long long>(e) * H) + i), wv);
#pragma unroll
                for (int q = 0; q < 8; ++q) logit[e] += f[q] * wv[q];
            }
        }
    }
#pragma unroll
    for (int e = 0; e < E; ++e) {
        logit[e] = warp_sum(logit[e]);
        if (lane == 0) red[warp][e] = logit[e];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = -INFINITY;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            logit[e] = (red[0][e] + red[1][e]) + (red[2][e] + red[3][e]);
            m = fmaxf(m, logit[e]);
        }
        float p[E], sum = 0.0f;
#pragma unroll
        for (int e = 0; e < E; ++e) { p[e] = expf(logit[e] - m); sum += p[e]; }
        int i0 = 0;
#pragma unroll
        for (int e = 1; e < E; ++e) if (p[e] > p[i0]) i0 = e;
        int i1 = (i0 == 0) ? 1 : 0;
#pragma unroll
        for (int e = 0; e < E; ++e) if (e != i0 && p[e] > p[i1]) i1 = e;
        const float p0 = p[i0] / sum, p1 = p[i1] / sum;
        const float den = p0 + p1;
        topk_ids[tok * 2] = i0;
        topk_ids[tok * 2 + 1] = i1;
        topk_w[tok * 2] = p0 / den;
        topk_w[tok * 2 + 1] = p1 / den;
    }
}

// The same router with the token permute fused in ("fused top-2 router + token permute/scatter"): every expert owns
// `capacity` consecutive rows of x_slots; the CTA of a token claims one row in each of its two experts (atomicAdd on the
// expert's counter) and stores the normed activations there directly -- no offsets pass, no gather pass.  The order of the
// rows inside an expert depends on the arrival order of the CTAs; every row is processed independently by the grouped
// GEMMs, so the results do not.  perm_row[t, k] = the claimed row (what vita_moe_combine gathers by).
template <int E>
__global__ void __launch_bounds__(128)
rmsnorm_router_scatter_kernel(const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ norm_w,
                              const __nv_bfloat16* __restrict__ gate_w, __nv_bfloat16* __restrict__ x_slots,
                              int* __restrict__ expert_counts, int* __restrict__ perm_row,
                              float* __restrict__ row_weight, int* __restrict__ topk_ids, float* __restrict__ topk_w,
                              int n_tok, int H, int capacity, float eps) {
    constexpr int MAXV = 4;
    __shared__ float red[4][E + 1];
    __shared__ int dst[2];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int tok = blockIdx.x;
    const uint4* hr = reinterpret_cast<const uint4*>(h + static_cast<long long>(tok) * H);
    const int nvec = H >> 3;
    uint4 hv[MAXV];
    float ss = 0.0f;
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int i = threadIdx.x + j * 128;
        if (i < nvec) {
            hv[j] = hr[i];
            float f[8];
            unpack8(hv[j], f);
#pragma unroll
            for (int q = 0; q < 8; ++q) ss += f[q] * f[q];
        }
    }
    ss = warp_sum(ss);
    if (lane == 0) red[warp][E] = ss;
    __syncthreads();
    const float inv = rsqrtf((red[0][E] + red[1][E] + red[2][E] + red[3][E]) / static_cast<float>(H) + eps);
    float logit[E];
#pragma unroll
    for (int e = 0; e < E; ++e) logit[e] = 0.0f;
    const uint4* nw = reinterpret_cast<const uint4*>(norm_w);
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int i = threadIdx.x + j * 128;
        if (i < nvec) {
            float f[8], g[8];
            unpack8(hv[j], f);
            unpack8(__ldg(nw + i), g);
#pragma unroll
            for (int q = 0; q < 8; ++q) f[q] = f[q] * inv * g[q];
            hv[j] = pack8(f);      // the normed row stays in registers until its two destinations are known
            unpack8(hv[j], f);     // router sees the bf16-rounded activations
#pragma unroll
            for (int e = 0; e < E; ++e) {
                float wv[8];
                unpack8(__ldg(reinterpret_cast<const uint4*>(gate_w + static_cast<long long>(e) * H) + i), wv);
#pragma unroll
                for (int q = 0; q < 8; ++q) logit[e] += f[q] * wv[q];
            }
        }
    }
#pragma unroll
    for (int e = 0; e < E; ++e) {
        logit[e] = warp_sum(logit[e]);
        if (lane == 0) red[warp][e] = logit[e];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = -INFINITY;
#pragma unroll
        for (int e = 0; e < E; ++e) {
            logit[e] = (red[0][e] + red[1][e]) + (red[2][e] + red[3][e]);
            m = fmaxf(m, logit[e]);
        }
        float p[E], sum = 0.0f;
#pragma unroll
        for (int e = 0; e < E; ++e) { p[e] = expf(logit[e] - m); sum += p[e]; }
        int i0 = 0;
#pragma unroll
        for (int e = 1; e < E; ++e) if (p[e] > p[i0]) i0 = e;
        int i1 = (i0 == 0) ? 1 : 0;
#pragma unroll
        for (int e = 0; e < E; ++e) if (e != i0 && p[e] > p[i1]) i1 = e;
        const float p0 = p[i0] / sum, p1 = p[i1] / sum;
        const float den = p0 + p1;
        const int r0 = i0 * capacity + atomicAdd(&expert_counts[i0], 1);
        const int r1 = i1 * capacity + atomicAdd(&expert_counts[i1], 1);
        dst[0] = r0;
        dst[1] = r1;
        perm_row[tok * 2] = r0;
        perm_row[tok * 2 + 1] = r1;
        row_weight[r0] = p0 / den;
        row_weight[r1] = p1 / den;
        if (topk_ids) {
            topk_ids[tok * 2] = i0;
            topk_ids[tok * 2 + 1] = i1;
            topk_w[tok * 2] = p0 / den;
            topk_w[tok * 2 + 1] = p1 / den;
        }
    }
    __syncthreads();
    uint4* x0 = reinterpret_cast<uint4*>(x_slots + static_cast<long long>(dst[0]) * H);
    uint4* x1 = reinterpret_cast<uint4*>(x_slots + static_cast<long long>(dst[1]) * H);
#pragma unroll
    for (int j = 0; j < MAXV; ++j) {
        const int i = threadIdx.x + j * 128;
        if (i < nvec) {
            x0[i] = hv[j];
            x1[i] = hv[j];
        }
    }
}

// ------------------------------------------------------------------------------------------------ MoE align
// Stable counting sort of the (token, k) assignments by expert.  Single block, warp e owns expert e.
//   expert_offsets[E+1] : first permuted row of each expert
//   perm_row[n*2]       : permuted row of assignment (t, k)
//   row_token[n*2]      : source token of each permuted row
//   row_weight[n*2]     : routing weight of each permuted row (fp32)
__global__ void __launch_bounds__(1024)
moe_align_kernel(const int* __restrict__ topk_ids, const float* __restrict__ topk_w, int* __restrict__ expert_offsets,
                 int* __restrict__ perm_row, int* __restrict__ row_token, float* __restrict__ row_weight,
                 int* __restrict__ row_assign, int n_assign, int E) {
    __shared__ int counts[32];
    __shared__ int offs[33];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp < E) {
        int c = 0;
        for (int i = lane; i < n_assign; i += 32) c += (topk_ids[i] == warp);
        c = static_cast<int>(warp_sum(static_cast<float>(c)) + 0.5f);
        if (lane == 0) counts[warp] = c;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int e = 0; e < E; ++e) { offs[e] = acc; acc += counts[e]; }
        offs[E] = acc;
        for (int e = 0; e <= E; ++e) expert_offsets[e] = offs[e];
    }
    __syncthreads();
    if (warp < E) {
        int base = offs[warp];
        for (int i0 = 0; i0 < n_assign; i0 += 32) {
            const int i = i0 + lane;
            const bool mine = (i < n_assign) && (topk_ids[i] == warp);
            const unsigned m = __ballot_sync(0xffffffffu, mine);
            if (mine) {
                const int r = base + __popc(m & ((1u << lane) - 1));
                perm_row[i] = r;
                row_token[r] = i >> 1;
                row_weight[r] = topk_w[i];
                if (row_assign) row_assign[r] = i;
            }
            base += __popc(m);
        }
    }
}

// E <= 8: every thread owns a contiguous chunk of the assignments (so the order inside an expert stays the assignment
// order), counts its chunk per expert, the block scans the counts (warp shuffles + one smem level), and the thread walks
// its chunk a second time handing out rows.  Two passes over 8 items per thread at S = 4096 instead of 256 ballot rounds
// per warp (56 us -> a few us per layer).
__global__ void __launch_bounds__(1024)
moe_align8_kernel(const int* __restrict__ topk_ids, const float* __restrict__ topk_w, int* __restrict__ expert_offsets,
                  int* __restrict__ perm_row, int* __restrict__ row_token, float* __restrict__ row_weight,
                  int* __restrict__ row_assign, int n_assign, int E) {
    __shared__ int warp_tot[32][8];
    __shared__ int base[9];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ipt = (n_assign + 1023) >> 10;
    const int i0 = threadIdx.x * ipt, i1 = min(n_assign, i0 + ipt);
    int cnt[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) cnt[e] = 0;
    for (int i = i0; i < i1; ++i) {
        const int id = topk_ids[i];
#pragma unroll
        for (int e = 0; e < 8; ++e) cnt[e] += (id == e);
    }
    int pre[8];   // exclusive prefix of this thread inside the block, per expert
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        int v = cnt[e];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int n = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += n;
        }
        pre[e] = v - cnt[e];
        if (lane == 31) warp_tot[warp][e] = v;
    }
    __syncthreads();
    if (warp < 8) {   // warp e scans the 32 warp totals of expert e
        const int t = warp_tot[lane][warp];
        int v = t;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int n = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += n;
        }
        warp_tot[lane][warp] = v - t;          // exclusive prefix of the warp
        if (lane == 31) base[warp] = v;        // total of the expert (turned into its first row below)
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int acc = 0;
        for (int e = 0; e < 8; ++e) { const int c = base[e]; base[e] = acc; acc += c; }
        base[8] = acc;
        for (int e = 0; e <= E; ++e) expert_offsets[e] = base[e < 8 ? e : 8];
    }
    __syncthreads();
    int nxt[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) nxt[e] = base[e] + warp_tot[warp][e] + pre[e];
    for (int i = i0; i < i1; ++i) {
        const int id = topk_ids[i];
        int r = 0;
#pragma unroll
        for (int e = 0; e < 8; ++e)
            if (id == e) { r = nxt[e]; nxt[e] = r + 1; }
        perm_row[i] = r;
        row_token[r] = i >> 1;
        row_weight[r] = topk_w[i];
        if (row_assign) row_assign[r] = i;
    }
}

// ------------------------------------------------------------------------------------------------ MoE combine
// MixtralExperts.forward index_add_ (modeling_mixtral.py:96) + the decoder-layer residual add, optionally followed
// by the next RMSNorm (next layer's input_layernorm or the final norm) so the residual stream is read once.
template <int THREADS, int VPT>
__global__ void __launch_bounds__(THREADS)
moe_combine_kernel(__nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ y_perm,
                   const int* __restrict__ perm_row, const __nv_bfloat16* __restrict__ next_norm_w,
                   __nv_bfloat16* __restrict__ xn_out, int H, float eps) {
    __shared__ float red[32];
    const long long tok = blockIdx.x;
    const int r0 = perm_row[tok * 2], r1 = perm_row[tok * 2 + 1];
    const int nvec = H >> 3;
    uint4* hr = reinterpret_cast<uint4*>(h + tok * H);
    const uint4* y0 = reinterpret_cast<const uint4*>(y_perm + static_cast<long long>(r0) * H);
    const uint4* y1 = reinterpret_cast<const uint4*>(y_perm + static_cast<long long>(r1) * H);
    uint4 v[VPT];
    float ss = 0.0f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        if (idx < nvec) {
            float a[8], b[8], c[8];
            unpack8(hr[idx], a);
            unpack8(y0[idx], b);
            unpack8(y1[idx], c);
#pragma unroll
            for (int j = 0; j < 8; ++j) a[j] = a[j] + (b[j] + c[j]);
            v[i] = pack8(a);
            hr[idx] = v[i];
            unpack8(v[i], a);
#pragma unroll
            for (int j = 0; j < 8; ++j) ss += a[j] * a[j];
        }
    }
    if (next_norm_w == nullptr) return;
    const float tot = block_sum<THREADS>(ss, red);
    const float inv = rsqrtf(tot / static_cast<float>(H) + eps);
    const uint4* wr = reinterpret_cast<const uint4*>(next_norm_w);
    uint4* xr = reinterpret_cast<uint4*>(xn_out + tok * H);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        if (idx < nvec) {
            float f[8], g[8];
            unpack8(v[i], f);
            unpack8(__ldg(wr + idx), g);
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] = f[j] * inv * g[j];
            xr[idx] = pack8(f);
        }
    }
}

// ------------------------------------------------------------------------------------------------ expert-parallel tail
// Flags live in symmetric memory: flags[which][src_rank] of every rank is written by src_rank with a monotonically
// increasing epoch (st.release.sys after a system fence), waited for with ld.acquire.sys.
__device__ __forceinline__ void sys_wait_flag(const int* flag, int epoch) {
    int v;
    long long t0 = clock64();
    do {
        asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
        if (v < epoch && clock64() - t0 > VITA_MBAR_TIMEOUT_CYCLES * 4) {
            printf("[vita] EP flag timeout: block %d waits for epoch %d, sees %d\n", blockIdx.x, epoch, v);
            __trap();
        }
    } while (v < epoch);
}

__global__ void ep_signal_kernel(int* const* __restrict__ peer_flags, int which, int n_ranks, int my_rank, int epoch) {
    __threadfence_system();
    if (threadIdx.x < n_ranks) {
        int* f = peer_flags[threadIdx.x] + which * n_ranks + my_rank;
        asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(f), "r"(epoch) : "memory");
    }
}

__global__ void ep_wait_kernel(const int* __restrict__ my_flags, int which, int n_ranks, int n_wait, int epoch) {
    if (threadIdx.x < n_wait) sys_wait_flag(my_flags + which * n_ranks + threadIdx.x, epoch);
}

// All-gather by P2P stores: byte ranges of this rank's symmetric buffer go to the same offsets of every peer.
struct PushRanges {
    long long off[4];
    long long bytes[4];
    int n;
};
__global__ void __launch_bounds__(256)
ep_push_kernel(uint8_t* const* __restrict__ peer_base, const PushRanges r, int n_ranks, int my_rank) {
    const uint8_t* src_base = peer_base[my_rank];
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    for (int i = 0; i < r.n; ++i) {
        const uint4* src = reinterpret_cast<const uint4*>(src_base + r.off[i]);
        const long long nvec = r.bytes[i] >> 4;
        for (long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; v < nvec; v += stride) {
            const uint4 x = src[v];
            for (int d = 1; d < n_ranks; ++d) {      // start at a different peer per rank: spreads the NVSwitch ports
                const int peer = (my_rank + d) % n_ranks;
                reinterpret_cast<uint4*>(peer_base[peer] + r.off[i])[v] = x;
            }
        }
        // tail of a range that is not a 16-byte multiple (e.g. an odd number of 8-byte routing records): 4-byte words
        const long long tail0 = nvec << 4, nword = (r.bytes[i] - tail0) >> 2;
        if (blockIdx.x == 0 && threadIdx.x < nword) {
            const uint32_t x = *reinterpret_cast<const uint32_t*>(src_base + r.off[i] + tail0 + threadIdx.x * 4);
            for (int d = 1; d < n_ranks; ++d) {
                const int peer = (my_rank + d) % n_ranks;
                *reinterpret_cast<uint32_t*>(peer_base[peer] + r.off[i] + tail0 + threadIdx.x * 4) = x;
            }
        }
    }
}

// Owner side of the expert-parallel combine: for each owned token t (one block each)
//   h[t] += slot0[t] + slot1[t]      (the two expert outputs, pushed by the ranks holding those experts)
//   xn[t] = RMSNorm(h[t]) * w        (optional)
// and both rows are written into every rank's h / xn (all-gather by P2P stores).
template <int THREADS, int VPT>
__global__ void __launch_bounds__(THREADS)
ep_reduce_norm_gather_kernel(const __nv_bfloat16* __restrict__ rs_buf, const int* __restrict__ my_flags,
                             __nv_bfloat16* const* __restrict__ peer_h, __nv_bfloat16* const* __restrict__ peer_xn,
                             const __nv_bfloat16* __restrict__ next_norm_w, int tok0, int n_ranks, int my_rank, int epoch,
                             int H, float eps, int gather) {
    __shared__ float red[32];
    if (threadIdx.x < n_ranks) sys_wait_flag(my_flags + threadIdx.x, epoch);   // flags[0][src]: partial rows landed
    __syncthreads();
    const int lt = blockIdx.x;                    // local token index inside my chunk
    const long long tok = tok0 + lt;
    const int nvec = H >> 3;
    const uint4* hr = reinterpret_cast<const uint4*>(peer_h[my_rank] + tok * H);
    const uint4* s0 = reinterpret_cast<const uint4*>(rs_buf + (static_cast<long long>(lt) * 2) * H);
    const uint4* s1 = reinterpret_cast<const uint4*>(rs_buf + (static_cast<long long>(lt) * 2 + 1) * H);
    uint4 v[VPT];
    float ss = 0.0f;
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        if (idx < nvec) {
            float a[8], b[8], c[8];
            unpack8(hr[idx], a);
            unpack8(__ldcv(s0 + idx), b);
            unpack8(__ldcv(s1 + idx), c);
#pragma unroll
            for (int j = 0; j < 8; ++j) a[j] = a[j] + (b[j] + c[j]);
            v[i] = pack8(a);
            unpack8(v[i], a);
#pragma unroll
            for (int j = 0; j < 8; ++j) ss += a[j] * a[j];
        }
    }
    const float tot = block_sum<THREADS>(ss, red);
    const float inv = rsqrtf(tot / static_cast<float>(H) + eps);
    const uint4* wr = reinterpret_cast<const uint4*>(next_norm_w);
#pragma unroll
    for (int i = 0; i < VPT; ++i) {
        const int idx = threadIdx.x + i * THREADS;
        if (idx < nvec) {
            uint4 xo = make_uint4(0, 0, 0, 0);
            if (next_norm_w) {
                float f[8], g[8];
                unpack8(v[i], f);
                unpack8(__ldg(wr + idx), g);
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] = f[j] * inv * g[j];
                xo = pack8(f);
            }
            for (int r = gather ? 0 : my_rank; r < (gather ? n_ranks : my_rank + 1); ++r) {
                reinterpret_cast<uint4*>(peer_h[r] + tok * H)[idx] = v[i];
                if (next_norm_w) reinterpret_cast<uint4*>(peer_xn[r] + tok * H)[idx] = xo;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ InternViT front/back
// Patch-embed Conv2d(3,1024,k=14,s=14) (modeling_intern_vit.py:80-85,109) as im2col + GEMM.  Row = (image, py, px),
// column = c*196 + ky*14 + kx (the conv weight's own [out, c, ky, kx] flattening), zero-padded to k_pad columns.
__global__ void __launch_bounds__(256)
vit_im2col_kernel(const __nv_bfloat16* __restrict__ img, __nv_bfloat16* __restrict__ out, int n_img, int C, int HW,
                  int P, int k_pad) {
    const int grid_w = HW / P;
    const long long patch = blockIdx.x;  // over n_img * grid_w * grid_w
    const int n = static_cast<int>(patch / (grid_w * grid_w));
    const int rem = static_cast<int>(patch % (grid_w * grid_w));
    const int py = rem / grid_w, px = rem % grid_w;
    const int kk = C * P * P;
    __nv_bfloat16* o = out + patch * k_pad;
    for (int i = threadIdx.x; i < k_pad; i += blockDim.x) {
        __nv_bfloat16 val = __float2bfloat16(0.0f);
        if (i < kk) {
            const int c = i / (P * P), r = i % (P * P);
            const int ky = r / P, kx = r % P;
            val = img[((static_cast<long long>(n) * C + c) * HW + (py * P + ky)) * HW + (px * P + kx)];
        }
        o[i] = val;
    }
}

// embeddings = cat([cls, patches]) + position_embedding  (modeling_intern_vit.py:112-121; at 448 px the bicubic
// resample of the position table is the identity).  patches: [n_img * n_patch, H] (bias already added by the GEMM).
__global__ void __launch_bounds__(128)
vit_assemble_kernel(const __nv_bfloat16* __restrict__ patches, const __nv_bfloat16* __restrict__ cls,
                    const __nv_bfloat16* __restrict__ pos, __nv_bfloat16* __restrict__ out, int n_patch, int H) {
    const int tok = blockIdx.x % (n_patch + 1);
    const long long n = blockIdx.x / (n_patch + 1);
    const uint4* src = reinterpret_cast<const uint4*>(tok == 0 ? cls : patches + (n * n_patch + tok - 1) * H);
    const uint4* pp = reinterpret_cast<const uint4*>(pos + static_cast<long long>(tok) * H);
    uint4* dst = reinterpret_cast<uint4*>(out + static_cast<long long>(blockIdx.x) * H);
    for (int i = threadIdx.x; i < (H >> 3); i += blockDim.x) {
        float a[8], b[8];
        unpack8(src[i], a);
        unpack8(pp[i], b);
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] += b[j];
        dst[i] = pack8(a);
    }
}

// feature_select (drop CLS) -> x0.5 -> pixel_shuffle(scale 0.5)  (internvit_encoder.py:35-53,71-77).
// Input h [n_img, 1 + g*g, C]; output [n_img, (g/2)*(g/2), 4C].  Following the two view/permute steps of the
// reference: out[n, a, b, q*2C + p*C + c] = 0.5 * x[n, w = 2a + q, h = 2b + p, c]  where x[n, w, h, c] is the
// g x g token grid in row-major token order (w = token // g, h = token % g) and the output token is a*(g/2) + b.
__global__ void __launch_bounds__(128)
vit_pixel_shuffle_kernel(const __nv_bfloat16* __restrict__ h, __nv_bfloat16* __restrict__ out, int g, int C,
                         float scale) {
    const int g2 = g / 2;
    const int o_tok = blockIdx.x % (g2 * g2);
    const long long n = blockIdx.x / (g2 * g2);
    const int a = o_tok / g2, b = o_tok % g2;
    uint4* dst = reinterpret_cast<uint4*>(out + static_cast<long long>(blockIdx.x) * 4 * C);
    const int cvec = C >> 3;
    for (int i = threadIdx.x; i < 4 * cvec; i += blockDim.x) {
        const int blk = i / cvec, ci = i % cvec;
        const int q = blk >> 1, p = blk & 1;
        const int w_idx = 2 * a + q;   // first grid index of the source token
        const int h_idx = 2 * b + p;   // second grid index
        const long long src_tok = 1 + static_cast<long long>(w_idx) * g + h_idx;
        const uint4 v = reinterpret_cast<const uint4*>(h + (n * (g * g + 1) + src_tok) * C)[ci];
        float f[8];
        unpack8(v, f);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] *= scale;
        dst[i] = pack8(f);
    }
}

// ------------------------------------------------------------------------------------------------ Whale front-end
// GlobalCMVN (cmvn.py:21-32) + Conv2d(1,C,3,2) + ReLU (subsampling.py:28-29), output channels-last [B, T1, F1, C].
// One block per (b, t1); feat: fp32 [B, T, F].
__global__ void __launch_bounds__(256)
whale_conv1_kernel(const float* __restrict__ feat, const float* __restrict__ mean, const float* __restrict__ istd,
                   const __nv_bfloat16* __restrict__ w, const __nv_bfloat16* __restrict__ bias,
                   __nv_bfloat16* __restrict__ out, int T, int F, int T1, int F1, int C) {
    extern __shared__ float s_in[];  // [3][F] normalised input rows, rounded to bf16 like the reference's cast
    const int t1 = blockIdx.x % T1;
    const long long b = blockIdx.x / T1;
    for (int i = threadIdx.x; i < 3 * F; i += blockDim.x) {
        const int kt = i / F, f = i % F;
        float v = feat[(b * T + (2 * t1 + kt)) * F + f];
        if (mean) v = (v - mean[f]) * istd[f];
        s_in[i] = __bfloat162float(__float2bfloat16(v));
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float wv[9];
#pragma unroll
        for (int k = 0; k < 9; ++k) wv[k] = __bfloat162float(w[c * 9 + k]);
        const float bv = __bfloat162float(bias[c]);
        for (int f1 = 0; f1 < F1; ++f1) {
            float acc = bv;
#pragma unroll
            for (int kt = 0; kt < 3; ++kt)
#pragma unroll
                for (int kf = 0; kf < 3; ++kf) acc += wv[kt * 3 + kf] * s_in[kt * F + 2 * f1 + kf];
            out[((b * T1 + t1) * F1 + f1) * C + c] = __float2bfloat16(fmaxf(acc, 0.0f));
        }
    }
}

// im2col for Conv2d(C,C,3,2) on a channels-last map (subsampling.py:30): row = (b, t2, f2), column = (kt*3+kf)*C + c.
__global__ void __launch_bounds__(256)
whale_im2col2_kernel(const __nv_bfloat16* __restrict__ in, __nv_bfloat16* __restrict__ out, int T1, int F1, int T2,
                     int F2, int C) {
    const int f2 = blockIdx.x % F2;
    const int t2 = (blockIdx.x / F2) % T2;
    const long long b = blockIdx.x / (F2 * T2);
    const int cvec = C >> 3;
    uint4* dst = reinterpret_cast<uint4*>(out + static_cast<long long>(blockIdx.x) * 9 * C);
    for (int i = threadIdx.x; i < 9 * cvec; i += blockDim.x) {
        const int k = i / cvec, ci = i % cvec;
        const int kt = k / 3, kf = k % 3;
        dst[i] = reinterpret_cast<const uint4*>(in + ((b * T1 + 2 * t2 + kt) * F1 + 2 * f2 + kf) * C)[ci];
    }
}

// Rel-pos attention operands (attention.py:379-398): scores = (q+u).k^T + (q+v).p^T  ==  [q+u | q+v] . [k | p]^T.
// qkv [B*T, 3*Hd] (q | k | v), p [T, Hd]; outputs Q2, K2: [B*T, heads, 2*dk].
__global__ void __launch_bounds__(256)
whale_qk_prep_kernel(const __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ p,
                     const __nv_bfloat16* __restrict__ bias_u, const __nv_bfloat16* __restrict__ bias_v,
                     __nv_bfloat16* __restrict__ q2, __nv_bfloat16* __restrict__ k2, int T, int heads, int dk) {
    const long long row = blockIdx.x;  // b*T + t
    const int t = static_cast<int>(row % T);
    const int Hd = heads * dk;
    const __nv_bfloat16* q = qkv + row * 3 * Hd;
    const __nv_bfloat16* k = q + Hd;
    const __nv_bfloat16* pr = p + static_cast<long long>(t) * Hd;
    for (int i = threadIdx.x; i < Hd; i += blockDim.x) {
        const int hd = i / dk, d = i % dk;
        const float qv = __bfloat162float(q[i]);
        const long long o = (row * heads + hd) * 2 * dk;
        q2[o + d] = __float2bfloat16(qv + __bfloat162float(bias_u[i]));
        q2[o + dk + d] = __float2bfloat16(qv + __bfloat162float(bias_v[i]));
        k2[o + d] = k[i];
        k2[o + dk + d] = pr[i];
    }
}

// Adapter front (adapter.py:112-121): zero padded frames, right-pad k-1 zeros, im2col for Conv1d(C, 2C, k, stride 2).
// x [B, T, C]; out row = (b, t3), column = kk*C + c.
__global__ void __launch_bounds__(256)
whale_adapter_im2col_kernel(const __nv_bfloat16* __restrict__ x, const int* __restrict__ lengths,
                            __nv_bfloat16* __restrict__ out, int T, int T3, int C, int ksize) {
    const int t3 = blockIdx.x % T3;
    const long long b = blockIdx.x / T3;
    const int len = lengths ? lengths[b] : T;
    const int cvec = C >> 3;
    uint4* dst = reinterpret_cast<uint4*>(out + static_cast<long long>(blockIdx.x) * ksize * C);
    for (int i = threadIdx.x; i < ksize * cvec; i += blockDim.x) {
        const int kk = i / cvec, ci = i % cvec;
        const int t = 2 * t3 + kk;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (t < T && t < len) v = reinterpret_cast<const uint4*>(x + (b * T + t) * C)[ci];
        dst[i] = v;
    }
}

template <typename F>
static int launch_rows(F f) { f(); return check_launch("row kernel"); }

}  // namespace vita

using namespace vita;

#define BF(p) static_cast<const __nv_bfloat16*>(p)
#define BFM(p) static_cast<__nv_bfloat16*>(p)

extern "C" int vita_rmsnorm(const void* x, const void* w, void* y, int64_t rows, int64_t H, float eps, void* stream) {
    VITA_REQUIRE(H % 8 == 0 && H <= 8 * 8 * 256, "H must be a multiple of 8 and <= 16384");
    if (rows == 0) return VITA_OK;
    auto st = static_cast<cudaStream_t>(stream);
    if (H <= 8 * 2 * 256)
        rmsnorm_kernel<256, 2><<<static_cast<unsigned>(rows), 256, 0, st>>>(BF(x), BF(w), BFM(y), (int)H, eps);
    else
        rmsnorm_kernel<256, 8><<<static_cast<unsigned>(rows), 256, 0, st>>>(BF(x), BF(w), BFM(y), (int)H, eps);
    return check_launch("rmsnorm");
}

extern "C" int vita_layernorm(const void* x, const void* w, const void* b, void* y, int64_t rows, int64_t H, float eps,
                              int act, float out_scale, void* stream) {
    VITA_REQUIRE(H % 8 == 0 && H <= 8 * 4 * 256, "H must be a multiple of 8 and <= 8192");
    if (rows == 0) return VITA_OK;
    auto st = static_cast<cudaStream_t>(stream);
    if (H <= 8 * 128)
        layernorm_kernel<128, 1><<<static_cast<unsigned>(rows), 128, 0, st>>>(BF(x), BF(w), BF(b), BFM(y), (int)H, eps,
                                                                              act, out_scale);
    else
        layernorm_kernel<256, 4><<<static_cast<unsigned>(rows), 256, 0, st>>>(BF(x), BF(w), BF(b), BFM(y), (int)H, eps,
                                                                              act, out_scale);
    return check_launch("layernorm");
}

extern "C" int vita_row_copy(const void* table, const int32_t* src_index, const int32_t* dst_index, void* out,
                             int64_t n_rows, int64_t H, void* stream) {
    VITA_REQUIRE(H % 8 == 0, "H must be a multiple of 8");
    if (n_rows == 0) return VITA_OK;
    const unsigned grid = static_cast<unsigned>(n_rows < 65535 * 16 ? n_rows : 65535 * 16);
    row_copy_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(BF(table), src_index, dst_index, BFM(out),
                                                                          (int)n_rows, (int)H);
    return check_launch("row_copy");
}

extern "C" int vita_rope_kv_write(void* qkv, const int32_t* positions, const int32_t* slot_mapping,
                                  const float* cos_sin, void* k_cache, void* v_cache, int64_t n_tok, int64_t n_q_heads,
                                  int64_t n_kv_heads, int64_t head_dim, void* stream) {
    VITA_REQUIRE(head_dim == 128, "head_dim must be 128");
    if (n_tok == 0) return VITA_OK;
    rope_kv_write_kernel<128><<<static_cast<unsigned>(n_tok), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        BFM(qkv), positions, slot_mapping, cos_sin, BFM(k_cache), BFM(v_cache), (int)n_tok, (int)n_q_heads,
        (int)n_kv_heads);
    return check_launch("rope_kv_write");
}

extern "C" int vita_moe_router(const void* h, const void* norm_w, const void* gate_w, void* xn, int32_t* topk_ids,
                               float* topk_w, int64_t n_tok, int64_t H, int64_t E, float eps, void* stream) {
    VITA_REQUIRE(E == 8, "router is specialised for 8 experts (Mixtral-8x7B)");
    VITA_REQUIRE(H % 8 == 0 && H <= 4096, "H must be a multiple of 8 and <= 4096");
    if (n_tok == 0) return VITA_OK;
    const unsigned grid = static_cast<unsigned>(n_tok);
    rmsnorm_router_kernel<8><<<grid, 128, 0, static_cast<cudaStream_t>(stream)>>>(
        BF(h), BF(norm_w), BF(gate_w), BFM(xn), topk_ids, topk_w, (int)n_tok, (int)H, eps);
    return check_launch("moe_router");
}

extern "C" int vita_moe_route_scatter(const void* h, const void* norm_w, const void* gate_w, void* x_slots,
                                      int32_t* expert_counts, int32_t* perm_row, float* row_weight, int32_t* topk_ids,
                                      float* topk_w, int64_t n_tok, int64_t H, int64_t E, int64_t capacity, float eps,
                                      void* stream) {
    VITA_REQUIRE(E == 8, "router is specialised for 8 experts (Mixtral-8x7B)");
    VITA_REQUIRE(H % 8 == 0 && H <= 4096, "H must be a multiple of 8 and <= 4096");
    VITA_REQUIRE(capacity >= n_tok, "an expert can receive every token: capacity must be >= n_tok");
    VITA_REQUIRE((topk_ids == nullptr) == (topk_w == nullptr), "topk_ids and topk_w go together");
    if (n_tok == 0) return VITA_OK;
    rmsnorm_router_scatter_kernel<8><<<static_cast<unsigned>(n_tok), 128, 0, static_cast<cudaStream_t>(stream)>>>(
        BF(h), BF(norm_w), BF(gate_w), BFM(x_slots), expert_counts, perm_row, row_weight, topk_ids, topk_w, (int)n_tok,
        (int)H, (int)capacity, eps);
    return check_launch("moe_route_scatter");
}

extern "C" int vita_moe_align(const int32_t* topk_ids, const float* topk_w, int32_t* expert_offsets,
                              int32_t* perm_row, int32_t* row_token, float* row_weight, int32_t* row_assign,
                              int64_t n_tok, int64_t E, void* stream) {
    VITA_REQUIRE(E >= 1 && E <= 32, "E must be in [1, 32]");
    if (E <= 8)
        moe_align8_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(topk_ids, topk_w, expert_offsets, perm_row,
                                                                             row_token, row_weight, row_assign,
                                                                             (int)(n_tok * 2), (int)E);
    else
        moe_align_kernel<<<1, 1024, 0, static_cast<cudaStream_t>(stream)>>>(topk_ids, topk_w, expert_offsets, perm_row,
                                                                            row_token, row_weight, row_assign,
                                                                            (int)(n_tok * 2), (int)E);
    return check_launch("moe_align");
}

extern "C" int vita_moe_combine(void* h, const void* y_perm, const int32_t* perm_row, const void* next_norm_w,
                                void* xn_out, int64_t n_tok, int64_t H, float eps, void* stream) {
    VITA_REQUIRE(H % 8 == 0 && H <= 8 * 2 * 256, "H must be a multiple of 8 and <= 4096");
    if (n_tok == 0) return VITA_OK;
    moe_combine_kernel<256, 2><<<static_cast<unsigned>(n_tok), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        BFM(h), BF(y_perm), perm_row, BF(next_norm_w), BFM(xn_out), (int)H, eps);
    return check_launch("moe_combine");
}

extern "C" int vita_ep_signal(void* const* peer_flags, int64_t which, int64_t n_ranks, int64_t my_rank, int64_t epoch,
                              void* stream) {
    VITA_REQUIRE(n_ranks >= 1 && n_ranks <= 32, "n_ranks must be in [1, 32]");
    ep_signal_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<int* const*>(peer_flags), (int)which,
                                                                      (int)n_ranks, (int)my_rank, (int)epoch);
    return check_launch("ep_signal");
}

extern "C" int vita_ep_push(void* const* peer_base, const int64_t* offsets, const int64_t* bytes, int64_t n_ranges,
                            int64_t n_ranks, int64_t my_rank, void* stream) {
    VITA_REQUIRE(n_ranges >= 0 && n_ranges <= 4 && n_ranks >= 1 && n_ranks <= 32, "at most 4 ranges, 32 ranks");
    PushRanges r{};
    long long total = 0;
    for (int i = 0; i < n_ranges; ++i) {
        VITA_REQUIRE(offsets[i] % 16 == 0 && bytes[i] % 4 == 0 && bytes[i] >= 0,
                     "range offsets must be 16-byte aligned, sizes multiples of 4");
        r.off[i] = offsets[i];
        r.bytes[i] = bytes[i];
        total += bytes[i];
    }
    r.n = static_cast<int>(n_ranges);
    if (total == 0 || n_ranks == 1) return VITA_OK;
    long long blocks = (total / 16 + 255) / 256 + 1;
    const int cap = 2 * (num_sms() > 0 ? num_sms() : 132);
    if (blocks > cap) blocks = cap;
    ep_push_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        reinterpret_cast<uint8_t* const*>(peer_base), r, (int)n_ranks, (int)my_rank);
    return check_launch("ep_push");
}

extern "C" int vita_ep_wait(const int32_t* my_flags, int64_t which, int64_t n_ranks, int64_t n_wait, int64_t epoch,
                            void* stream) {
    VITA_REQUIRE(n_ranks >= 1 && n_ranks <= 32, "n_ranks must be in [1, 32]");
    VITA_REQUIRE(n_wait >= 0 && n_wait <= n_ranks, "n_wait must be in [0, n_ranks]");
    ep_wait_kernel<<<1, 32, 0, static_cast<cudaStream_t>(stream)>>>(my_flags, (int)which, (int)n_ranks, (int)n_wait,
                                                                    (int)epoch);
    return check_launch("ep_wait");
}

extern "C" int vita_ep_reduce_norm_gather(const void* rs_buf, const int32_t* my_flags, void* const* peer_h,
                                          void* const* peer_xn, const void* next_norm_w, int64_t tok0, int64_t n_owned,
                                          int64_t n_ranks, int64_t my_rank, int64_t epoch, int64_t H, float eps,
                                          int64_t gather, void* stream) {
    VITA_REQUIRE(H % 8 == 0 && H <= 8 * 2 * 256, "H must be a multiple of 8 and <= 4096");
    VITA_REQUIRE(n_ranks >= 1 && n_ranks <= 32, "n_ranks must be in [1, 32]");
    if (n_owned == 0) return VITA_OK;
    ep_reduce_norm_gather_kernel<256, 2><<<static_cast<unsigned>(n_owned), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        BF(rs_buf), my_flags, reinterpret_cast<__nv_bfloat16* const*>(peer_h),
        reinterpret_cast<__nv_bfloat16* const*>(peer_xn), BF(next_norm_w), (int)tok0, (int)n_ranks, (int)my_rank,
        (int)epoch, (int)H, eps, gather ? 1 : 0);
    return check_launch("ep_reduce_norm_gather");
}

extern "C" int vita_vit_im2col(const void* images, void* out, int64_t n_img, int64_t C, int64_t HW, int64_t P,
                               int64_t k_pad, void* stream) {
    VITA_REQUIRE(HW % P == 0 && k_pad >= C * P * P && k_pad % 8 == 0, "bad patch geometry");
    const long long n = n_img * (HW / P) * (HW / P);
    if (n == 0) return VITA_OK;
    vit_im2col_kernel<<<static_cast<unsigned>(n), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        BF(images), BFM(out), (int)n_img, (int)C, (int)HW, (int)P, (int)k_pad);
    return check_launch("vit_im2col");
}

extern "C" int vita_vit_assemble(const void* patches, const void* cls, const void* pos, void* out, int64_t n_img,
                                 int64_t n_patch, int64_t H, void* stream) {
    VITA_REQUIRE(H % 8 == 0, "H must be a multiple of 8");
    if (n_img == 0) return VITA_OK;
    vit_assemble_kernel<<<static_cast<unsigned>(n_img * (n_patch + 1)), 128, 0, static_cast<cudaStream_t>(stream)>>>(
        BF(patches), BF(cls), BF(pos), BFM(out), (int)n_patch, (int)H);
    return check_launch("vit_assemble");
}

extern "C" int vita_vit_pixel_shuffle(const void* h, void* out, int64_t n_img, int64_t grid, int64_t C, float scale,
                                      void* stream) {
    VITA_REQUIRE(grid % 2 == 0 && C % 8 == 0, "grid must be even and C a multiple of 8");
    if (n_img == 0) return VITA_OK;
    const long long n = n_img * (grid / 2) * (grid / 2);
    vit_pixel_shuffle_kernel<<<static_cast<unsigned>(n), 128, 0, static_cast<cudaStream_t>(stream)>>>(
        BF(h), BFM(out), (int)grid, (int)C, scale);
    return check_launch("vit_pixel_shuffle");
}

extern "C" int vita_whale_conv1(const float* feat, const float* mean, const float* istd, const void* w,
                                const void* bias, void* out, int64_t B, int64_t T, int64_t F, int64_t C,
                                void* stream) {
    const int T1 = (int)((T - 1) / 2), F1 = (int)((F - 1) / 2);
    VITA_REQUIRE(T >= 3 && F >= 3, "input too short for a 3x3 stride-2 convolution");
    if (B == 0) return VITA_OK;
    whale_conv1_kernel<<<static_cast<unsigned>(B * T1), 256, 3 * F * sizeof(float),
                         static_cast<cudaStream_t>(stream)>>>(feat, mean, istd, BF(w), BF(bias), BFM(out), (int)T,
                                                              (int)F, T1, F1, (int)C);
    return check_launch("whale_conv1");
}

extern "C" int vita_whale_im2col2(const void* in, void* out, int64_t B, int64_t T1, int64_t F1, int64_t C,
                                  void* stream) {
    const int T2 = (int)((T1 - 1) / 2), F2 = (int)((F1 - 1) / 2);
    VITA_REQUIRE(T1 >= 3 && F1 >= 3 && C % 8 == 0, "bad conv2 geometry");
    if (B == 0) return VITA_OK;
    whale_im2col2_kernel<<<static_cast<unsigned>(B * T2 * F2), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        BF(in), BFM(out), (int)T1, (int)F1, T2, F2, (int)C);
    return check_launch("whale_im2col2");
}

extern "C" int vita_whale_qk_prep(const void* qkv, const void* p, const void* bias_u, const void* bias_v, void* q2,
                                  void* k2, int64_t B, int64_t T, int64_t heads, int64_t dk, void* stream) {
    if (B * T == 0) return VITA_OK;
    whale_qk_prep_kernel<<<static_cast<unsigned>(B * T), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        BF(qkv), BF(p), BF(bias_u), BF(bias_v), BFM(q2), BFM(k2), (int)T, (int)heads, (int)dk);
    return check_launch("whale_qk_prep");
}

extern "C" int vita_whale_adapter_im2col(const void* x, const int32_t* lengths, void* out, int64_t B, int64_t T,
                                         int64_t C, int64_t ksize, void* stream) {
    VITA_REQUIRE(C % 8 == 0, "C must be a multiple of 8");
    const int T3 = (int)((T - 1) / 2 + 1);
    if (B == 0 || T == 0) return VITA_OK;
    whale_adapter_im2col_kernel<<<static_cast<unsigned>(B * T3), 256, 0, static_cast<cudaStream_t>(stream)>>>(
        BF(x), lengths, BFM(out), (int)T, T3, (int)C, (int)ksize);
    return check_launch("whale_adapter_im2col");
}
