// Paged decode attention (the prefill-shaped FlashAttention lives in flash_tc.cu).
//
// decode_attn_kernel: single-query paged-KV attention for greedy decode.  One CTA per (kv head, context split);
//     the 4 query heads of a GQA group share every K/V load; 8-lane groups own one key each and reduce with warp
//     shuffles.  Under programmatic dependent launch the cached K/V rows are fetched ahead of the dependency wait
//     (only q and the newest row come from the QKV kernel).  Splits are merged all-to-all through tagged 64-bit
//     words, each CTA owning a slice of the outputs (TAGGED = true; latency chain of one publish + one poll), or by
//     the last CTA to take a ticket (TAGGED = false: odd split counts, grids too large to be resident at once).
//
// Reference call sites: flash_attn_varlen_qkvpacked_func (internvit/flash_attention.py:61) / naive softmax
// (modeling_intern_vit.py:170-174); whale attention.py:391-415; transformers sdpa/eager attention
// (modeling_mixtral.py:269-292); vLLM paged Attention (web_demo/vllm_tools/vllm_file/mixtral.py:484-501).
#include "common.h"
#include "ptx.cuh"
#include "kv_fp8.cuh"

#include <type_traits>

namespace vita {

// ------------------------------------------------------------------------------------------------ paged decode
constexpr int DEC_D = 128;     // head dim
constexpr int DEC_GROUP = 4;   // query heads per kv head (32 / 8)

struct DecodeAttnParams {
    const __nv_bfloat16* q;        // row b at q + b * q_stride: [n_q, D]
    long long q_stride;
    const __nv_bfloat16* k_cache;  // [slots, n_kv, D]
    const __nv_bfloat16* v_cache;
    const int* block_table;        // [B, max_pages]
    const int* cur_pos;            // [B] position of the current token; context = cur_pos + 1
    __nv_bfloat16* out;            // [B, n_q * D]
    float* part_o;                 // [B, n_kv, splits, GROUP, D]
    float* part_ml;                // [B, n_kv, splits, GROUP, 2]
    int* tickets;                  // [B, n_kv], zero-initialised, self-resetting
    int n_q, n_kv, page_size, max_pages, splits;
    float scale_log2;
    int early;                     // fetch cached K/V rows before the dependency wait
};
// e4m3 cache (kv_fp8.cuh): k_cache / v_cache hold 1-byte elements, read as bf16(float(c) * scale)
struct DecodeAttnParamsFp8 : DecodeAttnParams {
    float k_scale, v_scale;
};
template <bool KV8>
using DecodeAttnArgs = std::conditional_t<KV8, DecodeAttnParamsFp8, DecodeAttnParams>;

// ordered 16-byte load: volatile asm keeps it on its side of the dependency wait
__device__ __forceinline__ uint4 ld_early_v4(const void* ptr) {
    uint4 r;
    asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(ptr));
    return r;
}

__device__ __forceinline__ unsigned long long attn_ld_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void attn_st_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// waits for a tagged word {value, tag != 0}, returns the value and frees the slot
__device__ __forceinline__ float attn_take(unsigned long long* addr, unsigned long long w) {
    for (uint32_t spin = 0; (w >> 32) == 0; ++spin) {
        if (spin > (1u << 22)) __trap();   // a split never published
        w = attn_ld_u64(addr);
    }
    attn_st_u64(addr, 0ull);
    return __uint_as_float(static_cast<uint32_t>(w));
}
__device__ __forceinline__ float attn_rescale(float m_old, float m_new) {
    return m_old == -INFINITY ? 0.0f : exp2f(m_old - m_new);
}

// TAGGED = false: splits are combined by the last CTA to take a ticket (fence + atomic + reload).
// KV8 = true    : the cache rows are e4m3 (16 bytes for the 16 dims of a lane where bf16 takes two 16-byte loads), each
//                 element dequantized to its bf16 value before use: the same element-to-thread mapping and reduction
//                 order, so the output bits are those of KV8 = false on the dequantized cache.
// TAGGED = true : partials travel as 64-bit {value, tag} words in an all-to-all over the splits of a kv head: each CTA
//                 owns a slice of the outputs and collects the other splits' words for it (no fence, no atomic, no
//                 serial collector); lane groups are pre-merged with shuffles.
template <bool TAGGED, bool KV8>
__global__ void __launch_bounds__(128)
decode_attn_kernel(const DecodeAttnArgs<KV8> p, const ChainArgsDev chain VITA_TRACE_PARAM) {
    __shared__ float s_m[16][DEC_GROUP];
    __shared__ float s_l[16][DEC_GROUP];
    __shared__ __align__(16) float s_o[TAGGED ? 4 : 16][DEC_GROUP][DEC_D];
    __shared__ float s_ml[16][DEC_GROUP][2];
    __shared__ int s_last;

    const int split = blockIdx.x, kvh = blockIdx.y, b = blockIdx.z;
#ifdef VITA_TRACE
    if (kvh != 0 || b != 0) trace = nullptr;
    if (threadIdx.x == 0 && split == 0) { VITA_STAMP(1); VITA_STAMP_SET(0, 2ull); }
#endif
    pdl_launch_dependents();
    if (!p.early) {
        if (threadIdx.x == 0) chain_wait(chain);
        __syncthreads();
    }
    // ---- before the dependency wait -------------------------------------------------------------------------------
    // cur_pos (first kernel of the step), the block table and every cached K/V row except the newest one are NOT
    // written by the kernel right before this one (the QKV projection of this layer), and the kernel before that has
    // completed by the time this grid could be launched (each chain kernel waits before it triggers).  So with
    // programmatic dependent launch the old keys are already in registers when the QKV kernel retires.
    const int ctx = p.cur_pos[b] + 1;
    const int newest = ctx - 1;
    const int per = (ctx + p.splits - 1) / p.splits;
    const int k_begin = split * per;
    const int k_end = min(ctx, k_begin + per);

    const int lg = threadIdx.x >> 3;  // lane group 0..15: one key at a time
    const int sl = threadIdx.x & 7;   // 16 dims per lane
    const int d0 = sl * 16;
    const int* bt = p.block_table + static_cast<long long>(b) * p.max_pages;

    constexpr int NPRE = 4;           // keys per lane group fetched up front (covers ctx <= splits * 64)
    uint4 pk[NPRE][2], pv[NPRE][2];
    long long pslot[NPRE];
#pragma unroll
    for (int j = 0; j < NPRE; ++j) {
        const int key = k_begin + j * 16 + lg;
        pslot[j] = -1;
        if (key < k_end) {
            const int page = bt[key / p.page_size];
            pslot[j] = static_cast<long long>(page) * p.page_size + key % p.page_size;
        }
    }
#pragma unroll
    for (int j = 0; j < NPRE; ++j) {
        const int key = k_begin + j * 16 + lg;
        if (pslot[j] >= 0 && key != newest) {
            if constexpr (KV8) {
                const long long off = (pslot[j] * p.n_kv + kvh) * DEC_D + d0;
                pk[j][0] = ld_early_v4(reinterpret_cast<const uint8_t*>(p.k_cache) + off); pk[j][1] = make_uint4(0, 0, 0, 0);
                pv[j][0] = ld_early_v4(reinterpret_cast<const uint8_t*>(p.v_cache) + off); pv[j][1] = make_uint4(0, 0, 0, 0);
            } else {
            const __nv_bfloat16* kp = p.k_cache + (pslot[j] * p.n_kv + kvh) * DEC_D + d0;
            const __nv_bfloat16* vp = p.v_cache + (pslot[j] * p.n_kv + kvh) * DEC_D + d0;
            pk[j][0] = ld_early_v4(kp); pk[j][1] = ld_early_v4(kp + 8);
            pv[j][0] = ld_early_v4(vp); pv[j][1] = ld_early_v4(vp + 8);
            }
        } else {
            pk[j][0] = pk[j][1] = pv[j][0] = pv[j][1] = make_uint4(0, 0, 0, 0);
        }
    }
    if (threadIdx.x == 0) chain_wait(chain);   // q and the newest K/V row come from the QKV kernel
    __syncthreads();
    if (threadIdx.x == 0 && split == 0) VITA_STAMP(3);
#pragma unroll
    for (int j = 0; j < NPRE; ++j) {
        const int key = k_begin + j * 16 + lg;
        if (pslot[j] >= 0 && key == newest) {
            if constexpr (KV8) {
                const long long off = (pslot[j] * p.n_kv + kvh) * DEC_D + d0;
                pk[j][0] = ld_early_v4(reinterpret_cast<const uint8_t*>(p.k_cache) + off);
                pv[j][0] = ld_early_v4(reinterpret_cast<const uint8_t*>(p.v_cache) + off);
            } else {
            const __nv_bfloat16* kp = p.k_cache + (pslot[j] * p.n_kv + kvh) * DEC_D + d0;
            const __nv_bfloat16* vp = p.v_cache + (pslot[j] * p.n_kv + kvh) * DEC_D + d0;
            pk[j][0] = ld_early_v4(kp); pk[j][1] = ld_early_v4(kp + 8);
            pv[j][0] = ld_early_v4(vp); pv[j][1] = ld_early_v4(vp + 8);
            }
        }
    }

    float q[DEC_GROUP][16];
#pragma unroll
    for (int h = 0; h < DEC_GROUP; ++h) {
        const uint4* qp = reinterpret_cast<const uint4*>(p.q + static_cast<long long>(b) * p.q_stride + (kvh * DEC_GROUP + h) * DEC_D + d0);
        const uint4 a = qp[0], c = qp[1];
        const uint32_t w[8] = {a.x, a.y, a.z, a.w, c.x, c.y, c.z, c.w};
#pragma unroll
        for (int i = 0; i < 8; ++i) { q[h][2 * i] = bf16_lo(w[i]); q[h][2 * i + 1] = bf16_hi(w[i]); }
    }
    float m[DEC_GROUP], l[DEC_GROUP], acc[DEC_GROUP][16];
#pragma unroll
    for (int h = 0; h < DEC_GROUP; ++h) {
        m[h] = -INFINITY;
        l[h] = 0.0f;
#pragma unroll
        for (int i = 0; i < 16; ++i) acc[h][i] = 0.0f;
    }
    // one key per lane group: scores for the 4 query heads of this kv head, online softmax, P.V
    auto consume = [&](const uint4& ka, const uint4& kc, const uint4& va, const uint4& vc, bool valid) {
        const uint32_t kw[8] = {ka.x, ka.y, ka.z, ka.w, kc.x, kc.y, kc.z, kc.w};
        const uint32_t vw[8] = {va.x, va.y, va.z, va.w, vc.x, vc.y, vc.z, vc.w};
        float kf[16], vf[16];
        if constexpr (KV8) {   // ka / va: 16 e4m3 bytes, byte i = dim d0 + i
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                kv_fp8_dequant4(kw[i], p.k_scale, kf + 4 * i);
                kv_fp8_dequant4(vw[i], p.v_scale, vf + 4 * i);
            }
        } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            kf[2 * i] = bf16_lo(kw[i]); kf[2 * i + 1] = bf16_hi(kw[i]);
            vf[2 * i] = bf16_lo(vw[i]); vf[2 * i + 1] = bf16_hi(vw[i]);
        }
        }
#pragma unroll
        for (int h = 0; h < DEC_GROUP; ++h) {
            float dot = 0.0f;
#pragma unroll
            for (int i = 0; i < 16; ++i) dot += q[h][i] * kf[i];
            dot += __shfl_xor_sync(0xffffffffu, dot, 1);
            dot += __shfl_xor_sync(0xffffffffu, dot, 2);
            dot += __shfl_xor_sync(0xffffffffu, dot, 4);
            if (valid) {
                const float sc = dot * p.scale_log2;
                const float m_new = fmaxf(m[h], sc);
                const float alpha = exp2f(m[h] - m_new);
                const float pr = exp2f(sc - m_new);
                m[h] = m_new;
                l[h] = l[h] * alpha + pr;
#pragma unroll
                for (int i = 0; i < 16; ++i) acc[h][i] = acc[h][i] * alpha + pr * vf[i];
            }
        }
    };
    const int n_keys = max(k_end - k_begin, 0);
#pragma unroll
    for (int j = 0; j < NPRE; ++j) {
        if (j * 16 < n_keys)   // uniform across the CTA (shuffles inside)
            consume(pk[j][0], pk[j][1], pv[j][0], pv[j][1], pslot[j] >= 0);
    }
    // longer contexts: software pipeline, the K/V rows of the next key are in flight while the current one is reduced
    if (n_keys > NPRE * 16) {
        uint4 nk0, nk1, nv0, nv1;
        auto issue = [&](int key) {
            if constexpr (KV8) {
                nk1 = nv1 = make_uint4(0, 0, 0, 0);
                if (key < k_end) {
                    const int page = bt[key / p.page_size];
                    const long long slot = static_cast<long long>(page) * p.page_size + key % p.page_size;
                    const long long off = (slot * p.n_kv + kvh) * DEC_D + d0;
                    nk0 = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.k_cache) + off);
                    nv0 = *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(p.v_cache) + off);
                } else {
                    nk0 = nv0 = make_uint4(0, 0, 0, 0);
                }
                return;
            }
            if (key < k_end) {
                const int page = bt[key / p.page_size];
                const long long slot = static_cast<long long>(page) * p.page_size + key % p.page_size;
                const uint4* kp = reinterpret_cast<const uint4*>(p.k_cache + (slot * p.n_kv + kvh) * DEC_D + d0);
                const uint4* vp = reinterpret_cast<const uint4*>(p.v_cache + (slot * p.n_kv + kvh) * DEC_D + d0);
                nk0 = kp[0]; nk1 = kp[1]; nv0 = vp[0]; nv1 = vp[1];
            } else {
                nk0 = nk1 = nv0 = nv1 = make_uint4(0, 0, 0, 0);
            }
        };
        issue(k_begin + NPRE * 16 + lg);
        for (int key0 = k_begin + NPRE * 16; key0 < k_end; key0 += 16) {  // trip count is uniform across the warp
            const int key = key0 + lg;
            const uint4 ka = nk0, kc = nk1, va = nv0, vc = nv1;
            issue(key + 16);
            consume(ka, kc, va, vc, key < k_end);
        }
    }
    if constexpr (TAGGED) {
        // ---- the 4 lane groups of each warp first (shuffles), then the 4 warps through shared memory
#pragma unroll
        for (int off = 8; off <= 16; off <<= 1) {
#pragma unroll
            for (int h = 0; h < DEC_GROUP; ++h) {
                const float mo = __shfl_xor_sync(0xffffffffu, m[h], off);
                const float lo = __shfl_xor_sync(0xffffffffu, l[h], off);
                const float mn = fmaxf(m[h], mo);
                const float wa = attn_rescale(m[h], mn), wb = attn_rescale(mo, mn);
                l[h] = l[h] * wa + lo * wb;
#pragma unroll
                for (int i = 0; i < 16; ++i)
                    acc[h][i] = acc[h][i] * wa + __shfl_xor_sync(0xffffffffu, acc[h][i], off) * wb;
                m[h] = mn;
            }
        }
        const int wid = threadIdx.x >> 5;
        if ((threadIdx.x & 31) < 8) {
#pragma unroll
            for (int h = 0; h < DEC_GROUP; ++h) {
                if (sl == 0) { s_m[wid][h] = m[h]; s_l[wid][h] = l[h]; }
#pragma unroll
                for (int i = 0; i < 16; i += 4)
                    *reinterpret_cast<float4*>(&s_o[wid][h][d0 + i]) = make_float4(acc[h][i], acc[h][i + 1], acc[h][i + 2], acc[h][i + 3]);
            }
        }
        __syncthreads();
        const int d = threadIdx.x;  // one output dim per thread
        float mm[DEC_GROUP], ll[DEC_GROUP], oo[DEC_GROUP];
#pragma unroll
        for (int h = 0; h < DEC_GROUP; ++h) {
            mm[h] = fmaxf(fmaxf(s_m[0][h], s_m[1][h]), fmaxf(s_m[2][h], s_m[3][h]));
            ll[h] = 0.0f; oo[h] = 0.0f;
#pragma unroll
            for (int w = 0; w < 4; ++w) {
                const float sc = attn_rescale(s_m[w][h], mm[h]);
                ll[h] += sc * s_l[w][h];
                oo[h] += sc * s_o[w][h][d];
            }
        }
        __syncthreads();   // every thread is done reading s_m / s_l / s_o
        // ---- all-to-all over the splits of this kv head: every CTA publishes its partials as tagged words and owns
        // a 1/splits slice of the 4 x 128 outputs, for which it collects the other splits' words (one round trip,
        // no fence, no ticket, no serial collector).  Each word has exactly one reader, which clears the tag.
        const int S = p.splits;                    // 4, 8 or 16 (checked on the host)
        const int P = DEC_GROUP * DEC_D / S;       // outputs owned by this CTA
        unsigned long long* words = reinterpret_cast<unsigned long long*>(p.part_o);
        const long long n_words_o = static_cast<long long>(gridDim.z) * p.n_kv * S * DEC_GROUP * DEC_D;
        const long long grp = static_cast<long long>(b) * p.n_kv + kvh;
        unsigned long long* o_w = words + grp * S * DEC_GROUP * DEC_D;                    // [publisher][head][dim]
        unsigned long long* ml_w = words + n_words_o + grp * S * S * DEC_GROUP * 2;      // [publisher][reader][head][2]
#ifdef VITA_TRACE
        if (threadIdx.x == 0 && trace) trace[9 + (split & 15)] = global_timer_ns();
#endif
        // publish
#pragma unroll
        for (int h = 0; h < DEC_GROUP; ++h) {
            s_o[0][h][d] = oo[h];   // own slice is read back from shared memory (s_o[0] is free again: all reads done)
            if ((h * DEC_D + d) / P != split)
                attn_st_u64(o_w + (split * DEC_GROUP + h) * DEC_D + d,
                            (1ull << 32) | static_cast<unsigned long long>(__float_as_uint(oo[h])));
        }
        const int t = threadIdx.x;
        const bool ml_thread = t < S * DEC_GROUP * 2;
        const int peer = t >> 3, mh = (t & 7) >> 1, which = t & 1;
        if (ml_thread) {
            float val = 0.0f;
#pragma unroll
            for (int h = 0; h < DEC_GROUP; ++h)
                if (h == mh) val = which ? ll[h] : mm[h];
            if (peer == split) s_ml[split][mh][which] = val;
            else attn_st_u64(ml_w + ((split * S + peer) * DEC_GROUP + mh) * 2 + which,
                             (1ull << 32) | static_cast<unsigned long long>(__float_as_uint(val)));
        }
        // collect: all loads first, then poll what has not arrived yet
        constexpr int MAXS = 16;
        unsigned long long* ml_addr = ml_w + ((peer * S + split) * DEC_GROUP + mh) * 2 + which;
        unsigned long long ml_word = 0;
        if (ml_thread && peer != split) ml_word = attn_ld_u64(ml_addr);
        const int flat = split * P + t;            // output handled by thread t < P
        const int oh = flat / DEC_D, od = flat % DEC_D;
        unsigned long long w[MAXS];
        float os[MAXS];
        if (t < P) {
#pragma unroll
            for (int sp = 0; sp < MAXS; ++sp)
                if (sp < S && sp != split) w[sp] = attn_ld_u64(o_w + (sp * DEC_GROUP + oh) * DEC_D + od);
        }
        if (ml_thread && peer != split) s_ml[peer][mh][which] = attn_take(ml_addr, ml_word);
        if (t < P) {
#pragma unroll
            for (int sp = 0; sp < MAXS; ++sp)
                os[sp] = (sp < S && sp != split) ? attn_take(o_w + (sp * DEC_GROUP + oh) * DEC_D + od, w[sp]) : 0.0f;
        }
        __syncthreads();
        if (threadIdx.x == 0) VITA_STAMP(27);
        if (t < P) {
            float mt = -INFINITY;
#pragma unroll
            for (int sp = 0; sp < MAXS; ++sp)
                if (sp < S) mt = fmaxf(mt, s_ml[sp][oh][0]);
            float lt = 0.0f, ot = 0.0f;
#pragma unroll
            for (int sp = 0; sp < MAXS; ++sp) {
                if (sp < S) {
                    const float sc = attn_rescale(s_ml[sp][oh][0], mt);
                    lt += sc * s_ml[sp][oh][1];
                    ot += sc * (sp == split ? s_o[0][oh][od] : os[sp]);
                }
            }
            p.out[(static_cast<long long>(b) * p.n_q + kvh * DEC_GROUP + oh) * DEC_D + od] =
                __float2bfloat16(lt > 0.0f ? ot / lt : 0.0f);
        }
        __syncthreads();                                  // the CTA's output stores are issued
        if (threadIdx.x == 0) chain_arrive(chain);
        if (threadIdx.x == 0) VITA_STAMP(8);
        return;
    }
    // merge the 16 lane groups of this CTA
#pragma unroll
    for (int h = 0; h < DEC_GROUP; ++h) {
        if (sl == 0) { s_m[lg][h] = m[h]; s_l[lg][h] = l[h]; }
#pragma unroll
        for (int i = 0; i < 16; ++i) s_o[TAGGED ? 0 : lg][h][d0 + i] = acc[h][i];
    }
    __syncthreads();
    const int d = threadIdx.x;  // one output dim per thread
    const long long pbase = ((static_cast<long long>(b) * p.n_kv + kvh) * p.splits + split) * DEC_GROUP;
#pragma unroll
    for (int h = 0; h < DEC_GROUP; ++h) {
        float mm = -INFINITY;
#pragma unroll
        for (int gI = 0; gI < 16; ++gI) mm = fmaxf(mm, s_m[gI][h]);
        float ll = 0.0f, oo = 0.0f;
        if (mm > -INFINITY) {
#pragma unroll
            for (int gI = 0; gI < 16; ++gI) {
                const float w = exp2f(s_m[gI][h] - mm);
                ll += w * s_l[gI][h];
                oo += w * s_o[TAGGED ? 0 : gI][h][d];
            }
        }
        p.part_o[(pbase + h) * DEC_D + d] = oo;
        if (d == 0) { p.part_ml[(pbase + h) * 2] = mm; p.part_ml[(pbase + h) * 2 + 1] = ll; }
    }
#ifdef VITA_TRACE
    if (threadIdx.x == 0 && trace) trace[9 + (split & 15)] = global_timer_ns();
#endif
    // last CTA of this (batch, kv head) merges the splits
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const int t = atomicAdd(&p.tickets[b * p.n_kv + kvh], 1);
        s_last = (t == p.splits - 1);
        if (s_last) p.tickets[b * p.n_kv + kvh] = 0;
    }
    __syncthreads();
    if (!s_last) {
        if (threadIdx.x == 0) chain_arrive(chain);
        return;
    }
    if (threadIdx.x == 0) VITA_STAMP(25);
    __threadfence();
    const long long sbase = (static_cast<long long>(b) * p.n_kv + kvh) * p.splits * DEC_GROUP;
    constexpr int MAXS = 16;   // splits <= 16 (checked on the host); all loads of a head are issued before use
#pragma unroll
    for (int h = 0; h < DEC_GROUP; ++h) {
        float ms[MAXS], ls[MAXS], os[MAXS];
#pragma unroll
        for (int s = 0; s < MAXS; ++s) {
            if (s < p.splits) {
                ms[s] = __ldcg(&p.part_ml[(sbase + s * DEC_GROUP + h) * 2]);
                ls[s] = __ldcg(&p.part_ml[(sbase + s * DEC_GROUP + h) * 2 + 1]);
                os[s] = __ldcg(&p.part_o[(sbase + s * DEC_GROUP + h) * DEC_D + d]);
            } else {
                ms[s] = -INFINITY; ls[s] = 0.0f; os[s] = 0.0f;
            }
        }
        // consumed: hand the workspace back all-zero (the tagged variant shares it and reads a non-zero upper half
        // of an 8-byte word as "published"; each element below was read by this thread only)
#pragma unroll
        for (int s = 0; s < MAXS; ++s)
            if (s < p.splits) __stcg(&p.part_o[(sbase + s * DEC_GROUP + h) * DEC_D + d], 0.0f);
        float mm = -INFINITY;
#pragma unroll
        for (int s = 0; s < MAXS; ++s) mm = fmaxf(mm, ms[s]);
        float ll = 0.0f, oo = 0.0f;
#pragma unroll
        for (int s = 0; s < MAXS; ++s) {
            const float w = (ms[s] == -INFINITY) ? 0.0f : exp2f(ms[s] - mm);
            ll += w * ls[s];
            oo += w * os[s];
        }
        p.out[(static_cast<long long>(b) * p.n_q + kvh * DEC_GROUP + h) * DEC_D + d] =
            __float2bfloat16(ll > 0.0f ? oo / ll : 0.0f);
    }
    __syncthreads();   // every thread has read the (m, l) pairs
    if (d < p.splits * DEC_GROUP * 2) __stcg(&p.part_ml[sbase * 2 + d], 0.0f);
    __syncthreads();
    if (threadIdx.x == 0) chain_arrive(chain);
    if (threadIdx.x == 0) VITA_STAMP(8);
}

}  // namespace vita

using namespace vita;

// The merge a launch of (B, n_kv_heads, splits) takes.  The all-to-all protocol needs the split count to divide the
// 4 x 128 outputs into <= 128-wide slices ... and every CTA of a kv head polls its peers, so all of them have to be
// resident at once: keep that to grids that fit the machine (two 128-thread CTAs per SM), larger batches take the ticket
// variant (real occupancy of the tagged variant, not an estimate: every CTA of the grid polls its peers).
static bool decode_attn_tagged(int64_t B, int64_t n_kv_heads, int64_t splits) {
    static int resident_per_sm = -1;
    if (resident_per_sm < 0) {
        int n = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, decode_attn_kernel<true, false>, 128, 0) != cudaSuccess || n < 1) {
            (void)cudaGetLastError();
            n = 1;
        }
        resident_per_sm = n > 2 ? 2 : n;   // a chain neighbour may share the SM under programmatic launch
    }
    return option("attn_tagged") && (splits == 4 || splits == 8 || splits == 16) &&
           splits * n_kv_heads * B <= static_cast<long long>(resident_per_sm) * (num_sms() > 0 ? num_sms() : 132);
}

extern "C" int64_t vita_decode_attention_workspace_bytes(int64_t B, int64_t n_kv_heads, int64_t splits) {
    // 8-byte words {value, tag} for the split partials; the ticket variant uses the front of the same buffer as plain
    // floats.  Invariant kept by both variants: the workspace is all-zero between launches (tags cleared by their
    // readers, floats zeroed by the merging CTA, tickets reset), so calls may change B / splits / variant freely.
    const int64_t n = B * n_kv_heads * splits * DEC_GROUP;
    return n * DEC_D * 8 + B * n_kv_heads * splits * splits * DEC_GROUP * 2 * 8 + ((B * n_kv_heads * 4 + 255) / 256) * 256 + 256;
}

extern "C" int vita_decode_attention_merge(int64_t B, int64_t n_kv_heads, int64_t splits) {
    return decode_attn_tagged(B, n_kv_heads, splits) ? 1 : 0;
}

template <bool KV8>
static int decode_attention_launch(DecodeAttnArgs<KV8>& p, const void* q, const void* k_cache, const void* v_cache,
                                   const int32_t* block_table, const int32_t* cur_pos, void* out, void* workspace,
                                   int64_t B, int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim,
                                   int64_t page_size, int64_t max_pages, int64_t splits, float scale, int64_t q_stride,
                                   void* stream) {
    VITA_REQUIRE(head_dim == DEC_D && n_q_heads == n_kv_heads * DEC_GROUP, "decode attention: need D=128, GQA group 4");
    VITA_REQUIRE(splits >= 1 && splits <= 16 && workspace != nullptr, "1 <= splits <= 16 and a workspace are required");
    if (B == 0) return VITA_OK;
    p.q = BF16C(q); p.q_stride = q_stride > 0 ? q_stride : n_q_heads * head_dim;
    p.k_cache = BF16C(k_cache); p.v_cache = BF16C(v_cache);   // e4m3 bytes when KV8 (addressed per byte)
    p.block_table = block_table; p.cur_pos = cur_pos; p.out = static_cast<__nv_bfloat16*>(out);
    const int64_t n = B * n_kv_heads * splits * DEC_GROUP;
    // tickets first (must be zero-initialised once by the caller; the kernel resets them)
    p.tickets = static_cast<int*>(workspace);
    char* w = static_cast<char*>(workspace) + ((B * n_kv_heads * 4 + 255) / 256) * 256;
    p.part_o = reinterpret_cast<float*>(w);
    p.part_ml = reinterpret_cast<float*>(w + n * DEC_D * 4);
    p.n_q = (int)n_q_heads; p.n_kv = (int)n_kv_heads; p.page_size = (int)page_size; p.max_pages = (int)max_pages;
    p.splits = (int)splits;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.early = option("attn_early");
    dim3 grid((unsigned)splits, (unsigned)n_kv_heads, (unsigned)B);
    const bool tagged = decode_attn_tagged(B, n_kv_heads, splits);
    {
        static int carveout = -1;
        const int want = option("smem_carveout_max") ? cudaSharedmemCarveoutMaxShared : cudaSharedmemCarveoutDefault;
        if (carveout != want) {
            (void)cudaFuncSetAttribute(decode_attn_kernel<true, KV8>, cudaFuncAttributePreferredSharedMemoryCarveout, want);
            (void)cudaFuncSetAttribute(decode_attn_kernel<false, KV8>, cudaFuncAttributePreferredSharedMemoryCarveout, want);
            carveout = want;
        }
    }
    ChainArgsDev chain{nullptr, nullptr, nullptr, 0};
    if (B == 1) {
        const ChainArgs c = chain_next(static_cast<int>(splits * n_kv_heads));
        chain = ChainArgsDev{c.serial, c.wait_cnt, c.done_cnt, c.wait_arrivals};
    }
    cudaError_t e = tagged
        ? launch_chain(decode_attn_kernel<true, KV8>, grid, dim3(128), 0, static_cast<cudaStream_t>(stream), p, chain VITA_TRACE_ARG)
        : launch_chain(decode_attn_kernel<false, KV8>, grid, dim3(128), 0, static_cast<cudaStream_t>(stream), p, chain VITA_TRACE_ARG);
    if (e != cudaSuccess) return check_cuda(e, "decode_attn_kernel");
    return check_launch("decode_attn_kernel");
}

extern "C" int vita_decode_attention(const void* q, const void* k_cache, const void* v_cache,
                                     const int32_t* block_table, const int32_t* cur_pos, void* out, void* workspace,
                                     int64_t B, int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim,
                                     int64_t page_size, int64_t max_pages, int64_t splits, float scale, int64_t q_stride,
                                     void* stream) {
    DecodeAttnParams p{};
    return decode_attention_launch<false>(p, q, k_cache, v_cache, block_table, cur_pos, out, workspace, B, n_q_heads,
                                          n_kv_heads, head_dim, page_size, max_pages, splits, scale, q_stride, stream);
}

extern "C" int vita_decode_attention_fp8(const void* q, const void* k_cache, const void* v_cache,
                                         const int32_t* block_table, const int32_t* cur_pos, void* out, void* workspace,
                                         int64_t B, int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim,
                                         int64_t page_size, int64_t max_pages, int64_t splits, float scale,
                                         int64_t q_stride, float k_scale, float v_scale, void* stream) {
    VITA_REQUIRE(kv_fp8_scales_ok(k_scale, v_scale), "k_scale / v_scale must be finite and positive");
    DecodeAttnParamsFp8 p{};
    p.k_scale = k_scale; p.v_scale = v_scale;
    return decode_attention_launch<true>(p, q, k_cache, v_cache, block_table, cur_pos, out, workspace, B, n_q_heads,
                                         n_kv_heads, head_dim, page_size, max_pages, splits, scale, q_stride, stream);
}
