// Sampled next-token choice over bf16 logits (temperature, top-k, top-p, Gumbel-max draw), one CTA per row.
//
// Contract (vita_b200/sampling.py owns the policy; oracle/sampling_oracle.py restates it in fp64):
//   T == 0 (or negative) -> greedy: the packed (logit, ~index) word of argmax_rows, first index on ties
//   x_r = l_r / T in fp32 from the bf16 logit
//   top-k (0 < k < V): keep every token whose logit is >= the k-th largest (boundary ties kept)
//   top-p (p < 1): over the softmax of the top-k survivors keep r iff the mass of the survivors whose logit is strictly
//                  greater than l_r is < p (tied values are kept or dropped together); the largest logit always stays
//   draw: argmax_r over the kept set of x_r + g_r (lowest index on ties), g_r = -log(-log(u_r)),
//         u_r = ((w >> 8) + 0.5) * 2^-24, w = word (r & 3) of Philox4x32-10(counter (r >> 2, n, s, 0),
//         key (seed lo, seed hi)), n = counter[b], s = streams[b] (0 without a stream array)
// Streams: the sequences of one request (parallel sampling: generate(num_return_sequences=N), Request.n / best_of)
// share its key and draw from streams s = 0 .. N-1, so they are independent and reproducible from one seed, and
// sequence 0 draws what a single-sequence request with the same key draws.
// Logits are bf16 and the temperature is monotone, so both thresholds are found by radix selection over the 16-bit
// ordered keys of the logits (two 256-bin passes each): top-k over counts, top-p over fixed-point masses
// exp(x_r - x_max) * 2^40 summed as u64 (integer sums: the result does not depend on the order of the additions).
//
// Log-probabilities (the LOGPROBS variant, vita_sample_rows_logprobs): over the processed row -- the logits for greedy
// rows, x_r over the kept set and -inf outside it otherwise --
//   logprob(r) = x_r - x_max - log(Z * 2^-40), Z = sum over the kept set of the fixed-point masses above (u64);
//   rank(r) = 1 + #{kept tokens with a strictly greater logit}; top-N = the N largest logits, lowest index first on
//   ties (the N-th largest comes from the same radix selection as top-k, with k = N).
// Every comparison of logits -- the top-k and top-p thresholds, the kept test, ranks and top-N -- reads the ordered
// keys with -0.0 as +0.0 (canon_key), so equal logits are equal: -0.0 and +0.0 are kept or dropped together.
// A row with a target id scores that token and draws nothing (prompt rows: the next prompt token).
// The LSM variant (vita_sample_rows_logsoftmax) writes bf16(logprob(r)) of every token to the score row instead of the
// processed row: HF beam search's per-step scores, from the same Z as the logprob.
//
// Reference call sites: vLLM's Sampler (web_demo/vllm_tools/vllm_file/mixtral.py:1180-1186) and the sampling loop of
// HF generate() (video_audio_demo.py:257-270: TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper ->
// multinomial).
#include "common.h"
#include "ptx.cuh"

namespace vita {

constexpr int kSampleThreads = 1024;
constexpr int kSampleWarps = kSampleThreads / 32;
constexpr size_t kSampleHistBytes = static_cast<size_t>(kSampleWarps) * 256 * 8;   // per-warp 256-bin histograms

// bf16 bits <-> 16-bit key whose unsigned order is the numeric order (the order pack_argmax induces on floats)
__device__ __forceinline__ uint32_t bf16_key(uint32_t u) { return (u & 0x8000u) ? (~u & 0xFFFFu) : (u | 0x8000u); }
__device__ __forceinline__ float key_value(uint32_t k) {
    const uint32_t u = (k & 0x8000u) ? (k & 0x7FFFu) : (~k & 0xFFFFu);
    return __uint_as_float(u << 16);
}
// pack_argmax's key (decode.cu): -0.0 is packed as +0.0, equal values tie on the index
__device__ __forceinline__ unsigned long long pack_score(float v, int idx) {
    uint32_t u = __float_as_uint(v);
    if (u == 0x80000000u) u = 0u;
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return (static_cast<unsigned long long>(u) << 32) | static_cast<unsigned long long>(0xFFFFFFFFu - static_cast<uint32_t>(idx));
}

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// g = -log(-log(u)), u = ((w >> 8) + 0.5) * 2^-24.  -log(u) is taken as -log1p(-(1 - u)) in the upper half, where
// 1 - u = ((2^24 - 1 - (w >> 8)) + 0.5) * 2^-24 is exact in fp32 (u itself is not: it would round to 1 at the top).
__device__ __forceinline__ float gumbel(uint32_t w) {
    const uint32_t a = w >> 8;
    const float nl = a < (1u << 23) ? -logf((static_cast<float>(a) + 0.5f) * 0x1p-24f)
                                    : -log1pf(-(static_cast<float>(0xFFFFFFu - a) + 0.5f) * 0x1p-24f);
    return -logf(nl);
}
// Bounds of g over all 2^24 values of u: [-2.8527, 17.3287].  A token whose x is more than their spread (plus fp32
// slack) below x_max can never beat the largest logit's perturbed score, so it needs no noise.
constexpr float kGumbelPrune = 24.0f;

__device__ __forceinline__ unsigned long long block_max_u64(unsigned long long v, unsigned long long* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xffffffffu, v, o);
        v = other > v ? other : v;
    }
    __syncthreads();                                    // red may still be read from a previous reduction
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        v = red[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long other = __shfl_xor_sync(0xffffffffu, v, o);
            v = other > v ? other : v;
        }
        if (threadIdx.x == 0) red[0] = v;
    }
    __syncthreads();
    return red[0];
}

// -0.0 and +0.0 are one value: the key of -0.0 (0x7FFF) is read as that of +0.0
__device__ __forceinline__ uint32_t canon_key(uint32_t k) { return k == 0x7FFFu ? 0x8000u : k; }

// Histogram over the canonical keys >= floor_key: high bytes (hi_bin < 0) or the low bytes of the keys whose high
// byte is hi_bin.  Weight 1 (counts) or the fixed-point mass exp(x - x_max) * 2^40.  Result in tot[256].
// WARP_MATCH (counts only, no floor): the lanes of a warp that hit one bin add once.
template <bool WARP_MATCH = false>
__device__ void sample_hist(const uint16_t* keys, int V, unsigned long long* whist, unsigned long long* tot,
                            int hi_bin, uint32_t floor_key, bool mass, float T, float x_max) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    unsigned long long* h = whist + warp * 256;
#pragma unroll
    for (int j = 0; j < 8; ++j) h[lane + 32 * j] = 0ull;
    __syncwarp();
    if constexpr (WARP_MATCH) {
        // every lane runs every iteration (the bound is uniform), so the whole warp takes part in the match
        for (int base = 0; base < V; base += kSampleThreads) {
            const int i = base + static_cast<int>(threadIdx.x);
            int bin = -1;
            if (i < V) {
                const uint32_t k = canon_key(keys[i]);
                if (hi_bin < 0 || static_cast<int>(k >> 8) == hi_bin) bin = static_cast<int>(hi_bin < 0 ? (k >> 8) : (k & 255u));
            }
            const unsigned peers = __match_any_sync(0xffffffffu, bin);
            if (bin >= 0 && lane == __ffs(peers) - 1) atomicAdd(h + bin, static_cast<unsigned long long>(__popc(peers)));
        }
    }
    for (int i = threadIdx.x; i < V && !WARP_MATCH; i += kSampleThreads) {
        const uint32_t k = canon_key(keys[i]);
        if (k < floor_key) continue;
        if (hi_bin >= 0 && static_cast<int>(k >> 8) != hi_bin) continue;
        unsigned long long wt = 1ull;
        if (mass) {
            const float x = __fdiv_rn(key_value(k), T);
            wt = __float2ull_rn(expf(x - x_max) * 0x1p40f);
            if (wt == 0ull) continue;
        }
        atomicAdd(h + (hi_bin < 0 ? (k >> 8) : (k & 255u)), wt);
    }
    __syncthreads();
    if (threadIdx.x < 256) {
        unsigned long long s = 0ull;
        for (int w = 0; w < kSampleWarps; ++w) s += whist[w * 256 + threadIdx.x];
        tot[threadIdx.x] = s;
    }
    __syncthreads();
}

// Warp 0: the lowest bin b with base + (weight of the bins above b) < target.  The qualifying bins form a run from
// the top, so that is where the run ends.  Writes {bin or -1, weight above it} to res; res_total = sum of all bins.
__device__ void sample_search(const unsigned long long* tot, unsigned long long base, double target, int* res_bin,
                              unsigned long long* res_above, unsigned long long* res_total) {
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    unsigned long long s = 0ull;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += tot[255 - 8 * lane - j];       // lane 0 owns the 8 highest bins
    unsigned long long incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    unsigned long long above = base + incl - s;
    int last = -1;
    unsigned long long last_above = 0ull;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int b = 255 - 8 * lane - j;
        if (static_cast<double>(above) < target) { last = b; last_above = above; }
        above += tot[b];
    }
    const unsigned mask = __ballot_sync(0xffffffffu, last >= 0);
    const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
    if (mask == 0u) {
        if (lane == 0) { *res_bin = -1; *res_above = 0ull; *res_total = total; }
        return;
    }
    const int src = 31 - __clz(static_cast<int>(mask));
    const int bin = __shfl_sync(0xffffffffu, last, src);
    const unsigned long long ab = __shfl_sync(0xffffffffu, last_above, src);
    if (lane == 0) { *res_bin = bin; *res_above = ab; *res_total = total; }
}

__device__ __forceinline__ unsigned long long block_sum_u64(unsigned long long v, unsigned long long* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();                                    // red may still be read from a previous reduction
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        v = red[threadIdx.x];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (threadIdx.x == 0) red[0] = v;
    }
    __syncthreads();
    return red[0];
}

// Outputs of the LOGPROBS variant.  Output row of request b: b when rows == 0, else b * rows + counter[b] (nothing is
// written when the counter is outside [0, rows)), like the score log.
struct LogprobArgs {
    const int* target;          // [B] or null: a row with target[b] in [0, V) scores that token and draws nothing
    float* logprob;             // [out rows]
    int* rank;                  // [out rows]
    int* top_ids;               // [out rows, top_ld] (n_top > 0)
    float* top_logprobs;        // [out rows, top_ld] (n_top > 0)
    int n_top, top_ld, rows;
};
constexpr int kMaxTopLogprobs = 20;

// x of a staged key: l / T (SCALED) or l (greedy rows)
template <bool SCALED>
__device__ __forceinline__ float key_x(uint32_t k, float T) {
    if constexpr (SCALED) return __fdiv_rn(key_value(k), T);
    else return key_value(k);
}

// Logprob, rank and top-N of token `idx` over the processed row (kept set = staged keys >= thr).  Every thread
// calls it.
// LSM: srow (may be null) receives the log-softmax of the whole processed row.
template <bool SCALED, bool LSM>
__device__ void write_logprobs(const uint16_t* keys, int V, uint32_t thr, float T, float x_max, int idx,
                                            int n, int b, const LogprobArgs& lp, unsigned long long* whist,
                                            unsigned long long* tot, unsigned long long* red, int* s_bin,
                                            unsigned long long* s_above, unsigned long long* s_total,
                                            __nv_bfloat16* srow) {
    __shared__ int s_top[kMaxTopLogprobs];
    __shared__ int s_cnt, s_wcnt[kSampleWarps];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t kt = canon_key(keys[idx]), kept_t = keys[idx];
    // Z over the kept set (order-independent u64 sum) and the kept tokens strictly above the scored one
    unsigned long long z = 0ull, gt = 0ull;
    for (int i = tid; i < V; i += kSampleThreads) {
        const uint32_t k = keys[i];
        if (k < thr) continue;
        z += __float2ull_rn(expf(key_x<SCALED>(k, T) - x_max) * 0x1p40f);
        gt += canon_key(k) > kt ? 1ull : 0ull;
    }
    z = block_sum_u64(z, red);
    gt = block_sum_u64(gt, red);
    const float log_z = logf(__ull2float_rn(z) * 0x1p-40f);
    auto logprob_of = [&](uint32_t k) { return k >= thr ? (key_x<SCALED>(k, T) - x_max) - log_z : -INFINITY; };
    if constexpr (LSM) {
        if (srow != nullptr)
            for (int i = tid; i < V; i += kSampleThreads) srow[i] = __float2bfloat16(logprob_of(keys[i]));
    }

    long long row = b;
    if (lp.rows > 0) {
        if (n < 0 || n >= lp.rows) return;               // uniform over the block
        row = static_cast<long long>(b) * lp.rows + n;
    }
    if (tid == 0) {
        lp.logprob[row] = logprob_of(kept_t);
        lp.rank[row] = 1 + static_cast<int>(gt);
    }
    const int N = lp.n_top;
    if (N <= 0) return;
    // the N-th largest key (radix selection as for top-k), then every key above it and the lowest-index ties
    sample_hist<true>(keys, V, whist, tot, -1, 0u, false, 1.0f, 0.0f);
    sample_search(tot, 0ull, static_cast<double>(N), s_bin, s_above, s_total);
    __syncthreads();
    const int hb = *s_bin;
    const unsigned long long ab = *s_above;
    sample_hist<true>(keys, V, whist, tot, hb, 0u, false, 1.0f, 0.0f);
    sample_search(tot, ab, static_cast<double>(N), s_bin, s_above, s_total);
    if (tid == 0) s_cnt = 0;
    __syncthreads();
    const uint32_t thr_n = (static_cast<uint32_t>(hb) << 8) | static_cast<uint32_t>(*s_bin);
    const int above = static_cast<int>(*s_above);        // keys > thr_n: fewer than N
    for (int i = tid; i < V; i += kSampleThreads)
        if (canon_key(keys[i]) > thr_n) s_top[atomicAdd(&s_cnt, 1)] = i;
    int need = N - above;                                // ties at thr_n, taken in index order
    for (int base = 0; base < V && need > 0; base += kSampleThreads) {
        const int i = base + tid;
        const bool tie = i < V && canon_key(keys[i]) == thr_n;
        const unsigned bal = __ballot_sync(0xffffffffu, tie);
        if (lane == 0) s_wcnt[warp] = __popc(bal);
        __syncthreads();
        int before = 0, total = 0;
        for (int w = 0; w < kSampleWarps; ++w) {
            const int c = s_wcnt[w];
            before += w < warp ? c : 0;
            total += c;
        }
        const int r = before + __popc(bal & ((1u << lane) - 1u));
        if (tie && r < need) s_top[N - need + r] = i;
        need -= total < need ? total : need;
        __syncthreads();                                 // s_wcnt is rewritten by the next chunk
    }
    __syncthreads();
    if (tid < N) {                                       // order: key descending, index ascending
        const int i = s_top[tid];
        const uint32_t k = canon_key(keys[i]);
        int pos = 0;
        for (int j = 0; j < N; ++j) {
            const int o = s_top[j];
            const uint32_t ko = canon_key(keys[o]);
            pos += (ko > k || (ko == k && o < i)) ? 1 : 0;
        }
        const long long at = row * lp.top_ld + pos;
        lp.top_ids[at] = i;
        lp.top_logprobs[at] = logprob_of(keys[i]);
    }
}

template <bool LOGPROBS, bool LSM = false>
__global__ void __launch_bounds__(kSampleThreads, 1)
sample_rows_kernel(const __nv_bfloat16* __restrict__ logits, long long ld, int V, const float* __restrict__ temperature,
                   const int* __restrict__ top_k, const float* __restrict__ top_p,
                   const unsigned long long* __restrict__ seed, const int* __restrict__ counter,
                   const int* __restrict__ streams, unsigned long long* __restrict__ best, __nv_bfloat16* __restrict__ scores, long long score_ld,
                   int score_rows, int vec, LogprobArgs lp) {
    extern __shared__ __align__(16) uint8_t smem_s[];
    unsigned long long* whist = reinterpret_cast<unsigned long long*>(smem_s);
    uint16_t* keys = reinterpret_cast<uint16_t*>(smem_s + kSampleHistBytes);
    __shared__ unsigned long long tot[256];
    __shared__ unsigned long long red[32];
    __shared__ int s_bin;
    __shared__ unsigned long long s_above, s_total;

    const int b = blockIdx.x;
    const int tid = threadIdx.x;
    // Nothing is read before the wait: the logits come from the preceding kernel, and the counter (the decoder's
    // gen_count) is written on the device earlier in the same step by a kernel that triggers its dependents before
    // that write -- only griddepcontrol.wait makes it visible, whatever the chain options.  The parameter arrays and
    // the streams are read after it as well.
    pdl_wait();
    const float T = temperature[b];
    const int k = top_k[b];
    const float p = top_p[b];
    const unsigned long long key = seed[b];
    const int n = counter[b];
    const uint32_t sid = streams != nullptr ? static_cast<uint32_t>(streams[b]) : 0u;
    int tgt = -1;
    if constexpr (LOGPROBS) {
        if (lp.target != nullptr) tgt = lp.target[b];
        if (tgt >= V) tgt = -1;
    }

    // stage the row as ordered keys; greedy arg-max on the way (largest key, first index; -0.0 ties with +0.0)
    const __nv_bfloat16* row = logits + static_cast<long long>(b) * ld;
    uint32_t bk = 0u;
    int bi = 0x7fffffff;
    if (vec) {
        for (int j = tid; j < (V >> 3); j += kSampleThreads) {
            const uint4 q = __ldg(reinterpret_cast<const uint4*>(row) + j);
            const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
            uint32_t kk[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const uint32_t lo = bf16_key(w4[e] & 0xFFFFu), hi = bf16_key(w4[e] >> 16);
                kk[e] = lo | (hi << 16);
                const int i = 8 * j + 2 * e;
                const uint32_t cl = canon_key(lo), ch = canon_key(hi);
                if (cl > bk || (cl == bk && i < bi)) { bk = cl; bi = i; }
                if (ch > bk || (ch == bk && i + 1 < bi)) { bk = ch; bi = i + 1; }
            }
            reinterpret_cast<uint4*>(keys)[j] = make_uint4(kk[0], kk[1], kk[2], kk[3]);
        }
    } else {
        const uint16_t* r16 = reinterpret_cast<const uint16_t*>(row);
        for (int i = tid; i < V; i += kSampleThreads) {
            const uint32_t kk = bf16_key(r16[i]);
            keys[i] = static_cast<uint16_t>(kk);
            const uint32_t ck = canon_key(kk);
            if (ck > bk || (ck == bk && i < bi)) { bk = ck; bi = i; }
        }
    }
    const unsigned long long arg = block_max_u64(bi == 0x7fffffff ? 0ull : pack_score(key_value(bk), bi), red);
    const bool greedy = !(T > 0.0f);
    __nv_bfloat16* srow = nullptr;
    if (scores != nullptr && n >= 0 && n < score_rows)
        srow = scores + (static_cast<long long>(b) * score_rows + n) * score_ld;

    if (greedy) {                                        // bit-identical to argmax_rows; the score log gets the logits
        if (tid == 0) best[b] = arg;
        if (srow != nullptr && !LSM)
            for (int i = tid; i < V; i += kSampleThreads) srow[i] = __float2bfloat16(key_value(keys[i]));
        if constexpr (!LOGPROBS) return;
    }
    const uint32_t ord = static_cast<uint32_t>(arg >> 32);     // undo pack_score's float ordering, then re-key
    const uint32_t max_key = bf16_key(((ord & 0x80000000u) ? (ord & 0x7FFFFFFFu) : ~ord) >> 16);   // canonical
    if constexpr (LOGPROBS) {
        if (greedy) {                                    // the processed row is the logits: x = l, every token kept
            const int idx = tgt >= 0 ? tgt : static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(arg & 0xFFFFFFFFull));
            write_logprobs<false, LSM>(keys, V, 0u, 1.0f, key_value(max_key), idx, n, b, lp, whist, tot, red, &s_bin,
                                       &s_above, &s_total, srow);
            return;
        }
    }
    const float x_max = __fdiv_rn(key_value(max_key), T);

    // top-k threshold: the k-th largest canonical key
    uint32_t thr = 0u;
    if (k > 0 && k < V) {
        sample_hist(keys, V, whist, tot, -1, 0u, false, T, x_max);
        sample_search(tot, 0ull, static_cast<double>(k), &s_bin, &s_above, &s_total);
        __syncthreads();
        const int hb = s_bin;
        const unsigned long long ab = s_above;
        sample_hist(keys, V, whist, tot, hb, 0u, false, T, x_max);
        sample_search(tot, ab, static_cast<double>(k), &s_bin, &s_above, &s_total);
        __syncthreads();
        thr = (static_cast<uint32_t>(hb) << 8) | static_cast<uint32_t>(s_bin);
    }
    // top-p threshold over the top-k survivors: the lowest canonical key whose strictly-greater survivor mass is
    // < p * Z
    if (p < 1.0f) {
        sample_hist(keys, V, whist, tot, -1, thr, true, T, x_max);
        if (tid < 32) {                                  // Z = survivor mass = sum of all bins
            unsigned long long s = 0ull;
            for (int j = tid; j < 256; j += 32) s += tot[j];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            if (tid == 0) s_total = s;
        }
        __syncthreads();
        const double target = static_cast<double>(p) * static_cast<double>(s_total);
        __syncthreads();                                 // s_total is rewritten by the search
        sample_search(tot, 0ull, target, &s_bin, &s_above, &s_total);
        __syncthreads();
        const int hb = s_bin;
        const unsigned long long ab = s_above;
        uint32_t tp = max_key;                           // nothing qualifies (p == 0): the largest logit stays
        if (hb >= 0) {
            sample_hist(keys, V, whist, tot, hb, thr, true, T, x_max);
            sample_search(tot, ab, target, &s_bin, &s_above, &s_total);
            __syncthreads();
            tp = (static_cast<uint32_t>(hb) << 8) | static_cast<uint32_t>(s_bin < 0 ? 0 : s_bin);
        }
        thr = tp > thr ? tp : thr;
    }
    // the thresholds are canonical keys; the kept tests below read the staged keys, on which -0.0 (0x7FFF) sorts
    // just below +0.0 (0x8000): a threshold at zero is lowered to -0.0's key so that both zeros are kept
    if (thr == 0x8000u) thr = 0x7FFFu;

    // Gumbel-max over the kept keys (>= thr)
    const float x_floor = x_max - kGumbelPrune;
    const uint32_t k0 = static_cast<uint32_t>(key), k1 = static_cast<uint32_t>(key >> 32);
    unsigned long long loc = 0ull;
    const int n_groups = (V + 3) >> 2;
    for (int j = tid; j < n_groups; j += kSampleThreads) {
        float x[4];
        bool kept[4], need = false;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int i = 4 * j + e;
            const uint32_t kk = i < V ? keys[i] : 0u;
            kept[e] = i < V && kk >= thr;
            x[e] = __fdiv_rn(key_value(kk), T);
            need |= kept[e] && x[e] >= x_floor;
            if constexpr (LOGPROBS) need &= tgt < 0;    // a scored row draws nothing
            if (srow != nullptr && i < V) srow[i] = kept[e] ? __float2bfloat16(x[e]) : __float2bfloat16(-INFINITY);
        }
        if (!need) continue;
        const uint4 w = philox4x32_10(make_uint4(static_cast<uint32_t>(j), static_cast<uint32_t>(n), sid, 0u), k0, k1);
        const uint32_t ww[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            if (!kept[e] || x[e] < x_floor) continue;
            const unsigned long long s = pack_score(x[e] + gumbel(ww[e]), 4 * j + e);
            loc = s > loc ? s : loc;
        }
    }
    const unsigned long long win = block_max_u64(loc, red);
    if constexpr (LOGPROBS) {
        if (tgt >= 0) {                                  // a scored row leaves the greedy word in best
            if (tid == 0) best[b] = arg;
            write_logprobs<true, LSM>(keys, V, thr, T, x_max, tgt, n, b, lp, whist, tot, red, &s_bin, &s_above,
                                      &s_total, srow);
            return;
        }
    }
    // the winner's packed word keeps the arg-max layout: (bf16 logit as float, ~index)
    if (tid == 0) {
        const int idx = static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(win & 0xFFFFFFFFull));
        best[b] = pack_score(key_value(keys[idx]), idx);
    }
    if constexpr (LOGPROBS)
        write_logprobs<true, LSM>(keys, V, thr, T, x_max,
                                  static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(win & 0xFFFFFFFFull)), n, b, lp,
                                  whist, tot, red, &s_bin, &s_above, &s_total, srow);
}

}  // namespace vita

using namespace vita;

namespace {

template <bool LOGPROBS, bool LSM = false>
int launch_sample_rows(const void* logits, int64_t ld, int64_t B, int64_t V, const float* temperature,
                       const int32_t* top_k, const float* top_p, const uint64_t* seed, const int32_t* counter,
                       const int32_t* streams, uint64_t* best, void* scores, int64_t score_ld, int64_t score_rows,
                       const LogprobArgs& lp, void* stream) {
    VITA_REQUIRE(V > 0 && ld >= V, "need 0 < V <= ld");
    VITA_REQUIRE(temperature && top_k && top_p && seed && counter && best, "parameter arrays are required");
    VITA_REQUIRE(scores == nullptr || (score_ld >= V && score_rows > 0), "score log: need score_ld >= V, rows > 0");
    if (B == 0) return VITA_OK;
    // dynamic shared memory available = the device's opt-in per-block limit minus the kernel's static shared memory
    // (on an H100: 232448 - 2336 bytes, which leaves V <= 82288 next to the 64 KB of histograms)
    static size_t dyn_limit = 0;
    if (dyn_limit == 0) {
        int dev = 0, optin = 0;
        cudaFuncAttributes fa{};
        int rc = check_cuda(cudaGetDevice(&dev), "sample_rows");
        if (!rc) rc = check_cuda(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev), "sample_rows");
        if (!rc) rc = check_cuda(cudaFuncGetAttributes(&fa, sample_rows_kernel<LOGPROBS, LSM>), "sample_rows");
        if (rc) return rc;
        dyn_limit = static_cast<size_t>(optin) > fa.sharedSizeBytes ? static_cast<size_t>(optin) - fa.sharedSizeBytes : 0;
    }
    const size_t smem = kSampleHistBytes + ((static_cast<size_t>(V) * 2 + 15) / 16) * 16;
    VITA_REQUIRE(smem <= dyn_limit, "the row does not fit shared memory (V <= " +
                                        std::to_string(dyn_limit > kSampleHistBytes ? (dyn_limit - kSampleHistBytes) / 16 * 8 : 0) +
                                        " on this device)");
    static size_t configured = 0;
    if (smem > configured) {
        const int rc = check_cuda(cudaFuncSetAttribute(sample_rows_kernel<LOGPROBS, LSM>,
                                                       cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       static_cast<int>(smem)), "sample_rows");
        if (rc) return rc;
        configured = smem;
    }
    const int vec = (V % 8 == 0 && ld % 8 == 0 && aligned16(logits)) ? 1 : 0;
    // launched as a programmatic dependent of the LM head: the kernel waits (griddepcontrol.wait) before reading the
    // logits and never triggers its own dependents early, so the next step starts after its last write of `best`
    cudaError_t e = launch_chain(sample_rows_kernel<LOGPROBS, LSM>, dim3(static_cast<unsigned>(B)), dim3(kSampleThreads), smem,
                                 static_cast<cudaStream_t>(stream), BF16C(logits), (long long)ld, (int)V, temperature,
                                 top_k, top_p, reinterpret_cast<const unsigned long long*>(seed), counter, streams,
                                 reinterpret_cast<unsigned long long*>(best), static_cast<__nv_bfloat16*>(scores),
                                 (long long)score_ld, (int)score_rows, vec, lp);
    if (e != cudaSuccess) return check_cuda(e, "sample_rows");
    return check_launch("sample_rows");
}

template <bool LSM>
int launch_logprobs(const void* logits, int64_t ld, int64_t B, int64_t V, const float* temperature,
                    const int32_t* top_k, const float* top_p, const uint64_t* seed, const int32_t* counter,
                    const int32_t* streams, const int32_t* target, uint64_t* best, void* scores, int64_t score_ld,
                    int64_t score_rows, float* logprob, int32_t* rank, int32_t* top_ids, float* top_logprobs,
                    int64_t n_top, int64_t top_ld, int64_t out_rows, void* stream) {
    VITA_REQUIRE(logprob && rank, "logprob and rank outputs are required");
    VITA_REQUIRE(n_top >= 0 && n_top <= kMaxTopLogprobs && n_top <= V, "need 0 <= n_top <= min(20, V)");
    VITA_REQUIRE(n_top == 0 || (top_ids && top_logprobs && top_ld >= n_top), "top-N outputs: need top_ld >= n_top");
    VITA_REQUIRE(out_rows >= 0, "out_rows must be >= 0");
    const LogprobArgs lp{target, logprob, rank, top_ids, top_logprobs, (int)n_top, (int)top_ld, (int)out_rows};
    return launch_sample_rows<true, LSM>(logits, ld, B, V, temperature, top_k, top_p, seed, counter, streams, best,
                                         scores, score_ld, score_rows, lp, stream);
}

}  // namespace

extern "C" int vita_sample_rows_streams(const void* logits, int64_t ld, int64_t B, int64_t V,
                                        const float* temperature, const int32_t* top_k, const float* top_p,
                                        const uint64_t* seed, const int32_t* counter, const int32_t* streams,
                                        const int32_t* target, uint64_t* best, void* scores, int64_t score_ld,
                                        int64_t score_rows, float* logprob, int32_t* rank, int32_t* top_ids,
                                        float* top_logprobs, int64_t n_top, int64_t top_ld, int64_t out_rows,
                                        int64_t log_softmax, void* stream) {
    if (logprob == nullptr && rank == nullptr) {
        VITA_REQUIRE(target == nullptr && log_softmax == 0, "target / log-softmax scores need the logprob outputs");
        return launch_sample_rows<false>(logits, ld, B, V, temperature, top_k, top_p, seed, counter, streams, best,
                                         scores, score_ld, score_rows, LogprobArgs{}, stream);
    }
    if (log_softmax)
        return launch_logprobs<true>(logits, ld, B, V, temperature, top_k, top_p, seed, counter, streams, target, best,
                                     scores, score_ld, score_rows, logprob, rank, top_ids, top_logprobs, n_top, top_ld,
                                     out_rows, stream);
    return launch_logprobs<false>(logits, ld, B, V, temperature, top_k, top_p, seed, counter, streams, target, best,
                                  scores, score_ld, score_rows, logprob, rank, top_ids, top_logprobs, n_top, top_ld,
                                  out_rows, stream);
}

extern "C" int vita_sample_rows(const void* logits, int64_t ld, int64_t B, int64_t V, const float* temperature,
                                const int32_t* top_k, const float* top_p, const uint64_t* seed, const int32_t* counter,
                                uint64_t* best, void* scores, int64_t score_ld, int64_t score_rows, void* stream) {
    return vita_sample_rows_streams(logits, ld, B, V, temperature, top_k, top_p, seed, counter, nullptr, nullptr, best,
                                    scores, score_ld, score_rows, nullptr, nullptr, nullptr, nullptr, 0, 0, 0, 0,
                                    stream);
}

#define VITA_LOGPROBS_ARGS logits, ld, B, V, temperature, top_k, top_p, seed, counter, nullptr, target, best, scores, \
                           score_ld, score_rows, logprob, rank, top_ids, top_logprobs, n_top, top_ld, out_rows

extern "C" int vita_sample_rows_logprobs(const void* logits, int64_t ld, int64_t B, int64_t V,
                                         const float* temperature, const int32_t* top_k, const float* top_p,
                                         const uint64_t* seed, const int32_t* counter, const int32_t* target,
                                         uint64_t* best, void* scores, int64_t score_ld, int64_t score_rows,
                                         float* logprob, int32_t* rank, int32_t* top_ids, float* top_logprobs,
                                         int64_t n_top, int64_t top_ld, int64_t out_rows, void* stream) {
    VITA_REQUIRE(logprob && rank, "logprob and rank outputs are required");
    return vita_sample_rows_streams(VITA_LOGPROBS_ARGS, 0, stream);
}

extern "C" int vita_sample_rows_logsoftmax(const void* logits, int64_t ld, int64_t B, int64_t V,
                                           const float* temperature, const int32_t* top_k, const float* top_p,
                                           const uint64_t* seed, const int32_t* counter, const int32_t* target,
                                           uint64_t* best, void* scores, int64_t score_ld, int64_t score_rows,
                                           float* logprob, int32_t* rank, int32_t* top_ids, float* top_logprobs,
                                           int64_t n_top, int64_t top_ld, int64_t out_rows, void* stream) {
    VITA_REQUIRE(logprob && rank, "logprob and rank outputs are required");
    return vita_sample_rows_streams(VITA_LOGPROBS_ARGS, 1, stream);
}
