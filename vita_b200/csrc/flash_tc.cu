// FlashAttention forward for sm_90a on wgmma:  O = softmax(Q K^T * scale [masks]) V.
//
// One CTA owns a query tile of 128 rows and walks the keys in tiles of 128 (384 threads):
//   warpgroup 0    : TMA producer (one thread; cp.async.bulk.tensor 4-D boxes, 128B swizzle: Q once, K / V through
//                    mbarrier rings); gives its registers to the consumers with setmaxnreg
//   warpgroups 1-2 : consumers, 64 query rows each.  S = Q K_j^T as wgmma m64n128k16 with both operands from shared
//                    memory; running max / exp2 / sum on the accumulator fragment (a row lives in the four lanes of a
//                    quad); the bf16 probabilities stay in registers as the A operand of O += P V_j (wgmma with V as
//                    an MN-major shared operand).  The O accumulator is rescaled only when the running max moved by
//                    more than 2^8 (the final 1/l normalisation absorbs the stale reference).
// Inside a warpgroup MMA and softmax alternate; the two warpgroups are independent and can overlap each other.
//
// Serves the three prefill-shaped attentions of the path (reference call sites):
//   Mixtral causal GQA 128/128  transformers sdpa / eager attention (modeling_mixtral.py:269-292)
//   InternViT non-causal 64/64  flash_attn_varlen_qkvpacked_func (internvit/flash_attention.py:61)
//   Whale rel-pos 128/64        attention.py:391-415, both score terms as one contraction over [k | p], key padding
//
// The PAGED instantiation (Mixtral 128/128, causal) continues sequences whose keys sit in a paged KV cache: prompt
// chunks and prompts whose prefix is cached (vLLM's paged attention in MixtralAttention.forward, mixtral.py:484-501,
// when a prefill continues cached blocks).  Only the producer and the per-CTA set-up differ: a CTA takes its
// (sequence, query block) from a host-built tile list, and a K / V tile of 128 keys arrives as one TMA box per page and
// per 64-column half.  Pages start at multiples of 16 rows (2048 B), so the 128B-swizzled shared-memory image is the
// one the single 128-row box of the contiguous path writes, and the consumers run unchanged.  V rows at positions
// >= ctx (stale page tails, pages never loaded) are zeroed before the P V product; masked scores alone would leave
// 0 * NaN.
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace vita {

struct FaParams {
    __nv_bfloat16* o;
    long long o_bs, o_ts, o_hs;   // batch / token / head strides in elements
    int group;                    // query heads per kv head
    int Sq, Skv;
    const int* kv_lens;           // [B] valid keys per batch entry, or nullptr
    int causal;
    int q_pos0;                   // causal: key position of query row 0 (rows of a sequence shard start later)
    float scale_log2;             // softmax scale * log2(e)
    int n_qblk;                   // number of 128-row query blocks
    int poly_chunks;              // of the 4 column chunks of a tile, how many take exp2 on the FMA pipe (MUFU relief)
    // PAGED: CTA blockIdx.x serves tiles[2 blockIdx.x ..] = (sequence i, query block); sequence i owns packed query
    // rows [qsl[i], qsl[i + 1]) and ctx[i] keys (its cached prefix and the rows themselves) in the pages block_table[i]
    const int* tiles;             // int32 pairs: 4-byte alignment only
    const int* qsl;
    const int* ctx;
    const int* block_table;
    int bt_stride;
    int page_shift;               // log2(page_size)
};

constexpr int FA_BM = 128;   // query rows per tile (64 per consumer warpgroup)
constexpr int FA_BN = 128;   // keys per tile

template <int DQK, int DV>
struct FaCfg {
    static constexpr int STAGES = (DQK == 128 && DV == 128) ? 2 : (DQK == 128 ? 3 : 4);
    static constexpr int Q_BYTES = FA_BM * DQK * 2;
    static constexpr int K_BYTES = FA_BN * DQK * 2;
    static constexpr int V_BYTES = FA_BN * DV * 2;
    static constexpr int THREADS = 384;
    static constexpr int SMEM = Q_BYTES + STAGES * (K_BYTES + V_BYTES) + 1024 /*align*/ + 256 /*barriers*/;
};

template <int DQK, int DV, int POLY, bool PAGED>
__global__ void __launch_bounds__(FaCfg<DQK, DV>::THREADS, 1)
flash_tc_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                const __grid_constant__ CUtensorMap tmV, const FaParams p) {
    using Cfg = FaCfg<DQK, DV>;
    constexpr int ST = Cfg::STAGES;
    constexpr int HALF = FA_BM * 128;   // bytes of one 64-column block of a 128-row tile ([128 rows][128 B])

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sQ = smem;
    uint8_t* sK = sQ + Cfg::Q_BYTES;
    uint8_t* sV = sK + ST * Cfg::K_BYTES;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ST * Cfg::V_BYTES);
    uint64_t* q_full = bars;
    uint64_t* k_full = bars + 1;
    uint64_t* k_empty = k_full + ST;
    uint64_t* v_full = k_empty + ST;
    uint64_t* v_empty = v_full + ST;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int head = blockIdx.y;
    const int kvh = head / p.group;
    int b, q0, Sq, q_pos0, kv_len, q_row0;   // q_row0: TMA row coordinate of query row q0
    __nv_bfloat16* obase;                     // output row 0 of this (batch entry | sequence)
    const int* bt = nullptr;
    if constexpr (PAGED) {
        const int seq = p.tiles[2 * blockIdx.x];   // the host orders the list long causal rows first
        const int r0 = p.qsl[seq];
        b = 0;
        q0 = p.tiles[2 * blockIdx.x + 1] * FA_BM;
        Sq = p.qsl[seq + 1] - r0;
        kv_len = p.ctx[seq];
        q_pos0 = kv_len - Sq;
        q_row0 = r0 + q0;
        obase = p.o + static_cast<long long>(r0) * p.o_ts;
        bt = p.block_table + static_cast<long long>(seq) * p.bt_stride;
    } else {
        b = blockIdx.z;
        // long causal rows first
        const int bx = p.causal ? static_cast<int>(gridDim.x) - 1 - static_cast<int>(blockIdx.x) : static_cast<int>(blockIdx.x);
        q0 = bx * FA_BM;
        Sq = p.Sq;
        q_pos0 = p.q_pos0;
        kv_len = p.kv_lens ? p.kv_lens[b] : p.Skv;
        if (kv_len > p.Skv) kv_len = p.Skv;
        if (kv_len < 0) kv_len = 0;
        q_row0 = q0;
        obase = nullptr;   // p.o + b * p.o_bs, formed where it is used (keeps this instantiation's code as it was)
    }
    int n_tiles = (kv_len + FA_BN - 1) / FA_BN;
    if (p.causal) {
        const int lim = (q_pos0 + q0 + FA_BM + FA_BN - 1) / FA_BN;   // keys <= last row of the tile
        if (n_tiles > lim) n_tiles = lim;
    }

    if (n_tiles == 0) {   // no keys at all: zeros (uniform over the CTA)
        if (threadIdx.x >= 128 && threadIdx.x < 128 + FA_BM) {
            const int row = q0 + static_cast<int>(threadIdx.x) - 128;
            if (row < Sq) {
                uint4* orow = reinterpret_cast<uint4*>((PAGED ? obase : p.o + b * p.o_bs) + static_cast<long long>(row) * p.o_ts + head * p.o_hs);
                for (int i = 0; i < DV / 8; ++i) orow[i] = make_uint4(0, 0, 0, 0);
            }
        }
        return;
    }

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmQ);
        tma_prefetch_desc(&tmK);
        tma_prefetch_desc(&tmV);
        mbar_init(q_full, 1);
        for (int i = 0; i < ST; ++i) {
            mbar_init(&k_full[i], 1);
            mbar_init(&k_empty[i], 8);   // one arrival per consumer warp
            mbar_init(&v_full[i], 1);
            mbar_init(&v_empty[i], 8);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // ------------------------------------------------------------------------------------ TMA producer
        // 384 x 168 registers at launch = 128 x 40 + 256 x 232
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            mbar_arrive_expect_tx(q_full, Cfg::Q_BYTES);
#pragma unroll
            for (int c = 0; c < DQK / 64; ++c) tma_load_4d(sQ + c * HALF, &tmQ, q_full, c * 64, q_row0, head, b);
            int stage = 0;
            uint32_t phase = 0;
            if constexpr (PAGED) {
                // tmK / tmV: [slots][n_kv][D] with a box of {64, 1, page_size}; pages past ctx are never read
                constexpr int MAXPG = FA_BN / 16;
                const int ps = 1 << p.page_shift;
                const int ppt = FA_BN >> p.page_shift;   // pages per key tile
                for (int j = 0; j < n_tiles; ++j) {
                    const int pg0 = j * ppt;
                    const int npg = min(ppt, ((kv_len + ps - 1) >> p.page_shift) - pg0);
                    int slot0[MAXPG];
#pragma unroll
                    for (int g = 0; g < MAXPG; ++g) slot0[g] = g < npg ? bt[pg0 + g] << p.page_shift : 0;
                    const uint32_t rows = static_cast<uint32_t>(npg) << p.page_shift;
                    mbar_wait(&k_empty[stage], phase ^ 1, 10);
                    mbar_arrive_expect_tx(&k_full[stage], rows * DQK * 2);
#pragma unroll
                    for (int g = 0; g < MAXPG; ++g)
                        if (g < npg)
#pragma unroll
                            for (int c = 0; c < DQK / 64; ++c)
                                tma_load_3d(sK + stage * Cfg::K_BYTES + c * HALF + g * ps * 128, &tmK, &k_full[stage],
                                            c * 64, kvh, slot0[g]);
                    mbar_wait(&v_empty[stage], phase ^ 1, 11);
                    mbar_arrive_expect_tx(&v_full[stage], rows * DV * 2);
#pragma unroll
                    for (int g = 0; g < MAXPG; ++g)
                        if (g < npg)
#pragma unroll
                            for (int c = 0; c < DV / 64; ++c)
                                tma_load_3d(sV + stage * Cfg::V_BYTES + c * HALF + g * ps * 128, &tmV, &v_full[stage],
                                            c * 64, kvh, slot0[g]);
                    if (++stage == ST) { stage = 0; phase ^= 1; }
                }
            } else {
                for (int j = 0; j < n_tiles; ++j) {
                    mbar_wait(&k_empty[stage], phase ^ 1, 10);
                    mbar_arrive_expect_tx(&k_full[stage], Cfg::K_BYTES);
#pragma unroll
                    for (int c = 0; c < DQK / 64; ++c)
                        tma_load_4d(sK + stage * Cfg::K_BYTES + c * HALF, &tmK, &k_full[stage], c * 64, j * FA_BN, kvh, b);
                    mbar_wait(&v_empty[stage], phase ^ 1, 11);
                    mbar_arrive_expect_tx(&v_full[stage], Cfg::V_BYTES);
#pragma unroll
                    for (int c = 0; c < DV / 64; ++c)
                        tma_load_4d(sV + stage * Cfg::V_BYTES + c * HALF, &tmV, &v_full[stage], c * 64, j * FA_BN, kvh, b);
                    if (++stage == ST) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ------------------------------------------------------------------------------------ consumers
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = (warp >> 2) - 1;                    // rows [64 cw, 64 cw + 64) of the query tile
    const int qr = lane >> 2, qc = lane & 3;
    const int wg_q0 = q0 + cw * 64;
    int row[2];
    row[0] = wg_q0 + (warp & 3) * 16 + qr;
    row[1] = row[0] + 8;
    const uint32_t sQ_a = smem_u32(sQ) + cw * (64 * 128), sK_a = smem_u32(sK), sV_a = smem_u32(sV);
    float o[DV / 2];
#pragma unroll
    for (int i = 0; i < DV / 2; ++i) o[i] = 0.0f;
    float m_ref[2] = {-INFINITY, -INFINITY}, l[2] = {0.0f, 0.0f};   // l: this thread's share of the row sum
    int stage = 0;
    uint32_t phase = 0;
    mbar_wait(q_full, 0, 20);
    for (int j = 0; j < n_tiles; ++j) {
        // ---- S = Q K_j^T
        float s[FA_BN / 2];
        mbar_wait(&k_full[stage], phase, 21);
        wgmma_acc_fence(s);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < DQK / 16; ++k) {
            const uint32_t off = (k >> 2) * HALF + (k & 3) * 32;   // 64-column block, then 32 B per 16 elements
            wgmma_ss<FA_BN>(s, wgmma_desc_k_sw128(sQ_a + off), wgmma_desc_k_sw128(sK_a + stage * Cfg::K_BYTES + off),
                            k != 0 ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_acc_fence(s);
        if (lane == 0) mbar_arrive(&k_empty[stage]);

        // ---- softmax on the fragment: s[4 jb + 2 h + e] is row[h], key col0 + 8 jb + 2 qc + e
        const int col0 = j * FA_BN;
        const bool boundary = (col0 + FA_BN > kv_len) || (p.causal && col0 + FA_BN - 1 > q_pos0 + wg_q0);   // warp-uniform
        if (boundary) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int lim = p.causal ? min(kv_len, q_pos0 + row[h] + 1) : kv_len;   // columns >= lim are masked
#pragma unroll
                for (int jb = 0; jb < FA_BN / 8; ++jb)
#pragma unroll
                    for (int e = 0; e < 2; ++e)
                        if (col0 + jb * 8 + 2 * qc + e >= lim) s[4 * jb + 2 * h + e] = -INFINITY;
            }
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float mx = -INFINITY;
#pragma unroll
            for (int jb = 0; jb < FA_BN / 8; ++jb) mx = fmaxf(mx, fmaxf(s[4 * jb + 2 * h], s[4 * jb + 2 * h + 1]));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float m_new = fmaxf(m_ref[h], mx * p.scale_log2);
            if (m_new > m_ref[h] + 8.0f) {
                // move the reference of this row (the decision is per row, identical in its four lanes): rescale the
                // row sum and the accumulator
                const float alpha = ex2_approx(m_ref[h] - m_new);
                l[h] *= alpha;
                m_ref[h] = m_new;
                if (j > 0) {
#pragma unroll
                    for (int jb = 0; jb < DV / 8; ++jb) {
                        o[4 * jb + 2 * h] *= alpha;
                        o[4 * jb + 2 * h + 1] *= alpha;
                    }
                }
            }
            const float m_use = (m_ref[h] == -INFINITY) ? 0.0f : m_ref[h];
            float sum = 0.0f;
#pragma unroll
            for (int jb = 0; jb < FA_BN / 8; ++jb)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float x = fmaf(s[4 * jb + 2 * h + e], p.scale_log2, -m_use);
                    const float a = ((jb >> 2) < POLY) ? ex2_poly(x) : ex2_approx(x);
                    sum += a;
                    s[4 * jb + 2 * h + e] = a;
                }
            l[h] += sum;
        }

        // ---- O += P V_j: 16 keys per instruction, P from registers, V rows of 128 B as an MN-major operand (64-column
        // blocks FA_BN * 128 B apart, 8-key groups 1024 B apart)
        mbar_wait(&v_full[stage], phase, 22);
        if constexpr (PAGED) {
            if (col0 + FA_BN > kv_len) {   // CTA-uniform: zero V rows [kv_len - col0, FA_BN) (both consumer warpgroups)
                const int r_lo = kv_len - col0;
                const int n = (FA_BN - r_lo) * (DV / 8);   // 16-byte chunks; a row is 128 B in each 64-column half
                uint8_t* vt = sV + stage * Cfg::V_BYTES;
                for (int i = static_cast<int>(threadIdx.x) - 128; i < n; i += 256) {
                    const int r = r_lo + i / (DV / 8), c = i % (DV / 8);
                    *reinterpret_cast<uint4*>(vt + (c >> 3) * HALF + r * 128 + (c & 7) * 16) = make_uint4(0, 0, 0, 0);
                }
                fence_proxy_async_smem();
                asm volatile("bar.sync 1, 256;" ::: "memory");
            }
        }
        wgmma_acc_fence(o);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < FA_BN / 16; ++kk) {
            const uint32_t a[4] = {pack_bf16(s[8 * kk + 0], s[8 * kk + 1]), pack_bf16(s[8 * kk + 2], s[8 * kk + 3]),
                                   pack_bf16(s[8 * kk + 4], s[8 * kk + 5]), pack_bf16(s[8 * kk + 6], s[8 * kk + 7])};
            wgmma_rs_bt<DV>(o, a, wgmma_desc_mn_sw128(sV_a + stage * Cfg::V_BYTES + kk * 2048, FA_BN * 128, 1024),
                            (j > 0 || kk > 0) ? 1 : 0);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_acc_fence(o);
        if (lane == 0) mbar_arrive(&v_empty[stage]);
        if (++stage == ST) { stage = 0; phase ^= 1; }
    }

    // ---- epilogue: O / l -> bf16 -> global
    if constexpr (PAGED) {   // re-read rather than keep live through the loop (register pressure of the POLY variant)
        const int seq = p.tiles[2 * blockIdx.x];
        const int r0 = p.qsl[seq];
        Sq = p.qsl[seq + 1] - r0;
        obase = p.o + static_cast<long long>(r0) * p.o_ts;
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        float lt = l[h];
        lt += __shfl_xor_sync(0xffffffffu, lt, 1);
        lt += __shfl_xor_sync(0xffffffffu, lt, 2);
        const float inv = lt > 0.0f ? 1.0f / lt : 0.0f;
        if (row[h] < Sq) {
            __nv_bfloat16* orow = (PAGED ? obase : p.o + b * p.o_bs) + static_cast<long long>(row[h]) * p.o_ts + head * p.o_hs;
#pragma unroll
            for (int jb = 0; jb < DV / 8; ++jb)
                *reinterpret_cast<uint32_t*>(orow + jb * 8 + 2 * qc) = pack_bf16(o[4 * jb + 2 * h] * inv, o[4 * jb + 2 * h + 1] * inv);
        }
    }
}

template <int DQK, int DV, int POLY, bool PAGED>
static int launch_flash_tc_p(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const FaParams& p,
                             dim3 grid, cudaStream_t st) {
    using Cfg = FaCfg<DQK, DV>;
    static bool configured = false;
    auto kern = flash_tc_kernel<DQK, DV, POLY, PAGED>;
    if (!configured) {
        int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM),
                            "cudaFuncSetAttribute(flash_tc smem)");
        if (rc) return rc;
        configured = true;
    }
    kern<<<grid, Cfg::THREADS, Cfg::SMEM, st>>>(tmQ, tmK, tmV, p);
    return check_launch("flash_tc_kernel");
}

// POLY = column chunks (of 4 per key tile) whose exp2 runs as a polynomial on the FMA pipe (option "fa_poly")
template <int DQK, int DV, bool PAGED = false>
static int launch_flash_tc(const CUtensorMap& tmQ, const CUtensorMap& tmK, const CUtensorMap& tmV, const FaParams& p,
                           dim3 grid, cudaStream_t st) {
    if (p.poly_chunks >= 1) return launch_flash_tc_p<DQK, DV, 1, PAGED>(tmQ, tmK, tmV, p, grid, st);
    return launch_flash_tc_p<DQK, DV, 0, PAGED>(tmQ, tmK, tmV, p, grid, st);
}

// 4-D view (D, tokens, heads, batch) of a strided activation; box = 64 columns x 128 tokens, 128B swizzle
static int make_qkv_map(CUtensorMap* out, const void* base, int D, int64_t S, int64_t H, int64_t B, int64_t ts,
                        int64_t hs, int64_t bs) {
    const uint64_t dims[4] = {static_cast<uint64_t>(D), static_cast<uint64_t>(S), static_cast<uint64_t>(H),
                              static_cast<uint64_t>(B)};
    // a size-1 dimension may come with stride 0: give it any legal (non-zero, 16-byte multiple) stride
    const uint64_t ts_b = static_cast<uint64_t>(ts > 0 ? ts : D) * 2;
    const uint64_t hs_b = static_cast<uint64_t>(hs > 0 ? hs : D) * 2;
    const uint64_t bs_b = static_cast<uint64_t>(bs > 0 ? bs : D) * 2;
    const uint64_t strides[3] = {ts_b, hs_b, bs_b};
    const uint32_t box[4] = {64, 128, 1, 1};
    return make_tensor_map_bf16(out, base, 4, dims, strides, box, true);
}

template <int DQK, int DV>
static int flash_tc_dispatch(const void* q, const void* k, const void* v, const int64_t* qs, const int64_t* ks,
                             const int64_t* vs, FaParams p, int B, int Hq, int Hkv, cudaStream_t st) {
    CUtensorMap tmQ, tmK, tmV;
    int rc = make_qkv_map(&tmQ, q, DQK, p.Sq, Hq, B, qs[1], qs[2], qs[0]);
    if (rc) return rc;
    rc = make_qkv_map(&tmK, k, DQK, p.Skv, Hkv, B, ks[1], ks[2], ks[0]);
    if (rc) return rc;
    rc = make_qkv_map(&tmV, v, DV, p.Skv, Hkv, B, vs[1], vs[2], vs[0]);
    if (rc) return rc;
    p.n_qblk = (p.Sq + FA_BM - 1) / FA_BM;
    p.poly_chunks = option("fa_poly");
    dim3 grid(p.n_qblk, Hq, B);
    return launch_flash_tc<DQK, DV>(tmQ, tmK, tmV, p, grid, st);
}

}  // namespace vita

using namespace vita;

extern "C" int vita_attention_fwd(const void* q, const void* k, const void* v, void* o, const int64_t* q_strides,
                                  const int64_t* k_strides, const int64_t* v_strides, const int64_t* o_strides,
                                  int64_t B, int64_t n_q_heads, int64_t n_kv_heads, int64_t Sq, int64_t Skv,
                                  int64_t d_qk, int64_t d_v, const int32_t* kv_lens, int causal, int64_t q_pos0,
                                  float scale, void* stream) {
    VITA_REQUIRE(n_kv_heads > 0 && n_q_heads % n_kv_heads == 0, "n_q_heads must be a multiple of n_kv_heads");
    VITA_REQUIRE(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(o), "q/k/v/o must be 16-byte aligned");
    for (int i = 0; i < 3; ++i)
        VITA_REQUIRE(q_strides[i] % 8 == 0 && k_strides[i] % 8 == 0 && v_strides[i] % 8 == 0 && o_strides[i] % 8 == 0,
                     "strides must keep 16-byte row alignment");
    VITA_REQUIRE(scale > 0.0f, "softmax scale must be positive");
    VITA_REQUIRE(B <= 65535 && n_q_heads <= 65535, "batch / head count exceed the grid limits");
    if (B == 0 || Sq == 0) return VITA_OK;
    VITA_REQUIRE(Skv > 0, "Skv must be positive");
    VITA_REQUIRE(q_pos0 >= 0 && (causal || q_pos0 == 0), "q_pos0 is the causal offset of query row 0 (>= 0)");
    FaParams p{};
    p.o = static_cast<__nv_bfloat16*>(o);
    p.o_bs = o_strides[0]; p.o_ts = o_strides[1]; p.o_hs = o_strides[2];
    p.group = static_cast<int>(n_q_heads / n_kv_heads);
    p.Sq = static_cast<int>(Sq);
    p.Skv = static_cast<int>(Skv);
    p.kv_lens = kv_lens;
    p.causal = causal;
    p.q_pos0 = static_cast<int>(q_pos0);
    p.scale_log2 = scale * 1.4426950408889634f;
    auto st = static_cast<cudaStream_t>(stream);
    const int Bi = static_cast<int>(B), Hq = static_cast<int>(n_q_heads), Hkv = static_cast<int>(n_kv_heads);
    if (d_qk == 128 && d_v == 128)
        return flash_tc_dispatch<128, 128>(q, k, v, q_strides, k_strides, v_strides, p, Bi, Hq, Hkv, st);
    if (d_qk == 64 && d_v == 64)
        return flash_tc_dispatch<64, 64>(q, k, v, q_strides, k_strides, v_strides, p, Bi, Hq, Hkv, st);
    if (d_qk == 128 && d_v == 64)
        return flash_tc_dispatch<128, 64>(q, k, v, q_strides, k_strides, v_strides, p, Bi, Hq, Hkv, st);
    set_last_error("vita_attention_fwd: unsupported head dims (supported: 128/128, 64/64, 128/64)");
    return VITA_ERR_INVALID;
}

extern "C" int vita_attention_prefill_paged(const void* q, int64_t q_token_stride, const void* k_cache,
                                            const void* v_cache, int64_t n_slots, const int32_t* block_table,
                                            int64_t bt_stride, const int32_t* query_start_loc, const int32_t* ctx_lens,
                                            const int32_t* tiles, int64_t n_tiles, void* out, int64_t o_token_stride,
                                            int64_t T, int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim,
                                            int64_t page_size, float scale, void* stream) {
    VITA_REQUIRE(head_dim == 128, "head_dim must be 128 (Mixtral GQA)");
    VITA_REQUIRE(page_size == 16 || page_size == 32 || page_size == 64 || page_size == 128,
                 "page_size must be 16, 32, 64 or 128");
    VITA_REQUIRE(n_kv_heads > 0 && n_q_heads % n_kv_heads == 0, "n_q_heads must be a multiple of n_kv_heads");
    VITA_REQUIRE(n_q_heads <= 65535, "head count exceeds the grid limit");
    VITA_REQUIRE(aligned16(q) && aligned16(k_cache) && aligned16(v_cache) && aligned16(out),
                 "q / caches / out must be 16-byte aligned");
    VITA_REQUIRE(q_token_stride % 8 == 0 && o_token_stride % 8 == 0 && q_token_stride >= n_q_heads * head_dim &&
                     o_token_stride >= n_q_heads * head_dim,
                 "token strides must cover the q heads and keep 16-byte row alignment");
    VITA_REQUIRE(scale > 0.0f, "softmax scale must be positive");
    VITA_REQUIRE(n_tiles >= 0 && n_tiles <= 0x7fffffff && T >= 0 && n_slots > 0 && bt_stride > 0,
                 "bad tile count, token count, slot count or block-table stride");
    if (n_tiles == 0 || T == 0) return VITA_OK;
    VITA_REQUIRE(block_table && query_start_loc && ctx_lens && tiles, "null block_table / query_start_loc / ctx_lens / tiles");
    FaParams p{};
    p.o = static_cast<__nv_bfloat16*>(out);
    p.o_ts = o_token_stride;
    p.o_hs = head_dim;
    p.group = static_cast<int>(n_q_heads / n_kv_heads);
    p.causal = 1;
    p.scale_log2 = scale * 1.4426950408889634f;
    p.poly_chunks = option("fa_poly");
    p.tiles = tiles;
    p.qsl = query_start_loc;
    p.ctx = ctx_lens;
    p.block_table = block_table;
    p.bt_stride = static_cast<int>(bt_stride);
    p.page_shift = page_size == 16 ? 4 : page_size == 32 ? 5 : page_size == 64 ? 6 : 7;
    CUtensorMap tmQ, tmK, tmV;
    int rc = make_qkv_map(&tmQ, q, 128, T, n_q_heads, 1, q_token_stride, head_dim, 0);
    if (rc) return rc;
    const uint64_t dims[3] = {128, static_cast<uint64_t>(n_kv_heads), static_cast<uint64_t>(n_slots)};
    const uint64_t strides[2] = {128 * 2, static_cast<uint64_t>(n_kv_heads) * 128 * 2};
    const uint32_t box[3] = {64, 1, static_cast<uint32_t>(page_size)};
    rc = make_tensor_map_bf16(&tmK, k_cache, 3, dims, strides, box, true);
    if (rc) return rc;
    rc = make_tensor_map_bf16(&tmV, v_cache, 3, dims, strides, box, true);
    if (rc) return rc;
    const dim3 grid(static_cast<unsigned>(n_tiles), static_cast<unsigned>(n_q_heads), 1);
    return launch_flash_tc<128, 128, true>(tmQ, tmK, tmV, p, grid, static_cast<cudaStream_t>(stream));
}
