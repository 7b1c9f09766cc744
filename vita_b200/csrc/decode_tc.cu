// Decode-step linears on the tensor cores ("swap-AB" GEMV, stream-K):  y[rows] = W[rows, K] . x[K].
//
// A SIMT GEMV moves every byte at full TMA rate but needs ~80 issue slots per 32 bytes of weights for bf16->fp32
// unpacking and FMAs.  Here the weight tile is the *M* operand of wgmma (128 rows x 64 k = two m64n16k16 row halves,
// TMA-loaded with the 128B swizzle) and the activation vector is row 0 of a 16 x 64 *N* operand tile, so the CUDA
// cores only run the per-row epilogue:
//   warp 0  TMA producer: streams W tiles into an smem ring (starts before the PDL dependency resolves: weights
//           never depend on the previous kernel, except for the expert ids which it waits for); once its last tile is
//           issued it triggers the dependent launch, so the next kernel of the chain sets up and fills its own ring
//           while this one drains and reduces;
//   warps 1-2  idle (they only take part in the wide router prologue);
//   warp 3  x-tile writer: copies 128 B of the (bf16, smem-resident) activation vector into row 0 of the stage's
//           N tile (rows 1..15 stay zero), fence.proxy.async, arrives on the stage barrier;
//   warps 4-7  one warpgroup: prologue (RMSNorm / router / residual prefetch), then per ring stage 2 x 4 wgmma
//           (M=64, N=16, K=16) per part into register accumulators, and the fused per-row epilogue (column 0 of the
//           accumulator fragment goes through shared memory so that thread i owns row i of the block).
// Work is cut stream-K style: the (row-block, k-block) units are split evenly and contiguously over the CTAs, so all
// SMs stream the same number of bytes whatever the matrix shape.  A row block whose K range spans several CTAs
// is combined through per-contributor slots of 64-bit {partial, tag} words: no fence and no atomic, the CTA that ends
// on the row block polls the others' words (collecting early arrivals while its own MMAs still run), adds them in
// slot order (deterministic), clears the tags and runs the epilogue.
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"
#include "kv_fp8.cuh"

namespace vita {

constexpr int TC_XN = 16;                 // N of the MMA (activation tile rows; row 0 carries x)
constexpr int TC_A_BYTES = 128 * 64 * 2;  // one weight tile
constexpr int TC_X_BYTES = TC_XN * 64 * 2;
constexpr int TC_SLOTS = 8;               // max contributors per row block
constexpr int TC_THREADS = 256;

__device__ __forceinline__ void epi_barrier() { asm volatile("bar.sync 1, 128;" ::: "memory"); }
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// sum over the 128 epilogue threads (warps 4..7); scratch >= 4 floats
__device__ __forceinline__ float epi_sum(float v, float* scratch) {
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) scratch[(threadIdx.x >> 5) - 4] = v;
    epi_barrier();
    const float t = scratch[0] + scratch[1] + scratch[2] + scratch[3];
    epi_barrier();
    return t;
}

struct TcSmem {
    __nv_bfloat16* xs;  // compact activation vector(s)
    float* scratch;     // 64 floats
    float* prep;        // 256 floats
    int* misc;          // 8 ints
    float* pair;        // 128 floats (row exchange inside a row block)
    uint64_t* x_ready;  // arrives once the activation vector is in smem (ops that bulk-copy x arm it themselves)
};

// bf16(rmsnorm(h) * w) -> xs.  All global loads are issued up front (each of the 128 threads owns up to 4 chunks of
// 8 elements, kept in registers between the two passes); larger K falls back to a strided loop.
__device__ __forceinline__ void tc_load_x_rmsnorm(const __nv_bfloat16* h, const __nv_bfloat16* w, __nv_bfloat16* xs,
                                                  int K, float eps, float* scratch) {
    const int t = threadIdx.x - 128;
    constexpr int MAXV = 4;
    if (K <= 128 * 8 * MAXV) {
        uint4 hv[MAXV], gv[MAXV];
#pragma unroll
        for (int j = 0; j < MAXV; ++j) {
            const int i = (t + j * 128) * 8;
            if (i < K) {
                hv[j] = *reinterpret_cast<const uint4*>(h + i);
                gv[j] = __ldg(reinterpret_cast<const uint4*>(w + i));
            }
        }
        float ss = 0.0f;
#pragma unroll
        for (int j = 0; j < MAXV; ++j) {
            if ((t + j * 128) * 8 < K) {
                const uint32_t a[4] = {hv[j].x, hv[j].y, hv[j].z, hv[j].w};
#pragma unroll
                for (int e = 0; e < 4; ++e) ss += bf16_lo(a[e]) * bf16_lo(a[e]) + bf16_hi(a[e]) * bf16_hi(a[e]);
            }
        }
        const float inv = rsqrtf(epi_sum(ss, scratch) / static_cast<float>(K) + eps);
#pragma unroll
        for (int j = 0; j < MAXV; ++j) {
            const int i = (t + j * 128) * 8;
            if (i < K) {
                const uint32_t a[4] = {hv[j].x, hv[j].y, hv[j].z, hv[j].w}, gg[4] = {gv[j].x, gv[j].y, gv[j].z, gv[j].w};
                uint4 o;
                uint32_t* op = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    op[e] = pack_bf16(bf16_lo(a[e]) * inv * bf16_lo(gg[e]), bf16_hi(a[e]) * inv * bf16_hi(gg[e]));
                *reinterpret_cast<uint4*>(xs + i) = o;
            }
        }
        return;
    }
    float ss = 0.0f;
    for (int i = t * 8; i < K; i += 128 * 8) {
        const uint4 v = *reinterpret_cast<const uint4*>(h + i);
        const uint32_t a[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) ss += bf16_lo(a[e]) * bf16_lo(a[e]) + bf16_hi(a[e]) * bf16_hi(a[e]);
    }
    const float inv = rsqrtf(epi_sum(ss, scratch) / static_cast<float>(K) + eps);
    for (int i = t * 8; i < K; i += 128 * 8) {
        const uint4 v = *reinterpret_cast<const uint4*>(h + i);
        const uint4 g = __ldg(reinterpret_cast<const uint4*>(w + i));
        const uint32_t a[4] = {v.x, v.y, v.z, v.w}, gg[4] = {g.x, g.y, g.z, g.w};
        uint4 o;
        uint32_t* op = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int e = 0; e < 4; ++e)
            op[e] = pack_bf16(bf16_lo(a[e]) * inv * bf16_lo(gg[e]), bf16_hi(a[e]) * inv * bf16_hi(gg[e]));
        *reinterpret_cast<uint4*>(xs + i) = o;
    }
}
// RMSNorm statistics + the 8 router logits of one token, by the 128 epilogue threads (fp32 throughout, soft-max and
// top-2 as the reference's MixtralSparseMoeBlock).  Every caller gets the same bits: same loads, same summation order.
struct TcRoute {
    int e0, e1;
    float w0, w1;   // renormalised top-2 weights
    float inv;      // 1 / rms(h)
};
// per-thread partial sums over this thread's share of the K axis: [0] = sum h^2, [1 + e] = sum h * norm_w * gate_w[e]
__device__ __forceinline__ void tc_route_partials(const __nv_bfloat16* hr, const __nv_bfloat16* norm_w,
                                                  const __nv_bfloat16* gate_w, int K, int tid, int nthreads,
                                                  float (&part)[9]) {
#pragma unroll
    for (int e = 0; e < 9; ++e) part[e] = 0.0f;
#pragma unroll 2
    for (int i = tid * 8; i < K; i += nthreads * 8) {
        const uint4 hv = *reinterpret_cast<const uint4*>(hr + i);
        const uint4 g = __ldg(reinterpret_cast<const uint4*>(norm_w + i));
        uint4 ge[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) ge[e] = __ldg(reinterpret_cast<const uint4*>(gate_w + static_cast<long long>(e) * K + i));
        const uint32_t a[4] = {hv.x, hv.y, hv.z, hv.w}, gg[4] = {g.x, g.y, g.z, g.w};
        float xw[8];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float lo = bf16_lo(a[q]), hi = bf16_hi(a[q]);
            part[0] += lo * lo + hi * hi;
            xw[2 * q] = lo * bf16_lo(gg[q]);
            xw[2 * q + 1] = hi * bf16_hi(gg[q]);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            const uint32_t w[4] = {ge[e].x, ge[e].y, ge[e].z, ge[e].w};
#pragma unroll
            for (int q = 0; q < 4; ++q) part[1 + e] += xw[2 * q] * bf16_lo(w[q]) + xw[2 * q + 1] * bf16_hi(w[q]);
        }
    }
#pragma unroll
    for (int e = 0; e < 9; ++e) part[e] = warp_sum(part[e]);
}
// soft-max over the 8 logits, top-2, renormalised weights (fp32; MixtralSparseMoeBlock order of operations)
__device__ __forceinline__ TcRoute tc_route_finish(const float (&tot)[9], int K, float eps) {
    TcRoute r;
    r.inv = rsqrtf(tot[0] / static_cast<float>(K) + eps);
    float p[8], m = -INFINITY, sum = 0.0f;
#pragma unroll
    for (int e = 0; e < 8; ++e) { p[e] = tot[1 + e] * r.inv; m = fmaxf(m, p[e]); }
#pragma unroll
    for (int e = 0; e < 8; ++e) { p[e] = expf(p[e] - m); sum += p[e]; }
    int e0 = 0;
#pragma unroll
    for (int e = 1; e < 8; ++e) if (p[e] > p[e0]) e0 = e;
    int e1 = (e0 == 0) ? 1 : 0;
#pragma unroll
    for (int e = 0; e < 8; ++e) if (e != e0 && p[e] > p[e1]) e1 = e;
    float pe0 = 0.0f, pe1 = 0.0f;
#pragma unroll
    for (int e = 0; e < 8; ++e) { if (e == e0) pe0 = p[e]; if (e == e1) pe1 = p[e]; }
    const float p0 = pe0 / sum, p1 = pe1 / sum, den = p0 + p1;
    r.e0 = e0; r.e1 = e1; r.w0 = p0 / den; r.w1 = p1 / den;
    return r;
}
// narrow form: the 128 epilogue threads do everything
__device__ __forceinline__ TcRoute tc_route(const __nv_bfloat16* hr, const __nv_bfloat16* norm_w,
                                            const __nv_bfloat16* gate_w, int K, float eps, float* prep) {
    float part[9];
    tc_route_partials(hr, norm_w, gate_w, K, threadIdx.x - 128, 128, part);
    const int w4 = (threadIdx.x >> 5) - 4;
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int e = 0; e < 9; ++e) prep[w4 * 9 + e] = part[e];
    epi_barrier();
    float tot[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) tot[e] = prep[e] + prep[9 + e] + prep[18 + e] + prep[27 + e];
    epi_barrier();   // prep may be reused by the caller
    return tc_route_finish(tot, K, eps);
}
// Pull constant tensors into L2 while the kernel is still waiting for its predecessor (CTA-sharded, 128 B lines).
__device__ __forceinline__ void tc_prefetch_l2(const void* base, long long bytes) {
    const long long lines = (bytes + 127) / 128;
    for (long long l = static_cast<long long>(blockIdx.x) * 128 + (threadIdx.x - 128); l < lines;
         l += static_cast<long long>(gridDim.x) * 128)
        asm volatile("prefetch.global.L2 [%0];" ::"l"(static_cast<const char*>(base) + l * 128));
}

// Plain copy of an activation vector: one TMA 1-D bulk copy that completes straight onto the x_ready barrier.
__device__ __forceinline__ void tc_bulk_x(const __nv_bfloat16* src, __nv_bfloat16* xs, int n, uint64_t* bar) {
    if (threadIdx.x == 128) {
        mbar_arrive_expect_tx(bar, static_cast<uint32_t>(n) * 2);
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     ::"r"(smem_u32(xs)), "l"(src), "r"(static_cast<uint32_t>(n) * 2), "r"(smem_u32(bar))
                     : "memory");
    }
}

struct TcFinish {
    float best;
    int best_idx;
};

// PARTS: weight tiles per unit (1, or 2 for gate|up and for the two experts of the down projection).
// XPARTS: distinct activation vectors (2 only for the down projection).
template <class Op>
#ifndef TC_MIN_BLOCKS
#define TC_MIN_BLOCKS 1
#endif
// Register cap: a kernel and its successor in a programmatic-launch chain share an SM (2 x 256 threads), and the
// register file only holds both when their sum stays clearly below 256 per thread pair.
#ifdef TC_NO_MAXNREG
__global__ void __launch_bounds__(TC_THREADS, 1)
#else
__global__ void __maxnreg__(Op::kMaxRegs)
#endif
tc_gemv_kernel(const __grid_constant__ CUtensorMap tmW, const Op op, unsigned long long* __restrict__ g_scratch,
               const int l2_ahead, const int flags, const ChainArgsDev chain VITA_TRACE_PARAM) {
    constexpr int PARTS = Op::kParts, XPARTS = Op::kXParts, STAGES = Op::kStages;
    constexpr int STAGE_A = PARTS * TC_A_BYTES;
    constexpr int STAGE_X = XPARTS * TC_X_BYTES;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;
    uint8_t* sX = sA + STAGES * STAGE_A;
    __nv_bfloat16* xs = reinterpret_cast<__nv_bfloat16*>(sX + STAGES * STAGE_X);
    uint8_t* tail = reinterpret_cast<uint8_t*>(xs) + ((op.x_elems() * 2 + 127) / 128) * 128;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(tail);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* x_ready = empty_bar + STAGES;
    float* scratch = reinterpret_cast<float*>(x_ready + 1);
    float* prep = scratch + 64;
    float* pair = prep + 256;
    float* rows = pair + 128;          // [PARTS][128]: accumulator column 0, fragment layout -> one row per thread
    int* misc = reinterpret_cast<int*>(rows + 2 * 128);
    TcSmem sm{xs, scratch, prep, misc, pair, x_ready};

    const int b = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#ifdef VITA_TRACE
    if (blockIdx.y != 0 || (blockIdx.x != 0 && blockIdx.x != gridDim.x - 1)) trace = nullptr;
    if (trace && blockIdx.x != 0) trace += 16;         // last CTA: same events in words 17..24
    if (threadIdx.x == 0) { VITA_STAMP(1); if (blockIdx.x == 0) VITA_STAMP_SET(0, static_cast<unsigned long long>(Op::kId)); }
#endif
    const int K = op.K;
    const int n_kb = K >> 6;
    const int n_rb = op.num_row_blocks();
    const long long U = static_cast<long long>(n_rb) * n_kb;
    const int G = gridDim.x;
    const long long u0 = U * blockIdx.x / G, u1 = U * (blockIdx.x + 1) / G;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmW);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 2);   // TMA producer (expect_tx) + x-tile writer
            mbar_init(&empty_bar[i], 4);  // the MMA warps, once their wgmma group has read the stage
        }
        mbar_init(x_ready, 1);
        fence_barrier_init();
    }
    // N-operand tiles: rows 1..15 stay zero for the whole kernel, row 0 is rewritten per stage
    for (int i = threadIdx.x; i < STAGES * STAGE_X / 16; i += TC_THREADS) reinterpret_cast<uint4*>(sX)[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();
    __syncthreads();
    if (threadIdx.x == 0) VITA_STAMP(2);

    // router-carrying op, wide form: every thread of the CTA takes part in the router dot products before the roles
    // split up (the producer cannot start without the expert ids anyway)
    const bool wide = Op::kHasRoute && (flags & 8) != 0;
    if (wide) {
        if (warp >= 4) op.pre_wait(b, sm, (flags & 1) != 0);
        if (threadIdx.x == 0) chain_wait(chain);
        __syncthreads();
        op.wide_partials(b, sm);
        __syncthreads();
    }

    if (warp == 0) {
        if (lane == 0) {
            // ------------------------------------------------------------ TMA producer (weights)
            if (Op::kRowsNeedPrologue) mbar_wait(x_ready, 0, 21);      // expert ids computed by this CTA's prologue
            else if (Op::kRowsNeedUpstream) {
                // expert ids written by the previous kernel: either published early as one tagged word (then the
                // weight rows stream while the predecessor is still running) or read after the dependency wait
                if (!op.rows_from_route_word(b, sm)) {
                    chain_wait(chain);
                    op.rows_from_upstream(b, sm);
                }
            }
            int stage = 0;
            uint32_t phase = 0;
            // With programmatic dependent launch the next kernel of the chain may take the free half of the SM and fill
            // its ring while this CTA drains and reduces: trigger once all but `lead` of this CTA's loads are issued.
            // Waiting first (long since satisfied) makes the chain transitive: when kernel N+1 starts, N-1 is complete.
            // (an op that publishes its routing early triggers right away: its successor only needs the expert ids to
            // start streaming, and those are out since this CTA's prologue)
            const long long lead = op.trigger_at_start() ? (1ll << 60) : static_cast<long long>(flags >> 8);
            bool triggered = false;
            for (long long u = u0; u < u1; ++u) {
                if (!triggered && u1 - u <= lead) {
                    if ((flags & 2) && u > u0) chain_wait(chain);
                    pdl_launch_dependents();
                    triggered = true;
                }
                const int rb = static_cast<int>(u / n_kb), kb = static_cast<int>(u % n_kb);
                // ring full for the first time: nothing can drain it before the predecessor has completed (the
                // activations come from it), so park on the hardware dependency instead of spinning on the barrier
                // next to the predecessor's own producer / MMA threads
                if ((flags & 4) && u - u0 == STAGES) chain_wait(chain);
                mbar_wait(&empty_bar[stage], phase ^ 1, 22);
                mbar_arrive_expect_tx(&full_bar[stage], STAGE_A);
#pragma unroll
                for (int p = 0; p < PARTS; ++p)
                    tma_load_2d(sA + stage * STAGE_A + p * TC_A_BYTES, &tmW, &full_bar[stage], kb * 64,
                                op.a_row(b, rb, p, sm));
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
                if (l2_ahead > 0 && u - u0 == STAGES - 1) {
                    // the ring is full and (under programmatic launch) the predecessor is still reducing: HBM would
                    // idle, so pull the next tiles of this CTA into L2
                    for (long long v = u + 1; v < u1 && v <= u + l2_ahead; ++v) {
                        const int rb2 = static_cast<int>(v / n_kb), kb2 = static_cast<int>(v % n_kb);
#pragma unroll
                        for (int p = 0; p < PARTS; ++p) tma_prefetch_l2_2d(&tmW, kb2 * 64, op.a_row(b, rb2, p, sm));
                    }
                }
            }
            if (!triggered) {
                if (flags & 2) chain_wait(chain);
                pdl_launch_dependents();
            }
            VITA_STAMP(6);
        }
    } else if (warp == 3) {
        // ---------------------------------------------------------------- x-tile writer
        // per stage: copy 128 B of the activation vector into row 0 of the N tile
        int stage = 0;
        uint32_t phase = 0;
        if constexpr (Op::kXFromGlobal) {
            // the vectors stay in L2; this warp keeps the chunks of the next LOOK units in registers
            constexpr int LOOK = 4;
            if (lane == 0) chain_wait(chain);
            __syncwarp();
            const __nv_bfloat16* xg = op.x_global(b);
            const int px = lane >> 3, c = lane & 7;
            const bool active = lane < 8 * XPARTS;
            uint4 nxt[LOOK];
#pragma unroll
            for (int j = 0; j < LOOK; ++j)
                if (active && u0 + j < u1)
                    nxt[j] = *reinterpret_cast<const uint4*>(xg + static_cast<long long>(px) * K + ((u0 + j) % n_kb) * 64 + c * 8);
            for (long long u = u0; u < u1; u += LOOK) {
#pragma unroll
                for (int j = 0; j < LOOK; ++j) {
                    if (u + j < u1) {
                        mbar_wait(&empty_bar[stage], phase ^ 1, 26);
                        if (active) {
                            *reinterpret_cast<uint4*>(sX + stage * STAGE_X + px * TC_X_BYTES + c * 16) = nxt[j];
                            if (u + j + LOOK < u1)
                                nxt[j] = *reinterpret_cast<const uint4*>(xg + static_cast<long long>(px) * K +
                                                                         ((u + j + LOOK) % n_kb) * 64 + c * 8);
                        }
                        fence_proxy_async_smem();
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&full_bar[stage]);
                        if (++stage == STAGES) { stage = 0; phase ^= 1; }
                    }
                }
            }
        } else {
            if ((flags & 4) && lane == 0) chain_wait(chain);
            __syncwarp();
            mbar_wait(x_ready, 0, 25);
            for (long long u = u0; u < u1; ++u) {
                const int kb = static_cast<int>(u % n_kb);
                mbar_wait(&empty_bar[stage], phase ^ 1, 26);
                if (lane < 8 * XPARTS) {
                    const int px = lane >> 3, c = lane & 7;
                    *reinterpret_cast<uint4*>(sX + stage * STAGE_X + px * TC_X_BYTES + c * 16) =
                        *reinterpret_cast<const uint4*>(xs + static_cast<long long>(px) * K + kb * 64 + c * 8);
                }
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) mbar_arrive(&full_bar[stage]);
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
        }
    }
    if (warp < 4) return;   // the MMA warpgroup continues at the top level: wgmma inside a role branch is serialised by ptxas
    {
        // ---------------------------------------------------------------- prologue + MMA + epilogue (128 threads)
        if (!wide) op.pre_wait(b, sm, (flags & 1) != 0);   // constants only: L2 prefetch ahead of the dependency wait
        if (threadIdx.x == 128) chain_wait(chain);   // activations come from the previous kernel
        epi_barrier();
        if (threadIdx.x == 128) VITA_STAMP(3);
        op.prologue(b, sm, wide);
        epi_barrier();
        if (!Op::kBulkX && threadIdx.x == 128) mbar_arrive(x_ready);
        if (threadIdx.x == 128) VITA_STAMP(4);

        const int quad = warp - 4;
        const int row = quad * 32 + lane;
        const uint32_t sA_addr = smem_u32(sA), sX_addr = smem_u32(sX);
        int stage = 0;
        uint32_t phase = 0;
        TcFinish st{-INFINITY, 0x7fffffff};
        unsigned long long* my_scratch = g_scratch + static_cast<long long>(b) * n_rb * TC_SLOTS * PARTS * 128;
        long long u = u0;
        while (u < u1) {
            const int rb = static_cast<int>(u / n_kb);
            const long long rb_begin = static_cast<long long>(rb) * n_kb, rb_end = rb_begin + n_kb;
            const long long seg_end = rb_end < u1 ? rb_end : u1;
            // A K-partial segment is reduced through global slots in a fixed order (slot = contributor index).  Every
            // partial travels as ONE 64-bit word {value, tag}, so neither fences nor tickets are needed: the contributor
            // with the lowest index -- the CTA that ends on this row block, its neighbours did their part of it first --
            // reduces, and clears the tags for the next launch.  While its own MMAs are still running it already
            // collects whatever the others have published.
            const bool partial = (u != rb_begin || seg_end != rb_end);
            int slot = 0, n_contrib = 1;
            unsigned long long* base64 = nullptr;
            uint32_t have = 0;
            float oth[PARTS][TC_SLOTS];
            if (partial) {
                int c_first = blockIdx.x;
                while (c_first > 0 && U * c_first / G > rb_begin) --c_first;
                int c_last = blockIdx.x;
                while (c_last + 1 < G && U * (c_last + 1) / G < rb_end) ++c_last;
                slot = blockIdx.x - c_first;
                n_contrib = c_last - c_first + 1;
                base64 = my_scratch + static_cast<long long>(rb) * TC_SLOTS * PARTS * 128;
                if (slot == 0) {
#pragma unroll
                    for (int p = 0; p < PARTS; ++p) {
                        unsigned long long w[TC_SLOTS];
#pragma unroll
                        for (int q = 1; q < TC_SLOTS; ++q)
                            if (q < n_contrib) w[q] = ld_relaxed_u64(base64 + (q * PARTS + p) * 128 + row);
#pragma unroll
                        for (int q = 1; q < TC_SLOTS; ++q)
                            if (q < n_contrib && (w[q] >> 32) != 0) {
                                oth[p][q] = __uint_as_float(static_cast<uint32_t>(w[q]));
                                have |= 1u << (p * TC_SLOTS + q);
                            }
                    }
                }
            }
            // ---- the segment's MMAs: d[p][mh] is rows [64 mh, 64 mh + 64) of part p; one wgmma group in flight, a
            // ring stage goes back to the producer and the x-tile writer once the group that read it has completed
            float d[PARTS][2][TC_XN / 2];
            int prev = -1;
            for (long long w = u; w < seg_end; ++w) {
                mbar_wait(&full_bar[stage], phase, 24);
                if (threadIdx.x == 128 && w == u0) VITA_STAMP(5);
#pragma unroll
                for (int p = 0; p < PARTS; ++p) { wgmma_acc_fence(d[p][0]); wgmma_acc_fence(d[p][1]); }
                wgmma_fence();
#pragma unroll
                for (int p = 0; p < PARTS; ++p) {
                    const uint64_t dx = wgmma_desc_k_sw128(sX_addr + stage * STAGE_X + (XPARTS > 1 ? p : 0) * TC_X_BYTES);
#pragma unroll
                    for (int mh = 0; mh < 2; ++mh) {
                        const uint64_t da = wgmma_desc_k_sw128(sA_addr + stage * STAGE_A + p * TC_A_BYTES + mh * (64 * 128));
#pragma unroll
                        for (int k = 0; k < 4; ++k)
                            wgmma_ss<TC_XN>(d[p][mh], da + 2 * k, dx + 2 * k, (w > u || k > 0) ? 1 : 0);
                    }
                }
                wgmma_commit();
#pragma unroll
                for (int p = 0; p < PARTS; ++p) { wgmma_acc_fence(d[p][0]); wgmma_acc_fence(d[p][1]); }
                wgmma_wait<1>();   // unconditional (a no-op for the first stage): warpgroup-wide, must not sit in a branch
                if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
                prev = stage;
                if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int p = 0; p < PARTS; ++p) { wgmma_acc_fence(d[p][0]); wgmma_acc_fence(d[p][1]); }
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
            if (threadIdx.x == 128 && seg_end == u1) VITA_STAMP(7);
            // column 0 of the fragment (lanes 0, 4, ..: rows 16 quad + lane / 4 and + 8 of each half) -> thread-per-row.
            // (every lane reads its accumulators; only the store is conditional)
            float c0[PARTS][2][2];
#pragma unroll
            for (int p = 0; p < PARTS; ++p)
#pragma unroll
                for (int mh = 0; mh < 2; ++mh) { c0[p][mh][0] = d[p][mh][0]; c0[p][mh][1] = d[p][mh][2]; }
            if ((lane & 3) == 0) {
#pragma unroll
                for (int p = 0; p < PARTS; ++p)
#pragma unroll
                    for (int mh = 0; mh < 2; ++mh) {
                        rows[p * 128 + mh * 64 + quad * 16 + (lane >> 2)] = c0[p][mh][0];
                        rows[p * 128 + mh * 64 + quad * 16 + (lane >> 2) + 8] = c0[p][mh][1];
                    }
            }
            epi_barrier();
            float v[PARTS];
#pragma unroll
            for (int p = 0; p < PARTS; ++p) v[p] = rows[p * 128 + row];
            epi_barrier();

            bool do_finish = true;
            if (partial && slot != 0) {
#pragma unroll
                for (int p = 0; p < PARTS; ++p)
                    st_relaxed_u64(base64 + (slot * PARTS + p) * 128 + row,
                                   (1ull << 32) | static_cast<unsigned long long>(__float_as_uint(v[p])));
                do_finish = false;
            } else if (partial) {
#pragma unroll
                for (int p = 0; p < PARTS; ++p)
#pragma unroll
                    for (int q = 1; q < TC_SLOTS; ++q) {
                        if (q < n_contrib) {
                            unsigned long long* addr = base64 + (q * PARTS + p) * 128 + row;
                            if (!(have & (1u << (p * TC_SLOTS + q)))) {
                                unsigned long long w = ld_relaxed_u64(addr);
                                for (uint32_t spin = 0; (w >> 32) == 0; ++spin) {
                                    if (spin > (1u << 24)) __trap();   // a contributor never published (seconds, not minutes)
                                    w = ld_relaxed_u64(addr);
                                }
                                oth[p][q] = __uint_as_float(static_cast<uint32_t>(w));
                            }
                            st_relaxed_u64(addr, 0ull);   // consumed: the slot is free for the next launch
                        }
                    }
                // fixed order: own value (slot 0) first, then the slots ascending
#pragma unroll
                for (int p = 0; p < PARTS; ++p) {
                    float s = 0.0f + v[p];
#pragma unroll
                    for (int q = 1; q < TC_SLOTS; ++q)
                        if (q < n_contrib) s += oth[p][q];
                    v[p] = s;
                }
            }
            if (do_finish) op.finish(b, rb, row, v, st, sm);
            u = seg_end;
        }
        op.finalize(b, st);
        epi_barrier();                                   // every epilogue thread's stores are issued
        if (threadIdx.x == 128) chain_arrive(chain);     // (the other warps of the CTA never write global memory)
        if (threadIdx.x == 128) VITA_STAMP(8);
    }

}

// ------------------------------------------------------------------------------------------------ ops
struct TcQkvOp {
    __device__ bool rows_from_route_word(int, const TcSmem&) const { return false; }
    __device__ void rows_from_upstream(int, const TcSmem&) const {}
    __device__ bool trigger_at_start() const { return false; }
    static constexpr int kMaxRegs = 128;
    static constexpr int kId = 1;
    __device__ const __nv_bfloat16* x_global(int) const { return nullptr; }
    static constexpr bool kXFromGlobal = false;
    static constexpr bool kBulkX = false;
    static constexpr int kParts = 1, kXParts = 1, kStages = 5;
    static constexpr bool kHasRoute = false;
    static constexpr bool kRowsNeedPrologue = false, kRowsNeedUpstream = false;
    const __nv_bfloat16* h;
    const __nv_bfloat16* norm_w;
    const float* cos_sin;
    const int* cur_pos;
    const int* block_table;
    __nv_bfloat16* q_out;
    __nv_bfloat16* k_cache;
    __nv_bfloat16* v_cache;
    int K, n_q, n_kv, page_size, max_pages;
    float eps;

    __device__ int x_elems() const { return K; }
    __device__ int num_row_blocks() const { return n_q + 2 * n_kv; }   // one 128-row block per head
    __device__ int a_row(int, int rb, int, const TcSmem&) const { return rb * 128; }
    __device__ void pre_wait(int, const TcSmem&, bool on) const { if (on) tc_prefetch_l2(norm_w, K * 2ll); }
    __device__ void wide_partials(int, const TcSmem&) const {}
    __device__ void prologue(int b, const TcSmem& sm, bool) const {
        const int t = threadIdx.x - 128;
        const int pos = cur_pos[b];
        sm.prep[t] = cos_sin[static_cast<long long>(pos) * 128 + t];
        if (t == 0) {
            const int page = block_table[static_cast<long long>(b) * max_pages + pos / page_size];
            sm.misc[0] = page * page_size + pos % page_size;
        }
        tc_load_x_rmsnorm(h + static_cast<long long>(b) * K, norm_w, sm.xs, K, eps, sm.scratch);
    }
    // the output row of head block rb: projections are rounded to bf16 before RoPE, as the GEMM path (and the
    // reference) does; q and k heads are rotated
    __device__ __forceinline__ float rope_row(int rb, int row, const float (&v)[1], const TcSmem& sm) const {
        const float x = __bfloat162float(__float2bfloat16(v[0]));
        float o = x;
        if (rb < n_q + n_kv) {   // rotate-half RoPE: partner row is row ^ 64 of the same head
            sm.pair[row] = x;
            epi_barrier();
            const float partner = sm.pair[row ^ 64];
            const int j = row & 63;
            const float c = sm.prep[j], s = sm.prep[64 + j];
            o = (row < 64) ? x * c - partner * s : x * c + partner * s;
            epi_barrier();
        }
        return o;
    }
    __device__ void finish(int b, int rb, int row, const float (&v)[1], TcFinish&, const TcSmem& sm) const {
        const float o = rope_row(rb, row, v, sm);
        if (rb < n_q) {
            q_out[(static_cast<long long>(b) * n_q + rb) * 128 + row] = __float2bfloat16(o);
        } else {
            const long long slot = sm.misc[0];
            const bool is_k = rb < n_q + n_kv;
            const int kvh = is_k ? rb - n_q : rb - n_q - n_kv;
            ((is_k ? k_cache : v_cache) + (slot * n_kv + kvh) * 128)[row] = __float2bfloat16(o);
        }
    }
    __device__ void finalize(int, TcFinish&) const {}
};

// the same over e4m3 caches (kv_fp8.cuh): k_cache / v_cache hold bytes, each row stored as
// e4m3_rn_satfinite(bf16(o) / scale), q unchanged
struct TcQkvFp8Op : TcQkvOp {
    float k_scale, v_scale;

    __device__ void finish(int b, int rb, int row, const float (&v)[1], TcFinish&, const TcSmem& sm) const {
        const float o = rope_row(rb, row, v, sm);
        if (rb < n_q) {
            q_out[(static_cast<long long>(b) * n_q + rb) * 128 + row] = __float2bfloat16(o);
        } else {
            const long long slot = sm.misc[0];
            const bool is_k = rb < n_q + n_kv;
            const int kvh = is_k ? rb - n_q : rb - n_q - n_kv;
            const float ob = __bfloat162float(__float2bfloat16(o));   // the bf16 row the bf16 cache would hold
            (reinterpret_cast<uint8_t*>(is_k ? k_cache : v_cache) + (slot * n_kv + kvh) * 128)[row] =
                static_cast<uint8_t>(kv_fp8_quant2(ob, 0.0f, is_k ? k_scale : v_scale) & 0xffu);
        }
    }
};

struct TcOProjOp {
    __device__ bool rows_from_route_word(int, const TcSmem&) const { return false; }
    __device__ void rows_from_upstream(int, const TcSmem&) const {}
    __device__ bool trigger_at_start() const { return false; }
    static constexpr int kMaxRegs = 128;
    static constexpr int kId = 3;
    __device__ const __nv_bfloat16* x_global(int) const { return nullptr; }
    static constexpr bool kXFromGlobal = false;
    static constexpr bool kBulkX = true;
    static constexpr int kParts = 1, kXParts = 1, kStages = 5;
    static constexpr bool kHasRoute = false;
    static constexpr bool kRowsNeedPrologue = false, kRowsNeedUpstream = false;
    const __nv_bfloat16* x;
    __nv_bfloat16* h;
    int K, N;

    __device__ int x_elems() const { return K; }
    __device__ int num_row_blocks() const { return (N + 127) / 128; }
    __device__ int a_row(int, int rb, int, const TcSmem&) const { return rb * 128; }
    __device__ void pre_wait(int, const TcSmem&, bool) const {}
    __device__ void wide_partials(int, const TcSmem&) const {}
    __device__ void prologue(int b, const TcSmem& sm, bool) const { tc_bulk_x(x + static_cast<long long>(b) * K, sm.xs, K, sm.x_ready); }
    __device__ void finish(int b, int rb, int row, const float (&v)[1], TcFinish&, const TcSmem&) const {
        const int r = rb * 128 + row;
        if (r < N) {
            __nv_bfloat16* hr = h + static_cast<long long>(b) * N + r;
            *hr = __float2bfloat16(__bfloat162float(*hr) + v[0]);
        }
    }
    __device__ void finalize(int, TcFinish&) const {}
};

struct TcGateUpOp {
    static constexpr int kMaxRegs = 144;
    static constexpr int kId = 4;
    __device__ const __nv_bfloat16* x_global(int) const { return nullptr; }
    static constexpr bool kXFromGlobal = false;
    static constexpr bool kBulkX = false;
    static constexpr int kParts = 2, kXParts = 1, kStages = 3;
    static constexpr bool kHasRoute = true;
    static constexpr bool kRowsNeedPrologue = true, kRowsNeedUpstream = false;
    const __nv_bfloat16* h;
    const __nv_bfloat16* norm_w;
    const __nv_bfloat16* gate_w;   // [8, H]
    int* topk_ids;
    float* topk_w;
    __nv_bfloat16* act;            // [B, 2, I]
    int K, I;
    float eps;
    unsigned long long* route_word;   // [B] or nullptr: {tag, e0, e1} published as ONE word as soon as the router is done
    unsigned int route_tag;

    __device__ bool rows_from_route_word(int, const TcSmem&) const { return false; }
    __device__ void rows_from_upstream(int, const TcSmem&) const {}
    __device__ bool trigger_at_start() const { return route_word != nullptr; }
    __device__ int x_elems() const { return K; }
    __device__ int num_row_blocks() const { return 2 * (I / 128); }
    __device__ int a_row(int, int rb, int p, const TcSmem& sm) const {
        const int nb = I / 128, k = rb / nb, jb = rb % nb;
        return sm.misc[k] * 2 * I + p * I + jb * 128;   // rows of the fused [E * 2I, H] weight
    }
    __device__ void pre_wait(int b, const TcSmem&, bool on) const {
        // the word of the previous layer / step is dead by now (its reader completed before this kernel could start)
        if (route_word != nullptr && blockIdx.x == 0 && threadIdx.x == 128) st_relaxed_u64(route_word + b, 0ull);
        if (!on) return;
        tc_prefetch_l2(gate_w, 8ll * K * 2);
        tc_prefetch_l2(norm_w, K * 2ll);
    }
    // wide form, part 1: all 256 threads of the CTA take a share of the router dot products (one round trip to L2)
    __device__ void wide_partials(int b, const TcSmem& sm) const {
        float part[9];
        tc_route_partials(h + static_cast<long long>(b) * K, norm_w, gate_w, K, threadIdx.x, TC_THREADS, part);
        if ((threadIdx.x & 31) == 0)
#pragma unroll
            for (int e = 0; e < 9; ++e) sm.prep[(threadIdx.x >> 5) * 9 + e] = part[e];
    }
    __device__ void prologue(int b, const TcSmem& sm, bool wide) const {
        const int t = threadIdx.x - 128;
        const __nv_bfloat16* hr = h + static_cast<long long>(b) * K;
        TcRoute r;
        if (wide) {
            float tot[9];
#pragma unroll
            for (int e = 0; e < 9; ++e) {
                float s = 0.0f;
#pragma unroll
                for (int w = 0; w < TC_THREADS / 32; ++w) s += sm.prep[w * 9 + e];
                tot[e] = s;
            }
            r = tc_route_finish(tot, K, eps);
        } else {
            r = tc_route(hr, norm_w, gate_w, K, eps, sm.prep);
        }
        const float inv = r.inv;
        if (t == 0) {
            sm.misc[0] = r.e0;
            sm.misc[1] = r.e1;
            if (blockIdx.x == 0) {
                topk_ids[b * 2] = r.e0;
                topk_ids[b * 2 + 1] = r.e1;
                topk_w[b * 2] = r.w0;
                topk_w[b * 2 + 1] = r.w1;
                if (route_word != nullptr)
                    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(route_word + b),
                                 "l"((static_cast<unsigned long long>(route_tag) << 32) |
                                     static_cast<unsigned long long>((r.e0 << 8) | r.e1)) : "memory");
            }
        }
        for (int i = t * 8; i < K; i += 128 * 8) {
            const uint4 hv = *reinterpret_cast<const uint4*>(hr + i);
            const uint4 g = __ldg(reinterpret_cast<const uint4*>(norm_w + i));
            const uint32_t a[4] = {hv.x, hv.y, hv.z, hv.w}, gg[4] = {g.x, g.y, g.z, g.w};
            uint4 o;
            uint32_t* op = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
            for (int q = 0; q < 4; ++q)
                op[q] = pack_bf16(bf16_lo(a[q]) * inv * bf16_lo(gg[q]), bf16_hi(a[q]) * inv * bf16_hi(gg[q]));
            *reinterpret_cast<uint4*>(sm.xs + i) = o;
        }
    }
    __device__ void finish(int b, int rb, int row, const float (&v)[2], TcFinish&, const TcSmem&) const {
        const int nb = I / 128, k = rb / nb, jb = rb % nb;
        act[(static_cast<long long>(b) * 2 + k) * I + jb * 128 + row] = __float2bfloat16(silu(v[0]) * v[1]);
    }
    __device__ void finalize(int, TcFinish&) const {}
};

struct TcDownOp {
    static constexpr int kMaxRegs = 112;
    static constexpr int kId = 5;
    static constexpr bool kXFromGlobal = true;
    static constexpr bool kBulkX = false;
    static constexpr int kParts = 2, kXParts = 2, kStages = 3;
    static constexpr bool kHasRoute = false;
    static constexpr bool kRowsNeedPrologue = false, kRowsNeedUpstream = true;
    const __nv_bfloat16* act;   // [B, 2, I]
    const int* topk_ids;
    const float* topk_w;
    __nv_bfloat16* h;
    int K, H;                   // K = I
    const unsigned long long* route_word;   // [B] or nullptr (see TcGateUpOp)
    unsigned int route_tag;

    // producer lane only: the expert ids of this token, from the word the gate|up kernel published early ...
    __device__ bool rows_from_route_word(int b, const TcSmem& sm) const {
        if (route_word == nullptr) return false;
        for (int i = 0; i < 256; ++i) {   // published before this kernel could launch: the first load normally hits
            unsigned long long w;
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(w) : "l"(route_word + b) : "memory");
            if (static_cast<unsigned int>(w >> 32) == route_tag) {
                sm.misc[0] = static_cast<int>((w >> 8) & 0xff);
                sm.misc[1] = static_cast<int>(w & 0xff);
                return true;
            }
        }
        return false;
    }
    // ... or, after the dependency wait, from the ids array
    __device__ void rows_from_upstream(int b, const TcSmem& sm) const {
        sm.misc[0] = topk_ids[b * 2];
        sm.misc[1] = topk_ids[b * 2 + 1];
    }
    __device__ bool trigger_at_start() const { return false; }
    __device__ int x_elems() const { return 0; }   // the activation vectors are streamed from L2 by the x-tile writer
    __device__ const __nv_bfloat16* x_global(int b) const { return act + static_cast<long long>(b) * 2 * K; }
    __device__ int num_row_blocks() const { return (H + 127) / 128; }
    __device__ int a_row(int, int rb, int p, const TcSmem& sm) const { return sm.misc[p] * H + rb * 128; }
    __device__ void pre_wait(int, const TcSmem&, bool) const {}
    __device__ void wide_partials(int, const TcSmem&) const {}
    __device__ void prologue(int b, const TcSmem& sm, bool) const {
        const int t = threadIdx.x - 128;
        if (t < 2) sm.prep[t] = topk_w[b * 2 + t];
    }
    __device__ void finish(int b, int rb, int row, const float (&v)[2], TcFinish&, const TcSmem& sm) const {
        const int r = rb * 128 + row;
        if (r < H) {
            __nv_bfloat16* hr = h + static_cast<long long>(b) * H + r;
            *hr = __float2bfloat16(__bfloat162float(*hr) + sm.prep[0] * v[0] + sm.prep[1] * v[1]);
        }
    }
    __device__ void finalize(int, TcFinish&) const {}
};

// same key as decode.cu's pack_argmax (-0.0 packed as +0.0, so equal logits tie on the index across warps as well)
__device__ __forceinline__ unsigned long long tc_pack_argmax(float v, int idx) {
    uint32_t u = __float_as_uint(v);
    if (u == 0x80000000u) u = 0u;
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return (static_cast<unsigned long long>(u) << 32) |
           static_cast<unsigned long long>(0xFFFFFFFFu - static_cast<uint32_t>(idx));
}

struct TcLmHeadOp {
    __device__ bool rows_from_route_word(int, const TcSmem&) const { return false; }
    __device__ void rows_from_upstream(int, const TcSmem&) const {}
    __device__ bool trigger_at_start() const { return false; }
    static constexpr int kMaxRegs = 128;
    static constexpr int kId = 6;
    __device__ const __nv_bfloat16* x_global(int) const { return nullptr; }
    static constexpr bool kXFromGlobal = false;
    static constexpr bool kBulkX = false;
    static constexpr int kParts = 1, kXParts = 1, kStages = 5;
    static constexpr bool kHasRoute = false;
    static constexpr bool kRowsNeedPrologue = false, kRowsNeedUpstream = false;
    const __nv_bfloat16* h;
    long long h_stride;
    const __nv_bfloat16* norm_w;
    __nv_bfloat16* logits;
    unsigned long long* best;
    int K, V;
    float eps;

    __device__ int x_elems() const { return K; }
    __device__ int num_row_blocks() const { return (V + 127) / 128; }
    __device__ int a_row(int, int rb, int, const TcSmem&) const { return rb * 128; }
    __device__ void pre_wait(int, const TcSmem&, bool on) const { if (on) tc_prefetch_l2(norm_w, K * 2ll); }
    __device__ void wide_partials(int, const TcSmem&) const {}
    __device__ void prologue(int b, const TcSmem& sm, bool) const {
        tc_load_x_rmsnorm(h + static_cast<long long>(b) * h_stride, norm_w, sm.xs, K, eps, sm.scratch);
    }
    __device__ void finish(int b, int rb, int row, const float (&v)[1], TcFinish& st, const TcSmem&) const {
        const int r = rb * 128 + row;
        if (r >= V) return;
        const __nv_bfloat16 l = __float2bfloat16(v[0]);   // logits stay bf16; arg-max runs on them
        if (logits) logits[static_cast<long long>(b) * V + r] = l;
        const float f = __bfloat162float(l);
        if (f > st.best || (f == st.best && r < st.best_idx)) { st.best = f; st.best_idx = r; }
    }
    __device__ void finalize(int b, TcFinish& st) const {
        // warp arg-max, then one atomic per warp
        float bv = st.best;
        int bi = st.best_idx;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
        }
        if ((threadIdx.x & 31) == 0 && bi != 0x7fffffff) atomicMax(&best[b], tc_pack_argmax(bv, bi));
    }
};

struct TcWorkspace {
    unsigned long long* scratch;   // [B][row blocks][TC_SLOTS][2][128] words {value, tag}; all tags zero between launches
};

template <class Op>
static int launch_tc(const Op& op, const void* W, long long w_rows, int K, int n_rb, int x_elems, int B,
                     const TcWorkspace& ws, cudaStream_t st, const char* name) {
    CUtensorMap tm;
    const uint64_t dims[2] = {static_cast<uint64_t>(K), static_cast<uint64_t>(w_rows)};
    const uint64_t strides[1] = {static_cast<uint64_t>(K) * 2};
    const uint32_t box[2] = {64, 128};
    int rc = make_tensor_map_bf16(&tm, W, 2, dims, strides, box, true);
    if (rc) return rc;
    const int smem_bytes = Op::kStages * (Op::kParts * TC_A_BYTES + Op::kXParts * TC_X_BYTES) +
                           ((x_elems * 2 + 127) / 128) * 128 + (2 * Op::kStages + 1) * 8 +
                           (64 + 256 + 128 + 256 + 8) * 4 + 1024 + 128;
    auto kern = tc_gemv_kernel<Op>;
    static int configured = 0;
    if (smem_bytes > configured) {
        rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes), name);
        if (rc) return rc;
        configured = smem_bytes;
    }
    // co-residency with the neighbours of a programmatic-launch chain needs the SM configured for maximum shared
    // memory (the default carve-out only covers this kernel's own footprint)
    static int carveout = -1;
    const int want = option("smem_carveout_max") ? cudaSharedmemCarveoutMaxShared : cudaSharedmemCarveoutDefault;
    if (carveout != want) {
        rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, want), name);
        if (rc) return rc;
        carveout = want;
    }
    // keep the number of contributors per row block <= TC_SLOTS: every CTA gets at least ceil(n_kb / 6) units
    const int n_kb = K / 64;
    const long long U = static_cast<long long>(n_rb) * n_kb;
    const int min_units = (n_kb + 5) / 6;
    long long g = U / (min_units > 0 ? min_units : 1);
    if (g > num_sms()) g = num_sms();
    if (g < 1) g = 1;
    dim3 grid(static_cast<unsigned>(g), B);
    const int l2_ahead = option("tc_l2_ahead");   // tiles per CTA prefetched into L2 behind the ring
    const int flags = (option("tc_prefetch_consts") ? 1 : 0) | (option("chain_wait") ? 2 : 0) |
                      (option("tc_wide_route") ? 8 : 0) | (option("tc_park") ? 4 : 0) |
                      (option("tc_trigger_lead") << 8);
    ChainArgsDev chain{nullptr, nullptr, nullptr, 0};
    if (B == 1) {   // the counters protocol covers the bs = 1 step (fixed grids per chain position)
        const ChainArgs c = chain_next(static_cast<int>(g));
        chain = ChainArgsDev{c.serial, c.wait_cnt, c.done_cnt, c.wait_arrivals};
    }
    cudaError_t e = launch_chain(kern, grid, dim3(TC_THREADS), smem_bytes, st, tm, op, ws.scratch, l2_ahead, flags, chain VITA_TRACE_ARG);
    if (e != cudaSuccess) return check_cuda(e, name);
    return check_launch(name);
}

static inline bool tc_shape_ok(long long K) { return K % 64 == 0 && K >= 64; }

}  // namespace vita

using namespace vita;

// workspace: [B * max_rb * SLOTS * 2 * 128 words of 8 bytes {partial sum, tag}]; zero-initialised once, the kernels
// leave every tag cleared.
extern "C" int64_t vita_decode_tc_workspace_bytes(int64_t B, int64_t max_row_blocks) {
    return B * max_row_blocks * TC_SLOTS * 2 * 128 * 8;
}

static TcWorkspace split_ws(void* workspace, int64_t, int64_t) {
    TcWorkspace ws;
    ws.scratch = static_cast<unsigned long long*>(workspace);
    return ws;
}

extern "C" int vita_decode_tc_qkv_rope(const void* h, const void* norm_w, const void* w_qkv, const float* cos_sin,
                                       const int32_t* cur_pos, const int32_t* block_table, void* q_out, void* k_cache,
                                       void* v_cache, void* workspace, int64_t ws_row_blocks, int64_t B, int64_t H,
                                       int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim, int64_t page_size,
                                       int64_t max_pages, float eps, void* stream) {
    VITA_REQUIRE(head_dim == 128 && tc_shape_ok(H), "head_dim must be 128 and H a multiple of 64");
    const int n_rb = static_cast<int>(n_q_heads + 2 * n_kv_heads);
    VITA_REQUIRE(workspace && n_rb <= ws_row_blocks, "workspace too small");
    if (B == 0) return VITA_OK;
    TcQkvOp op{BF16C(h), BF16C(norm_w), cos_sin, cur_pos, block_table, static_cast<__nv_bfloat16*>(q_out),
               static_cast<__nv_bfloat16*>(k_cache), static_cast<__nv_bfloat16*>(v_cache), (int)H, (int)n_q_heads,
               (int)n_kv_heads, (int)page_size, (int)max_pages, eps};
    return launch_tc(op, w_qkv, n_rb * 128ll, (int)H, n_rb, (int)H, (int)B, split_ws(workspace, B, ws_row_blocks),
                     static_cast<cudaStream_t>(stream), "decode_tc_qkv_rope");
}

extern "C" int vita_decode_tc_qkv_rope_fp8(const void* h, const void* norm_w, const void* w_qkv, const float* cos_sin,
                                           const int32_t* cur_pos, const int32_t* block_table, void* q_out,
                                           void* k_cache, void* v_cache, void* workspace, int64_t ws_row_blocks,
                                           int64_t B, int64_t H, int64_t n_q_heads, int64_t n_kv_heads,
                                           int64_t head_dim, int64_t page_size, int64_t max_pages, float eps,
                                           float k_scale, float v_scale, void* stream) {
    VITA_REQUIRE(head_dim == 128 && tc_shape_ok(H), "head_dim must be 128 and H a multiple of 64");
    VITA_REQUIRE(kv_fp8_scales_ok(k_scale, v_scale), "k_scale / v_scale must be finite and positive");
    const int n_rb = static_cast<int>(n_q_heads + 2 * n_kv_heads);
    VITA_REQUIRE(workspace && n_rb <= ws_row_blocks, "workspace too small");
    if (B == 0) return VITA_OK;
    TcQkvFp8Op op{};
    static_cast<TcQkvOp&>(op) = TcQkvOp{BF16C(h), BF16C(norm_w), cos_sin, cur_pos, block_table,
                                        static_cast<__nv_bfloat16*>(q_out), static_cast<__nv_bfloat16*>(k_cache),
                                        static_cast<__nv_bfloat16*>(v_cache), (int)H, (int)n_q_heads, (int)n_kv_heads,
                                        (int)page_size, (int)max_pages, eps};
    op.k_scale = k_scale;
    op.v_scale = v_scale;
    return launch_tc(op, w_qkv, n_rb * 128ll, (int)H, n_rb, (int)H, (int)B, split_ws(workspace, B, ws_row_blocks),
                     static_cast<cudaStream_t>(stream), "decode_tc_qkv_rope_fp8");
}

extern "C" int vita_decode_tc_oproj(const void* x, const void* w, void* h, void* workspace, int64_t ws_row_blocks,
                                    int64_t B, int64_t N, int64_t K, void* stream) {
    VITA_REQUIRE(tc_shape_ok(K), "K must be a multiple of 64");
    const int n_rb = static_cast<int>((N + 127) / 128);
    VITA_REQUIRE(workspace && n_rb <= ws_row_blocks, "workspace too small");
    if (B == 0) return VITA_OK;
    TcOProjOp op{BF16C(x), static_cast<__nv_bfloat16*>(h), (int)K, (int)N};
    return launch_tc(op, w, N, (int)K, n_rb, (int)K, (int)B, split_ws(workspace, B, ws_row_blocks),
                     static_cast<cudaStream_t>(stream), "decode_tc_oproj");
}

extern "C" int vita_decode_tc_moe_gate_up(const void* h, const void* norm_w, const void* gate_w, const void* w13,
                                          int32_t* topk_ids, float* topk_w, void* act, void* workspace,
                                          int64_t ws_row_blocks, int64_t B, int64_t H, int64_t I, int64_t E, float eps,
                                          uint64_t* route_word, int64_t route_tag, void* stream) {
    VITA_REQUIRE(E == 8, "router is specialised for 8 experts (Mixtral-8x7B)");
    VITA_REQUIRE(tc_shape_ok(H) && I % 128 == 0, "H must be a multiple of 64 and I a multiple of 128");
    const int n_rb = static_cast<int>(2 * (I / 128));
    VITA_REQUIRE(workspace && n_rb <= ws_row_blocks, "workspace too small");
    if (B == 0) return VITA_OK;
    VITA_REQUIRE(route_word == nullptr || (route_tag > 0 && route_tag < (1ll << 32)), "route_tag must be in [1, 2^32)");
    // the early hand-over relies on the chain being transitive (option chain_wait) -- otherwise it stays off
    unsigned long long* rw = option("chain_wait") ? reinterpret_cast<unsigned long long*>(route_word) : nullptr;
    TcGateUpOp op{BF16C(h), BF16C(norm_w), BF16C(gate_w), topk_ids, topk_w, static_cast<__nv_bfloat16*>(act), (int)H,
                  (int)I, eps, rw, static_cast<unsigned int>(route_tag)};
    return launch_tc(op, w13, E * 2 * I, (int)H, n_rb, (int)H, (int)B, split_ws(workspace, B, ws_row_blocks),
                     static_cast<cudaStream_t>(stream), "decode_tc_moe_gate_up");
}

extern "C" int vita_decode_tc_moe_down(const void* act, const void* w2, const int32_t* topk_ids, const float* topk_w,
                                       void* h, void* workspace, int64_t ws_row_blocks, int64_t B, int64_t H,
                                       int64_t I, int64_t E, const uint64_t* route_word, int64_t route_tag,
                                       void* stream) {
    VITA_REQUIRE(tc_shape_ok(I) && H % 128 == 0, "I must be a multiple of 64 and H a multiple of 128");
    const int n_rb = static_cast<int>(H / 128);
    VITA_REQUIRE(workspace && n_rb <= ws_row_blocks, "workspace too small");
    if (B == 0) return VITA_OK;
    VITA_REQUIRE(route_word == nullptr || (route_tag > 0 && route_tag < (1ll << 32)), "route_tag must be in [1, 2^32)");
    const unsigned long long* rw = option("chain_wait") ? reinterpret_cast<const unsigned long long*>(route_word) : nullptr;
    TcDownOp op{BF16C(act), topk_ids, topk_w, static_cast<__nv_bfloat16*>(h), (int)I, (int)H, rw,
                static_cast<unsigned int>(route_tag)};
    return launch_tc(op, w2, E * H, (int)I, n_rb, 0, (int)B, split_ws(workspace, B, ws_row_blocks),
                     static_cast<cudaStream_t>(stream), "decode_tc_moe_down");
}

extern "C" int vita_tc_lm_head_argmax(const void* h, int64_t h_stride, const void* norm_w, const void* w, void* logits,
                                      uint64_t* best, void* workspace, int64_t ws_row_blocks, int64_t B, int64_t H,
                                      int64_t V, float eps, void* stream) {
    VITA_REQUIRE(tc_shape_ok(H), "H must be a multiple of 64");
    const int n_rb = static_cast<int>((V + 127) / 128);
    VITA_REQUIRE(workspace && n_rb <= ws_row_blocks, "workspace too small");
    if (B == 0) return VITA_OK;
    TcLmHeadOp op{BF16C(h), h_stride, BF16C(norm_w), static_cast<__nv_bfloat16*>(logits),
                  reinterpret_cast<unsigned long long*>(best), (int)H, (int)V, eps};
    return launch_tc(op, w, V, (int)H, n_rb, (int)H, (int)B, split_ws(workspace, B, ws_row_blocks),
                     static_cast<cudaStream_t>(stream), "tc_lm_head_argmax");
}
