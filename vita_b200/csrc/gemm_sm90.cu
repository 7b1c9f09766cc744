// bf16 "TN" GEMM for sm_90a:  C[M,N] = epilogue(A[M,K] . B[N,K]^T), fp32 accumulation in registers (wgmma).
//
// Structure (one persistent CTA per SM, 384 threads):
//   warpgroup 0   : TMA producer (one thread: cp.async.bulk.tensor -> 128B-swizzled smem ring, mbarrier complete_tx);
//                   gives its registers to the consumers with setmaxnreg
//   warpgroups 1-2: consumers; each owns 64 rows of the 128 x BLOCK_N tile (wgmma.mma_async m64nNk16, A and B from
//                   shared memory) and runs the fused epilogue on its accumulator fragment
// While the consumers run the epilogue of tile i the producer already fills the ring with tile i+1.  The same kernel serves the plain linears (ViT / Whale / projector / Mixtral qkv,o) and the
// grouped expert GEMMs of the MoE (ragged row groups given by a device-side offsets array, no host sync).
//
// Reference call sites this replaces (all nn.Linear / F.linear -> cuBLAS in the reference):
//   vita/model/multimodal_encoder/internvit/modeling_intern_vit.py:180,192,214,216
//   vita/model/multimodal_encoder/whale/module/layer/attention.py:371-373,381,419 ; :145-147
//   vita/model/multimodal_projector/builder.py:164-168
//   transformers MixtralAttention q/k/v/o_proj, MixtralExperts.forward (gate_up_proj / down_proj)
#include <cstdlib>

#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"
#include "kv_fp8.cuh"

namespace vita {

struct GemmArgs {
    int M;                      // rows of A / C (total over groups)
    int N;                      // output columns (per group)
    int K;
    int num_groups;             // >= 1
    const int* group_offsets;   // device [num_groups + 1] row offsets, or nullptr (single group = all rows)
    const int* group_counts;    // or: group g occupies rows [g * group_stride, g * group_stride + group_counts[g])
    int group_stride;           //     ("slot" layout written by vita_moe_route_scatter: a fixed capacity per expert)
    int est_rows;               // host-side estimate of the occupied rows (tile-shape heuristics); 0 = M
    __nv_bfloat16* C;
    long long ldc;
    const __nv_bfloat16* bias;  // [num_groups, N] or nullptr
    const __nv_bfloat16* colscale;  // [N] or nullptr   (InternViT layer-scale ls1/ls2)
    const float* rowscale;          // [M] or nullptr   (MoE routing weight)
    const __nv_bfloat16* residual;  // [M, ldr] or nullptr
    long long ldr;
    int act;                    // VITA_ACT_*
    // expert-parallel scatter epilogue (down projection): output row r goes to the rank that owns its token,
    //   dst = peer_out[t / chunk] + ((t % chunk) * 2 + k) * ldc   with (t, k) = (row_assign[r] >> 1, row_assign[r] & 1)
    const int* row_assign;
    __nv_bfloat16* const* peer_out;
    int chunk;
    int tail_split;             // cut the tiles of the last partial wave along N (see Sched)
    // fused RoPE + paged KV append epilogue of the qkv projection (N = (n_q + 2 n_kv) * 128; MixtralAttention.forward
    // modeling_mixtral.py:312-340 + the cache update): column block h of 128 is head h; q and k heads are rotated with
    // the row's position, k and v heads are also written to their cache slot.  nullptr = plain epilogue.
    const float* rope_cos_sin;  // fp32 [max_pos, 2, 64]
    const int* rope_pos;        // [M] position of each row
    const int* rope_slot;       // [M] cache slot of each row, or nullptr (no cache write)
    __nv_bfloat16* k_cache;
    __nv_bfloat16* v_cache;
    int n_q, n_kv;
    float k_scale, v_scale;     // e4m3 cache (kernel template KV8): k_cache / v_cache hold bytes, kv_fp8.cuh
};

__device__ __forceinline__ void group_rows(const GemmArgs& a, int g, int& r0, int& r1) {
    if (a.group_counts) { r0 = g * a.group_stride; r1 = r0 + a.group_counts[g]; }
    else if (a.group_offsets) { r0 = a.group_offsets[g]; r1 = a.group_offsets[g + 1]; }
    else { r0 = 0; r1 = a.M; }
}

struct Tile {
    int group, m0, m_end, n0;
    int bn;   // MMA N of this work item: BLOCK_N for a whole tile, BLOCK_N / split for a piece of a tail tile
};

// Work list of one launch.  Tiles are ordered group-major, n-block major, m-block minor (CTAs that run together share
// the weight tile in L2) and dealt round-robin to the persistent CTAs.  The tiles of the last, partly filled wave are
// cut along N into `split` pieces (2 or 4) when that still fits one wave: a 512-tile problem on 132 SMs then costs
// 3 + 1/2 waves instead of 4.  (The fused gate|up variant is not cut: its N
// tile is two half tiles and it runs ~50 waves.)
struct Sched {
    int total;      // whole tiles
    int full_end;   // tiles [0, full_end) are processed whole
    int split;      // the others in `split` pieces each
    __device__ __forceinline__ int items() const { return full_end + (total - full_end) * split; }
};

template <int BLOCK_N, int BN_OUT, bool SILU, int TILE_M>
__device__ __forceinline__ Sched make_sched(const GemmArgs& a) {
    const int num_n = (a.N + BN_OUT - 1) / BN_OUT;
    int total = 0;
    for (int g = 0; g < a.num_groups; ++g) {
        int r0, r1;
        group_rows(a, g, r0, r1);
        total += ((r1 - r0 + TILE_M - 1) / TILE_M) * num_n;
    }
    Sched s{total, total, 1};
    if (!SILU && a.tail_split) {
        const int G = static_cast<int>(gridDim.x);
        const int R = total % G;
        constexpr int MAX_SPLIT = BLOCK_N / 32 < 4 ? BLOCK_N / 32 : 4;   // pieces of at least 32 columns, at most 4
        const int max_split = a.rope_cos_sin ? BLOCK_N / 128 : MAX_SPLIT;   // RoPE pairs column j with j + 64 of a head
        int sp = 1;
        while (R > 0 && sp * 2 <= max_split && sp * 2 * R <= G) sp *= 2;
        if (sp > 1) { s.full_end = total - R; s.split = sp; }
    }
    return s;
}

template <int BLOCK_N, int BN_OUT, int TILE_M>
__device__ __forceinline__ bool tile_at(const GemmArgs& a, const Sched& sc, int item, Tile& t) {
    if (item >= sc.items()) return false;
    int tile_idx = item, part = 0;
    t.bn = BLOCK_N;
    if (item >= sc.full_end) {
        const int j = item - sc.full_end;
        tile_idx = sc.full_end + j / sc.split;
        part = j % sc.split;
        t.bn = BLOCK_N / sc.split;
    }
    const int num_n = (a.N + BN_OUT - 1) / BN_OUT;
    int base = 0;
    for (int g = 0; g < a.num_groups; ++g) {
        int r0, r1;
        group_rows(a, g, r0, r1);
        const int mt = (r1 - r0 + TILE_M - 1) / TILE_M;
        const int nt = mt * num_n;
        if (tile_idx < base + nt) {
            const int local = tile_idx - base;
            t.group = g;
            t.n0 = (local / mt) * BN_OUT + part * t.bn;
            t.m0 = r0 + (local % mt) * TILE_M;
            t.m_end = r1;
            return true;
        }
        base += nt;
    }
    return false;
}

constexpr int GEMM_THREADS = 384;   // producer warpgroup + two consumer warpgroups of 64 tile rows each

// One consumer warpgroup's share of a tile's main loop: rows [64 cw, 64 cw + 64) of the A stage times N rows of the B
// stage, accumulated into the first N / 2 registers of `acc`.  One wgmma group stays in flight: a ring stage is handed
// back to the producer once the group that read it has completed (one arrival per warp).
template <int N, int STAGES, int ACC>
__device__ __forceinline__ void gemm_mainloop(float (&acc)[ACC], uint32_t sA_addr, uint32_t sB_addr, int a_stage_bytes,
                                              int b_stage_bytes, uint64_t* full_bar, uint64_t* empty_bar, int num_kb,
                                              int& stage, uint32_t& phase, int lane) {
    static_assert(N / 2 <= ACC, "accumulator too small");
    float (&d)[N / 2] = reinterpret_cast<float (&)[N / 2]>(acc);
    int prev = -1;
    for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase, 3);
        wgmma_acc_fence(d);
        wgmma_fence();
        const uint64_t da = wgmma_desc_k_sw128(sA_addr + stage * a_stage_bytes);
        const uint64_t db = wgmma_desc_k_sw128(sB_addr + stage * b_stage_bytes);
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<N>(d, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1 : 0);
        wgmma_commit();
        wgmma_acc_fence(d);
        if (prev >= 0) {
            wgmma_wait<1>();
            if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_acc_fence(d);
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
}

// what the epilogue knows about one output row of a thread's accumulator fragment
struct EpiRow {
    bool valid;
    float rs;                      // routing weight (1 without rowscale)
    __nv_bfloat16* crow;
    const __nv_bfloat16* rrow;     // residual row or nullptr
};

// columns (col, col + 1) of one row: bias -> activation -> column scale -> row scale -> residual -> bf16
__device__ __forceinline__ void epi_store2(const GemmArgs& a, const EpiRow& r, const __nv_bfloat16* bias, int col,
                                           float x0, float x1) {
    if (!r.valid || col >= a.N) return;
    const bool two = col + 1 < a.N;
    if (bias) {
        x0 += __bfloat162float(bias[col]);
        if (two) x1 += __bfloat162float(bias[col + 1]);
    }
    if (a.act == VITA_ACT_GELU) { x0 = gelu_erf(x0); x1 = gelu_erf(x1); }
    else if (a.act == VITA_ACT_RELU) { x0 = fmaxf(x0, 0.0f); x1 = fmaxf(x1, 0.0f); }
    if (a.colscale) {
        x0 *= __bfloat162float(a.colscale[col]);
        if (two) x1 *= __bfloat162float(a.colscale[col + 1]);
    }
    if (a.rowscale) { x0 *= r.rs; x1 *= r.rs; }
    if (two) {
        if (r.rrow) {
            const uint32_t w = *reinterpret_cast<const uint32_t*>(r.rrow + col);
            x0 += bf16_lo(w);
            x1 += bf16_hi(w);
        }
        *reinterpret_cast<uint32_t*>(r.crow + col) = pack_bf16(x0, x1);
    } else {
        if (r.rrow) x0 += __bfloat162float(r.rrow[col]);
        r.crow[col] = __float2bfloat16(x0);
    }
}

// Persistent CTA, 384 threads.  Thread 0 is the TMA producer; each consumer warpgroup owns 64 rows of the 128-row tile
// and keeps its 64 x BLOCK_N accumulator in registers (wgmma m64nNk16, both operands from the 128B-swizzled ring).
template <int BLOCK_N, bool SILU, int STAGES, bool KV8 = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmBs /* B in boxes of 32 rows: pieces of tail tiles */,
                    const GemmArgs args) {
    constexpr int BLOCK_M = 128, BLOCK_K = 64;
    constexpr int A_BYTES = BLOCK_M * BLOCK_K * 2;
    constexpr int B_BYTES = BLOCK_N * BLOCK_K * 2;
    constexpr int BN_OUT = SILU ? BLOCK_N / 2 : BLOCK_N;
    constexpr int TILE_M = BLOCK_M;

    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* sA = smem;
    uint8_t* sB = smem + STAGES * A_BYTES;
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int num_kb = (args.K + BLOCK_K - 1) / BLOCK_K;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        if (!SILU) tma_prefetch_desc(&tmBs);
        for (int i = 0; i < STAGES; ++i) {
            mbar_init(&full_bar[i], 1);
            mbar_init(&empty_bar[i], 8);   // one arrival per consumer warp
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (warp < 4) {
        // the producer warpgroup hands its registers to the consumers (384 x 168 = 128 x 40 + 256 x 232)
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            // ------------------------------------------------------------ TMA producer
            int stage = 0;
            uint32_t phase = 0;
            Tile t;
            const Sched sc = make_sched<BLOCK_N, BN_OUT, SILU, TILE_M>(args);
            for (int tile = blockIdx.x; tile_at<BLOCK_N, BN_OUT, TILE_M>(args, sc, tile, t); tile += gridDim.x) {
                for (int kb = 0; kb < num_kb; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1, 1);
                    mbar_arrive_expect_tx(&full_bar[stage], A_BYTES + t.bn * (BLOCK_K * 2));
                    tma_load_2d(sA + stage * A_BYTES, &tmA, &full_bar[stage], kb * BLOCK_K, t.m0);
                    if (!SILU && t.bn != BLOCK_N) {
                        for (int r = 0; r < t.bn; r += 32)
                            tma_load_3d(sB + stage * B_BYTES + r * (BLOCK_K * 2), &tmBs, &full_bar[stage], kb * BLOCK_K,
                                        t.n0 + r, t.group);
                    } else if constexpr (SILU) {
                        // gate rows [n0, n0 + BN_OUT) and up rows [N + n0, N + n0 + BN_OUT) of the fused [2N, K] weight
                        tma_load_3d(sB + stage * B_BYTES, &tmB, &full_bar[stage], kb * BLOCK_K, t.n0, t.group);
                        tma_load_3d(sB + stage * B_BYTES + B_BYTES / 2, &tmB, &full_bar[stage], kb * BLOCK_K,
                                    args.N + t.n0, t.group);
                    } else {
                        tma_load_3d(sB + stage * B_BYTES, &tmB, &full_bar[stage], kb * BLOCK_K, t.n0, t.group);
                    }
                    if (++stage == STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }

    // ---------------------------------------------------------------- consumers: MMA + epilogue
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int cw = (warp >> 2) - 1;   // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
    const int qr = lane >> 2, qc = lane & 3;
    const uint32_t sA_addr = smem_u32(sA) + cw * (64 * BLOCK_K * 2), sB_addr = smem_u32(sB);
    int stage = 0;
    uint32_t phase = 0;
    float acc[BLOCK_N / 2];
    Tile t;
    const Sched sc = make_sched<BLOCK_N, BN_OUT, SILU, TILE_M>(args);
    for (int tile = blockIdx.x; tile_at<BLOCK_N, BN_OUT, TILE_M>(args, sc, tile, t); tile += gridDim.x) {
        if (t.bn == BLOCK_N)
            gemm_mainloop<BLOCK_N, STAGES>(acc, sA_addr, sB_addr, A_BYTES, B_BYTES, full_bar, empty_bar, num_kb, stage, phase, lane);
        else if (t.bn == BLOCK_N / 2)
            gemm_mainloop<BLOCK_N / 2, STAGES>(acc, sA_addr, sB_addr, A_BYTES, B_BYTES, full_bar, empty_bar, num_kb, stage, phase, lane);
        else
            gemm_mainloop<BLOCK_N / 4, STAGES>(acc, sA_addr, sB_addr, A_BYTES, B_BYTES, full_bar, empty_bar, num_kb, stage, phase, lane);

        EpiRow row[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int grow = t.m0 + cw * 64 + (warp & 3) * 16 + qr + 8 * h;
            row[h].valid = grow < t.m_end;
            row[h].rs = (args.rowscale && row[h].valid) ? args.rowscale[grow] : 1.0f;
            row[h].crow = args.C + static_cast<long long>(grow) * args.ldc;
            if (args.peer_out != nullptr && row[h].valid) {
                const int a = args.row_assign[grow], tk = a >> 1;
                const int owner = tk / args.chunk;
                row[h].crow = args.peer_out[owner] + (static_cast<long long>(tk - owner * args.chunk) * 2 + (a & 1)) * args.ldc;
            }
            row[h].rrow = args.residual ? args.residual + static_cast<long long>(grow) * args.ldr : nullptr;
        }
        const __nv_bfloat16* bias = args.bias ? args.bias + static_cast<long long>(t.group) * args.N : nullptr;

        if constexpr (!SILU) {
            if (args.rope_cos_sin != nullptr) {
                // ---- qkv projection: RoPE on the bf16-rounded projections, K / V rows appended to the paged cache.
                // Column j of a head and its partner j + 64 sit in the same thread (fragment blocks jb and jb + 8).
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!row[h].valid) continue;
                    const int grow = t.m0 + cw * 64 + (warp & 3) * 16 + qr + 8 * h;
                    const int pos = args.rope_pos[grow];
                    const long long slot = args.rope_slot ? args.rope_slot[grow] : -1;
                    const float* cs = args.rope_cos_sin + static_cast<long long>(pos) * 128;
#pragma unroll
                    for (int hh = 0; hh < BLOCK_N / 128; ++hh) {
                        const int head = (t.n0 >> 7) + hh;
                        if (hh * 128 >= t.bn || head * 128 >= args.N) break;   // warp-uniform
                        const bool rot = head < args.n_q + args.n_kv;
                        __nv_bfloat16* cdst = nullptr;
                        uint8_t* cdst8 = nullptr;   // KV8: e4m3 row, quantized from the bf16 values stored above
                        float cscale = 1.0f;
                        if constexpr (KV8) {
                            if (slot >= 0 && head >= args.n_q) {
                                const bool is_k = head < args.n_q + args.n_kv;
                                const int kvh = is_k ? head - args.n_q : head - args.n_q - args.n_kv;
                                cdst8 = reinterpret_cast<uint8_t*>(is_k ? args.k_cache : args.v_cache) + (slot * args.n_kv + kvh) * 128;
                                cscale = is_k ? args.k_scale : args.v_scale;
                            }
                        } else {
                        if (slot >= 0 && head >= args.n_q) {
                            const bool is_k = head < args.n_q + args.n_kv;
                            const int kvh = is_k ? head - args.n_q : head - args.n_q - args.n_kv;
                            cdst = (is_k ? args.k_cache : args.v_cache) + (slot * args.n_kv + kvh) * 128;
                        }
                        }
#pragma unroll
                        for (int jb = 0; jb < 8; ++jb) {
                            const int j = jb * 8 + 2 * qc;   // column inside the first half of the head
                            float2 cc = make_float2(1.f, 1.f), ss = make_float2(0.f, 0.f);
                            if (rot) {
                                cc = __ldg(reinterpret_cast<const float2*>(cs + j));
                                ss = __ldg(reinterpret_cast<const float2*>(cs + 64 + j));
                            }
                            const float c2[2] = {cc.x, cc.y}, s2[2] = {ss.x, ss.y};
                            float r1[2], r2[2];
#pragma unroll
                            for (int e = 0; e < 2; ++e) {
                                // projections are rounded to bf16 first, as the stand-alone pass sees them
                                const float x1 = __bfloat162float(__float2bfloat16(acc[4 * (hh * 16 + jb) + 2 * h + e]));
                                const float x2 = __bfloat162float(__float2bfloat16(acc[4 * (hh * 16 + jb + 8) + 2 * h + e]));
                                if (rot) rope_rotate(x1, x2, c2[e], s2[e], r1[e], r2[e]);
                                else { r1[e] = x1; r2[e] = x2; }
                            }
                            const uint32_t o1 = pack_bf16(r1[0], r1[1]), o2 = pack_bf16(r2[0], r2[1]);
                            *reinterpret_cast<uint32_t*>(row[h].crow + head * 128 + j) = o1;
                            *reinterpret_cast<uint32_t*>(row[h].crow + head * 128 + 64 + j) = o2;
                            if constexpr (KV8) {
                                if (cdst8 != nullptr) {
                                    *reinterpret_cast<uint16_t*>(cdst8 + j) =
                                        static_cast<uint16_t>(kv_fp8_quant2(bf16_lo(o1), bf16_hi(o1), cscale));
                                    *reinterpret_cast<uint16_t*>(cdst8 + 64 + j) =
                                        static_cast<uint16_t>(kv_fp8_quant2(bf16_lo(o2), bf16_hi(o2), cscale));
                                }
                            } else {
                            if (cdst != nullptr) {
                                *reinterpret_cast<uint32_t*>(cdst + j) = o1;
                                *reinterpret_cast<uint32_t*>(cdst + 64 + j) = o2;
                            }
                            }
                        }
                    }
                }
                continue;
            }
        }
#pragma unroll
        for (int jb = 0; jb < BN_OUT / 8; ++jb) {
            if (jb * 8 >= (SILU ? BN_OUT : t.bn)) break;   // piece of a tail tile: warp-uniform
            const int col = t.n0 + jb * 8 + 2 * qc;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float x0 = acc[4 * jb + 2 * h], x1 = acc[4 * jb + 2 * h + 1];
                if constexpr (SILU) {
                    x0 = silu(x0) * acc[4 * (jb + BN_OUT / 8) + 2 * h];
                    x1 = silu(x1) * acc[4 * (jb + BN_OUT / 8) + 2 * h + 1];
                }
                epi_store2(args, row[h], bias, col, x0, x1);
            }
        }
    }
}

template <int BLOCK_N, bool SILU, int STAGES, bool KV8 = false>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmBs, const GemmArgs& args,
                       int max_tiles, cudaStream_t stream) {
    constexpr int smem_bytes = STAGES * (128 * 64 * 2 + BLOCK_N * 64 * 2) + 1024 + 256;
    static bool configured = false;
    auto kern = gemm_bf16_tn_kernel<BLOCK_N, SILU, STAGES, KV8>;
    if (!configured) {
        int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes),
                            "cudaFuncSetAttribute(gemm smem)");
        if (rc) return rc;
        configured = true;
    }
    int grid = num_sms();
    // with the tail split a problem of fewer tiles than SMs still spreads over the whole machine
    const long long items = static_cast<long long>(max_tiles) * ((!SILU && args.tail_split) ? (BLOCK_N / 32 < 4 ? BLOCK_N / 32 : 4) : 1);
    if (items < grid) grid = static_cast<int>(items);
    if (grid < 1) grid = 1;
    kern<<<grid, GEMM_THREADS, smem_bytes, stream>>>(tmA, tmB, tmBs, args);
    return check_launch("gemm_bf16_tn_kernel");
}

// a_rows: number of valid rows in A (TMA zero-fills beyond); b: [num_groups, b_rows, K] contiguous.
static int gemm_dispatch(const void* A, long long lda, int a_rows, const void* B, int b_rows, const GemmArgs& args,
                         bool silu, cudaStream_t stream, bool kv8 = false) {
    VITA_REQUIRE(args.K > 0 && args.N > 0 && args.M >= 0, "bad shape");
    VITA_REQUIRE(args.K % 8 == 0 && lda % 8 == 0, "K and lda must be multiples of 8 (16-byte TMA strides)");
    VITA_REQUIRE(aligned16(A) && aligned16(B) && aligned16(args.C), "A, B, C must be 16-byte aligned");
    VITA_REQUIRE(args.ldc % 8 == 0, "ldc must be a multiple of 8");
    VITA_REQUIRE(!args.residual || (args.ldr % 8 == 0 && aligned16(args.residual)), "residual alignment");
    VITA_REQUIRE(!args.bias || aligned16(args.bias), "bias alignment");
    VITA_REQUIRE(!args.bias || args.num_groups == 1 || args.N % 8 == 0, "grouped bias needs N % 8 == 0");
    VITA_REQUIRE(!args.colscale || aligned16(args.colscale), "colscale alignment");
    if (args.M == 0) return VITA_OK;

    const int n_sms = num_sms();
    const int occ_rows = args.est_rows > 0 ? args.est_rows : args.M;   // rows that carry work (slot layout: M is the capacity)
    const long long m_tiles_ub = (occ_rows / 128) + args.num_groups;  // valid for any ragged split of the occupied rows
    // Tile-shape choice.  Small-M problems stream each weight tile once and are HBM-bound, so what matters is how
    // evenly the tiles fill the SMs (wave quantisation); large-M problems want the 256-wide tile (the A operand is
    // read from shared memory half as often per flop).  Estimate the tile count and take the widest tile whose last wave
    // is not mostly idle.
    const long long m_tiles_est = (occ_rows + 127) / 128 + (args.num_groups > 1 ? args.num_groups / 2 : 0);
    const char* ts_env = getenv("VITA_B200_GEMM_TAIL_SPLIT");   // tuning aid: 0 switches the tail split off
    const bool tail_split = !silu && !(ts_env && atoi(ts_env) == 0);
    // Estimated duration in units of one 128 x 256 tile on one SM.  Cost model (not a measurement): a 128-wide tile
    // costs 0.76 of a 256-wide one when compute-bound (its A operand is read twice as often per flop), half when the
    // weights are streamed once from HBM (few row tiles); the pieces of a cut tail tile likewise 0.75 / 0.6 of the
    // whole for 1/2 and 1/4 of the width when compute-bound, 1/2 and 1/4 when HBM-bound.
    const bool hbm_bound = m_tiles_est <= 2;
    auto est_time = [&](int bn) {
        const long long tiles = m_tiles_est * ((args.N + bn - 1) / bn);
        const long long whole = tiles / n_sms, rest = tiles % n_sms;
        double waves = static_cast<double>(whole);
        if (rest > 0) {
            int sp = 1;
            while (tail_split && sp < 4 && sp * 2 * rest <= n_sms) sp *= 2;
            waves += hbm_bound ? 1.0 / sp : (sp == 1 ? 1.0 : (sp == 2 ? 0.75 : 0.6));
        }
        return waves * (bn == 256 ? 1.0 : (hbm_bound ? 0.5 : 0.76));
    };
    int block_n;
    const char* force = getenv("VITA_B200_GEMM_BN");   // tuning aid: force the tile width (128 / 256)
    if (kv8) {
        block_n = 256;   // the e4m3 KV append has one instantiation: two whole heads per tile
    } else if (force && (atoi(force) == 128 || atoi(force) == 256)) {
        block_n = atoi(force);
        if (!silu && args.N < 256) block_n = 128;
    } else if (silu) {
        // the 64-wide variant halves the weight tile but re-reads the activation tile twice as often from L2, so it
        // is only used when forced
        block_n = 256;
    } else if (args.rope_cos_sin != nullptr) {
        block_n = 256;   // two whole heads per tile
    } else if (args.N < 256) {
        block_n = 128;
    } else {
        block_n = (est_time(256) <= est_time(128) * 1.02) ? 256 : 128;
    }
    const int bn_out = silu ? block_n / 2 : block_n;
    const long long max_tiles_ll = m_tiles_ub * ((args.N + bn_out - 1) / bn_out);
    const int max_tiles = max_tiles_ll > (1 << 30) ? (1 << 30) : static_cast<int>(max_tiles_ll);

    GemmArgs a2 = args;
    a2.tail_split = tail_split ? 1 : 0;
    CUtensorMap tmA, tmB, tmBs;
    {
        const uint64_t dims[2] = {static_cast<uint64_t>(args.K), static_cast<uint64_t>(a_rows)};
        const uint64_t strides[1] = {static_cast<uint64_t>(lda) * 2};
        const uint32_t box[2] = {64, 128};
        int rc = make_tensor_map_bf16(&tmA, A, 2, dims, strides, box, true);
        if (rc) return rc;
    }
    {
        const uint64_t dims[3] = {static_cast<uint64_t>(args.K), static_cast<uint64_t>(b_rows),
                                  static_cast<uint64_t>(args.num_groups)};
        const uint64_t strides[2] = {static_cast<uint64_t>(args.K) * 2,
                                     static_cast<uint64_t>(args.K) * 2 * static_cast<uint64_t>(b_rows)};
        const uint32_t box[3] = {64, static_cast<uint32_t>(silu ? block_n / 2 : block_n), 1};
        int rc = make_tensor_map_bf16(&tmB, B, 3, dims, strides, box, true);
        if (rc) return rc;
    }
    tmBs = tmB;
    if (tail_split) {
        const uint64_t dims[3] = {static_cast<uint64_t>(args.K), static_cast<uint64_t>(b_rows),
                                  static_cast<uint64_t>(args.num_groups)};
        const uint64_t strides[2] = {static_cast<uint64_t>(args.K) * 2,
                                     static_cast<uint64_t>(args.K) * 2 * static_cast<uint64_t>(b_rows)};
        const uint32_t box[3] = {64, 32, 1};
        int rc = make_tensor_map_bf16(&tmBs, B, 3, dims, strides, box, true);
        if (rc) return rc;
    }
    if (kv8) return launch_gemm<256, false, 4, true>(tmA, tmB, tmBs, a2, max_tiles, stream);   // block_n is 256 (qkv)
    if (silu && block_n == 256) return launch_gemm<256, true, 4>(tmA, tmB, tmBs, a2, max_tiles, stream);
    if (silu) return launch_gemm<128, true, 6>(tmA, tmB, tmBs, a2, max_tiles, stream);
    if (block_n == 256) return launch_gemm<256, false, 4>(tmA, tmB, tmBs, a2, max_tiles, stream);
    return launch_gemm<128, false, 6>(tmA, tmB, tmBs, a2, max_tiles, stream);
}

}  // namespace vita

using namespace vita;

extern "C" int vita_gemm_bf16(const void* A, int64_t lda, const void* B, void* C, int64_t ldc, int64_t M, int64_t N,
                              int64_t K, const void* bias, int act, const void* colscale, const void* residual,
                              int64_t ldr, void* stream) {
    GemmArgs a{};
    a.M = static_cast<int>(M);
    a.N = static_cast<int>(N);
    a.K = static_cast<int>(K);
    a.num_groups = 1;
    a.group_offsets = nullptr;
    a.C = static_cast<__nv_bfloat16*>(C);
    a.ldc = ldc;
    a.bias = static_cast<const __nv_bfloat16*>(bias);
    a.colscale = static_cast<const __nv_bfloat16*>(colscale);
    a.rowscale = nullptr;
    a.residual = static_cast<const __nv_bfloat16*>(residual);
    a.ldr = ldr;
    a.act = act;
    VITA_REQUIRE(act == VITA_ACT_NONE || act == VITA_ACT_GELU || act == VITA_ACT_RELU, "unknown activation");
    return gemm_dispatch(A, lda, a.M, B, a.N, a, false, static_cast<cudaStream_t>(stream));
}

// qkv projection with the RoPE + paged-KV-append epilogue (see GemmArgs): qkv_out [M, (n_q + 2 n_kv) * 128] receives the
// rotated q and k heads and the v heads (what the prefill attention reads), k_cache / v_cache the rows of the slots.
static int gemm_qkv_rope(const void* X, int64_t ldx, const void* W_qkv, void* qkv_out, int64_t M, int64_t K,
                                  int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim, const int32_t* positions,
                                  const int32_t* slot_mapping, const float* cos_sin, void* k_cache, void* v_cache,
                                  void* stream, bool kv8, float k_scale, float v_scale) {
    VITA_REQUIRE(head_dim == 128, "head_dim must be 128");
    VITA_REQUIRE(positions != nullptr && cos_sin != nullptr, "positions and cos_sin are required");
    VITA_REQUIRE(slot_mapping == nullptr || (k_cache != nullptr && v_cache != nullptr), "slot_mapping needs both caches");
    VITA_REQUIRE(aligned16(cos_sin) && (!k_cache || aligned16(k_cache)) && (!v_cache || aligned16(v_cache)), "alignment");
    GemmArgs a{};
    a.M = static_cast<int>(M);
    a.N = static_cast<int>((n_q_heads + 2 * n_kv_heads) * 128);
    a.K = static_cast<int>(K);
    a.num_groups = 1;
    a.C = static_cast<__nv_bfloat16*>(qkv_out);
    a.ldc = a.N;
    a.act = VITA_ACT_NONE;
    a.rope_cos_sin = cos_sin;
    a.rope_pos = positions;
    a.rope_slot = slot_mapping;
    a.k_cache = static_cast<__nv_bfloat16*>(k_cache);
    a.v_cache = static_cast<__nv_bfloat16*>(v_cache);
    a.n_q = static_cast<int>(n_q_heads);
    a.n_kv = static_cast<int>(n_kv_heads);
    a.k_scale = k_scale;
    a.v_scale = v_scale;
    return gemm_dispatch(X, ldx, a.M, W_qkv, a.N, a, false, static_cast<cudaStream_t>(stream), kv8);
}

extern "C" int vita_gemm_qkv_rope(const void* X, int64_t ldx, const void* W_qkv, void* qkv_out, int64_t M, int64_t K,
                                  int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim, const int32_t* positions,
                                  const int32_t* slot_mapping, const float* cos_sin, void* k_cache, void* v_cache,
                                  void* stream) {
    return gemm_qkv_rope(X, ldx, W_qkv, qkv_out, M, K, n_q_heads, n_kv_heads, head_dim, positions, slot_mapping, cos_sin,
                         k_cache, v_cache, stream, false, 1.0f, 1.0f);
}

// the same with e4m3 caches: each K / V row is stored as e4m3_rn_satfinite(bf16 value / scale) (kv_fp8.cuh)
extern "C" int vita_gemm_qkv_rope_fp8(const void* X, int64_t ldx, const void* W_qkv, void* qkv_out, int64_t M,
                                      int64_t K, int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim,
                                      const int32_t* positions, const int32_t* slot_mapping, const float* cos_sin,
                                      void* k_cache, void* v_cache, float k_scale, float v_scale, void* stream) {
    VITA_REQUIRE(kv_fp8_scales_ok(k_scale, v_scale), "k_scale / v_scale must be finite and positive");
    return gemm_qkv_rope(X, ldx, W_qkv, qkv_out, M, K, n_q_heads, n_kv_heads, head_dim, positions, slot_mapping, cos_sin,
                         k_cache, v_cache, stream, true, k_scale, v_scale);
}

extern "C" int vita_moe_gemm_gate_up_silu(const void* X_perm, const void* W_gate_up, void* Act,
                                          const int32_t* expert_offsets, int64_t rows, int64_t num_experts,
                                          int64_t H, int64_t I, void* stream) {
    GemmArgs a{};
    a.M = static_cast<int>(rows);
    a.N = static_cast<int>(I);
    a.K = static_cast<int>(H);
    a.num_groups = static_cast<int>(num_experts);
    a.group_offsets = expert_offsets;
    a.C = static_cast<__nv_bfloat16*>(Act);
    a.ldc = I;
    a.act = VITA_ACT_NONE;
    VITA_REQUIRE(expert_offsets != nullptr, "expert_offsets required");
    VITA_REQUIRE(I % 8 == 0, "I must be a multiple of 8");
    return gemm_dispatch(X_perm, H, a.M, W_gate_up, static_cast<int>(2 * I), a, true,
                         static_cast<cudaStream_t>(stream));
}

// The two grouped GEMMs over the "slot" layout of vita_moe_route_scatter: expert e owns rows [e * capacity,
// e * capacity + expert_counts[e]) of X_slots / Act_slots / Y_slots (counts on the device, no host sync).
extern "C" int vita_moe_gemm_gate_up_silu_slots(const void* X_slots, const void* W_gate_up, void* Act_slots,
                                                const int32_t* expert_counts, int64_t capacity, int64_t rows_hint,
                                                int64_t num_experts, int64_t H, int64_t I, void* stream) {
    VITA_REQUIRE(expert_counts != nullptr && capacity > 0, "expert_counts and capacity required");
    VITA_REQUIRE(I % 8 == 0 && num_experts * capacity < (1ll << 31), "I % 8 == 0 and E * capacity < 2^31");
    GemmArgs a{};
    a.M = static_cast<int>(num_experts * capacity);
    a.N = static_cast<int>(I);
    a.K = static_cast<int>(H);
    a.num_groups = static_cast<int>(num_experts);
    a.group_counts = expert_counts;
    a.group_stride = static_cast<int>(capacity);
    a.est_rows = static_cast<int>(rows_hint);
    a.C = static_cast<__nv_bfloat16*>(Act_slots);
    a.ldc = I;
    a.act = VITA_ACT_NONE;
    return gemm_dispatch(X_slots, H, a.M, W_gate_up, static_cast<int>(2 * I), a, true, static_cast<cudaStream_t>(stream));
}

extern "C" int vita_moe_gemm_down_slots(const void* Act_slots, const void* W_down, void* Y_slots,
                                        const int32_t* expert_counts, const float* row_weight, int64_t capacity,
                                        int64_t rows_hint, int64_t num_experts, int64_t H, int64_t I, void* stream) {
    VITA_REQUIRE(expert_counts != nullptr && capacity > 0, "expert_counts and capacity required");
    VITA_REQUIRE(num_experts * capacity < (1ll << 31), "E * capacity < 2^31");
    GemmArgs a{};
    a.M = static_cast<int>(num_experts * capacity);
    a.N = static_cast<int>(H);
    a.K = static_cast<int>(I);
    a.num_groups = static_cast<int>(num_experts);
    a.group_counts = expert_counts;
    a.group_stride = static_cast<int>(capacity);
    a.est_rows = static_cast<int>(rows_hint);
    a.C = static_cast<__nv_bfloat16*>(Y_slots);
    a.ldc = H;
    a.rowscale = row_weight;
    a.act = VITA_ACT_NONE;
    return gemm_dispatch(Act_slots, I, a.M, W_down, static_cast<int>(H), a, false, static_cast<cudaStream_t>(stream));
}

// Expert-parallel down projection: the GEMM epilogue stores every output row straight into the symmetric-memory
// receive buffer of the rank that owns the token (P2P stores over NVLink), so compute and the "combine" transfer are
// one kernel; the owner later sums its two slots per token (vita_ep_reduce_norm_gather).
extern "C" int vita_moe_gemm_down_ep(const void* Act, const void* W_down, const int32_t* expert_offsets,
                                     const float* row_weight, const int32_t* row_assign, void* const* peer_out,
                                     int64_t rows, int64_t num_local_experts, int64_t H, int64_t I, int64_t chunk,
                                     void* stream) {
    GemmArgs a{};
    a.M = static_cast<int>(rows);
    a.N = static_cast<int>(H);
    a.K = static_cast<int>(I);
    a.num_groups = static_cast<int>(num_local_experts);
    a.group_offsets = expert_offsets;
    a.C = const_cast<__nv_bfloat16*>(static_cast<const __nv_bfloat16*>(Act));   // unused when peer_out is set; keeps checks happy
    a.ldc = H;
    a.rowscale = row_weight;
    a.act = VITA_ACT_NONE;
    a.row_assign = row_assign;
    a.peer_out = reinterpret_cast<__nv_bfloat16* const*>(peer_out);
    a.chunk = static_cast<int>(chunk);
    VITA_REQUIRE(expert_offsets && row_assign && peer_out && chunk > 0, "offsets, row_assign, peer_out and chunk required");
    return gemm_dispatch(Act, I, a.M, W_down, static_cast<int>(H), a, false, static_cast<cudaStream_t>(stream));
}

extern "C" int vita_moe_gemm_down(const void* Act, const void* W_down, void* Y_perm, const int32_t* expert_offsets,
                                  const float* row_weight, int64_t rows, int64_t num_experts, int64_t H, int64_t I,
                                  void* stream) {
    GemmArgs a{};
    a.M = static_cast<int>(rows);
    a.N = static_cast<int>(H);
    a.K = static_cast<int>(I);
    a.num_groups = static_cast<int>(num_experts);
    a.group_offsets = expert_offsets;
    a.C = static_cast<__nv_bfloat16*>(Y_perm);
    a.ldc = H;
    a.rowscale = row_weight;
    a.act = VITA_ACT_NONE;
    VITA_REQUIRE(expert_offsets != nullptr, "expert_offsets required");
    return gemm_dispatch(Act, I, a.M, W_down, static_cast<int>(H), a, false, static_cast<cudaStream_t>(stream));
}
