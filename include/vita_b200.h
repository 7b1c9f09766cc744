/* libvita_b200.so -- C ABI of the H100-native (sm_90a) kernels behind VITA's omni-modal prefill + decode forward.
 *
 * The reference (VITA-MLLM/VITA) is pure Python and has no FFI of its own: every GPU op is reached through
 * torch / transformers / flash-attn / vLLM wheels.  This header is therefore the boundary a maintainer binds with
 * ctypes (see INTEGRATION.md); each entry point names the reference call site (file:line under the reference tree)
 * whose library kernel it replaces.
 *
 * Conventions
 *   - plain pointers and sizes only; all tensor pointers are DEVICE pointers unless stated otherwise;
 *   - bf16 storage (uint16 payload), fp32 accumulation; row-major; weights are [out_features, in_features]
 *     exactly as torch.nn.Linear stores them;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - every function returns VITA_OK (0) or a negative error code and records a message retrievable with
 *     vita_last_error(); nothing allocates device memory (workspaces are passed in);
 *   - there is no CPU fallback: on a machine without an sm_90 GPU the launches fail with VITA_ERR_CUDA.
 */
#ifndef VITA_B200_H
#define VITA_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VITA_OK 0
#define VITA_ERR_INVALID (-1)
#define VITA_ERR_CUDA (-2)

#define VITA_ACT_NONE 0
#define VITA_ACT_GELU 1 /* erf GELU (torch.nn.GELU default) */
#define VITA_ACT_RELU 2

/* ---- library ---------------------------------------------------------------------------------------------- */
int vita_version(void);
const char* vita_last_error(void);
/* number of SMs of the current device (0 if no CUDA device is usable) */
int vita_num_sms(void);
/* counts kernels launched through this library since the last reset (bench.py's gpu_launches) */
int64_t vita_launch_count(int reset);
/* Tunables (each also has an environment default, INTEGRATION.md section 3): "pdl", "attn_early", "chain_wait",
 * "tc_prefetch_consts", "tc_wide_route", "tc_l2_ahead", "tc_trigger_lead".
 * Takes effect for launches issued afterwards (a captured CUDA graph keeps what it was captured with). */
int vita_set_option(const char* name, int64_t value);
int64_t vita_get_option(const char* name);

/* Decode-chain completion counters (bs = 1 greedy step).  Between vita_chain_begin and vita_chain_end the chain-capable
 * launches of the calling thread (vita_decode_tc_*, vita_decode_attention, vita_tc_lm_head_argmax) are linked in call
 * order: each bumps its own 64-bit counter when its CTAs are done and polls its predecessor's instead of waiting for
 * the grid dependency (which resolves ~3.5 us after the last CTA has exited).  mem = [1 + n_links] uint64, zeroed once
 * (and again after a failed launch); mem[0] is the step serial that vita_decode_embed(..., serial = mem) bumps once per
 * step.  Purely an accelerator: a counter that does not arrive in time falls back to the hardware dependency. */
int vita_chain_begin(uint64_t* mem, int64_t n_links);
int vita_chain_end(void);

/* ---- dense linear:  C[M,N] = residual + colscale * act(A[M,K] . B[N,K]^T + bias) ----------------------------
 * wgmma / TMA GEMM.  Replaces nn.Linear -> cuBLAS at
 *   internvit/modeling_intern_vit.py:180 (qkv), :192 (proj, with ls1 + residual :245-247),
 *   :214,216 (fc1+GELU, fc2 with ls2 + residual :249-251); multimodal_projector/builder.py:164-168;
 *   whale/module/layer/attention.py:371-373,381,419; :145-147; component/subsampling.py:34;
 *   component/transformer.py:313; adapter.py:94,104; transformers MixtralAttention q/k/v/o_proj;
 *   lm_head on all rows (vita_mixtral.py:171-173).
 * bias [N] / colscale [N] / residual [M, ldr] may be NULL.  K, lda, ldc, ldr multiples of 8; 16-byte aligned. */
int vita_gemm_bf16(const void* A, int64_t lda, const void* B, void* C, int64_t ldc, int64_t M, int64_t N, int64_t K,
                   const void* bias, int act, const void* colscale, const void* residual, int64_t ldr, void* stream);

/* ---- row kernels ------------------------------------------------------------------------------------------ */
/* transformers MixtralRMSNorm.forward (modeling_mixtral.py:148-153). */
int vita_rmsnorm(const void* x, const void* w, void* y, int64_t rows, int64_t H, float eps, void* stream);
/* torch.nn.LayerNorm + optional activation + output scale: modeling_intern_vit.py:229-230;
 * whale transformer.py:88-89,313-318 (LayerNorm -> ReLU, then x sqrt(d) attention.py:109),:371; adapter.py:98-104. */
int vita_layernorm(const void* x, const void* w, const void* b, void* y, int64_t rows, int64_t H, float eps, int act,
                   float out_scale, void* stream);
/* out[dst_index[i]] = table[src_index[i]] (NULL index = identity, negative = skip): embed_tokens
 * (vita_arch.py:274), placeholder splice (vita_arch.py:277-303; mixtral.py:1116,1126), MoE token gather. */
int vita_row_copy(const void* table, const int32_t* src_index, const int32_t* dst_index, void* out, int64_t n_rows,
                  int64_t H, void* stream);
/* rotate-half RoPE on the q and k heads of a fused qkv activation, in place, and append k/v to the paged cache
 * (modeling_mixtral.py:224-254; vLLM twin mixtral.py:477-501).  cos_sin fp32 [max_pos, 2, D/2]; slot_mapping[tok] =
 * page * page_size + offset (NULL = do not write the cache). */
int vita_rope_kv_write(void* qkv, const int32_t* positions, const int32_t* slot_mapping, const float* cos_sin,
                       void* k_cache, void* v_cache, int64_t n_tok, int64_t n_q_heads, int64_t n_kv_heads,
                       int64_t head_dim, void* stream);

/* The qkv projection with both of the above in its epilogue: qkv_out[M, (n_q + 2 n_kv) * 128] = X[M, K] . W_qkv^T, the
 * q and k heads rotated with positions[row] (on the bf16-rounded projections, bit-identical to vita_gemm_bf16 followed
 * by vita_rope_kv_write), k / v heads also stored at slot_mapping[row] of the paged caches (NULL = no cache write).
 * Replaces q_proj/k_proj/v_proj + apply_rotary_pos_emb + the cache update of MixtralAttention.forward
 * (modeling_mixtral.py:312-340; vLLM twin mixtral.py:470-501). */
int vita_gemm_qkv_rope(const void* X, int64_t ldx, const void* W_qkv, void* qkv_out, int64_t M, int64_t K,
                       int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim, const int32_t* positions,
                       const int32_t* slot_mapping, const float* cos_sin, void* k_cache, void* v_cache, void* stream);
/* FP8 (e4m3) KV cache, vLLM's kv_cache_dtype="fp8": caches of 1-byte elements in the same [slots, n_kv, head_dim]
 * layout, one k_scale / v_scale per layer (> 0).  Write: c = e4m3_rn_satfinite(float(bf16(x)) / scale), x the row the
 * bf16 entry point stores (fp32 division, round to nearest even, saturation at +-448).  Read: bf16(float(c) * scale).
 * The *_fp8 entry points take the same arguments as their bf16 twins plus the two scales; every other output is
 * bit-identical to the bf16 entry point's. */
int vita_gemm_qkv_rope_fp8(const void* X, int64_t ldx, const void* W_qkv, void* qkv_out, int64_t M, int64_t K,
                           int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim, const int32_t* positions,
                           const int32_t* slot_mapping, const float* cos_sin, void* k_cache, void* v_cache,
                           float k_scale, float v_scale, void* stream);

/* ---- attention -------------------------------------------------------------------------------------------- */
/* softmax(Q K^T * scale [causal] [kv_lens mask]) V, FlashAttention style.  Strides are {batch, token, head} in
 * elements.  Supported (d_qk, d_v): (128,128) Mixtral GQA, (64,64) InternViT, (128,64) Whale rel-pos with the
 * operands prepared by vita_whale_qk_prep.  Replaces flash_attn_varlen_qkvpacked_func
 * (internvit/flash_attention.py:61), whale attention.py:391-415, transformers sdpa (modeling_mixtral.py:269-292).
 * causal: query row i attends keys <= q_pos0 + i (q_pos0 = 0 for a whole sequence; a sequence shard passes the
 * position of its first row). */
int vita_attention_fwd(const void* q, const void* k, const void* v, void* o, const int64_t* q_strides,
                       const int64_t* k_strides, const int64_t* v_strides, const int64_t* o_strides, int64_t B,
                       int64_t n_q_heads, int64_t n_kv_heads, int64_t Sq, int64_t Skv, int64_t d_qk, int64_t d_v,
                       const int32_t* kv_lens, int causal, int64_t q_pos0, float scale, void* stream);
/* causal attention of prompt continuations over a paged KV cache: sequence i owns the packed query rows
 * [query_start_loc[i], query_start_loc[i + 1]) (C_i rows of q, token stride q_token_stride, heads head_dim apart) and
 * ctx_lens[i] = P_i + C_i keys in the pages block_table[i * bt_stride ...], its own keys already appended; row r
 * attends keys <= P_i + r.  k_cache / v_cache: [n_slots, n_kv_heads, head_dim], slot = page * page_size + offset.
 * tiles: n_tiles pairs (sequence, 128-row query block), one CTA per pair and q head, in launch order (longest rows
 * first is fastest).  Pages past ceil(ctx_lens[i] / page_size) are never read; keys at positions >= ctx_lens[i] never
 * reach the output.  The same rows through vita_attention_fwd over the gathered keys give bit-identical output.
 * head_dim 128, page_size 16 / 32 / 64 / 128.  Replaces vLLM's paged attention in MixtralAttention.forward
 * (web_demo/vllm_tools/vllm_file/mixtral.py:484-501) when a prefill continues cached blocks (chunked prefill,
 * prefix caching). */
int vita_attention_prefill_paged(const void* q, int64_t q_token_stride, const void* k_cache, const void* v_cache,
                                 int64_t n_slots, const int32_t* block_table, int64_t bt_stride,
                                 const int32_t* query_start_loc, const int32_t* ctx_lens, const int32_t* tiles,
                                 int64_t n_tiles, void* out, int64_t o_token_stride, int64_t T, int64_t n_q_heads,
                                 int64_t n_kv_heads, int64_t head_dim, int64_t page_size, float scale, void* stream);
/* vita_attention_prefill_paged over e4m3 pages: for each (sequence, page index, scratch page) triple of work, page
 * block_table[sequence * bt_stride + page index] of k_cache / v_cache is dequantized into page `scratch page` of
 * k_out / v_out (bf16, same layout); rows at positions >= ctx_lens[sequence] are written as zeros.  The paged
 * attention then runs on the scratch with a block table that points at the scratch pages, bit for bit the bf16 kernel
 * over the dequantized pages. */
int vita_kv_fp8_stage_pages(const void* k_cache, const void* v_cache, const int32_t* block_table, int64_t bt_stride,
                            const int32_t* ctx_lens, const int32_t* work, int64_t n_work, void* k_out, void* v_out,
                            int64_t n_kv_heads, int64_t head_dim, int64_t page_size, float k_scale, float v_scale,
                            void* stream);
/* single-query paged-KV attention for decode (vLLM paged Attention, mixtral.py:484-501).  workspace must be
 * zero-initialised once and be at least vita_decode_attention_workspace_bytes() large for the largest (B, splits) it
 * is used with; every launch hands it back all-zero, so B and splits may change from call to call.  The context
 * splits of a kv head are merged all-to-all through tagged 64-bit words when splits is 4, 8 or 16 and the grid is
 * resident at once, otherwise by the last CTA to take a ticket ("attn_tagged"). */
int64_t vita_decode_attention_workspace_bytes(int64_t B, int64_t n_kv_heads, int64_t splits);
/* the merge vita_decode_attention takes for (B, n_kv_heads, splits) under the current options: 1 tagged, 0 ticket */
int vita_decode_attention_merge(int64_t B, int64_t n_kv_heads, int64_t splits);
int vita_decode_attention(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_table,
                          const int32_t* cur_pos, void* out, void* workspace, int64_t B, int64_t n_q_heads,
                          int64_t n_kv_heads, int64_t head_dim, int64_t page_size, int64_t max_pages, int64_t splits,
                          float scale, int64_t q_stride /* elements between batch rows of q; 0 = dense */, void* stream);
/* over e4m3 caches: each K / V element is read as bf16(float(c) * scale), the bf16 kernel's arithmetic unchanged (its
 * output bits on the dequantized cache); same workspace, merges and chain protocol */
int vita_decode_attention_fp8(const void* q, const void* k_cache, const void* v_cache, const int32_t* block_table,
                              const int32_t* cur_pos, void* out, void* workspace, int64_t B, int64_t n_q_heads,
                              int64_t n_kv_heads, int64_t head_dim, int64_t page_size, int64_t max_pages,
                              int64_t splits, float scale, int64_t q_stride, float k_scale, float v_scale,
                              void* stream);

/* ---- sparse MoE (prefill) --------------------------------------------------------------------------------- */
/* post_attention_layernorm + MixtralTopKRouter (modeling_mixtral.py:109-116; vLLM FusedMoE renormalize=True,
 * mixtral.py:405-414): writes the normed activations xn, top-2 expert ids and renormalised weights. */
int vita_moe_router(const void* h, const void* norm_w, const void* gate_w, void* xn, int32_t* topk_ids, float* topk_w,
                    int64_t n_tok, int64_t H, int64_t E, float eps, void* stream);
/* stable counting sort of the (token, k) assignments by expert: expert_offsets [E+1], perm_row [n_tok*2],
 * row_token [n_tok*2], row_weight [n_tok*2] (replaces the one_hot / torch.where bookkeeping, modeling_mixtral.py:81-90). */
int vita_moe_align(const int32_t* topk_ids, const float* topk_w, int32_t* expert_offsets, int32_t* perm_row,
                   int32_t* row_token, float* row_weight, int32_t* row_assign /* [n_tok*2] t*2+k per row, may be NULL */,
                   int64_t n_tok, int64_t E, void* stream);
/* grouped expert GEMMs over the permuted rows (modeling_mixtral.py:91-95):
 *   Act[r, :]    = silu(X[r] . Wg_e^T) * (X[r] . Wu_e^T)   with W_gate_up [E, 2I, H] (gate rows first)
 *   Y_perm[r, :] = row_weight[r] * (Act[r] . Wd_e^T)       with W_down [E, H, I] */
int vita_moe_gemm_gate_up_silu(const void* X_perm, const void* W_gate_up, void* Act, const int32_t* expert_offsets,
                               int64_t rows, int64_t num_experts, int64_t H, int64_t I, void* stream);
int vita_moe_gemm_down(const void* Act, const void* W_down, void* Y_perm, const int32_t* expert_offsets,
                       const float* row_weight, int64_t rows, int64_t num_experts, int64_t H, int64_t I, void* stream);
/* h[t] += Y_perm[perm_row[t,0]] + Y_perm[perm_row[t,1]] (index_add_ + residual, modeling_mixtral.py:96,386-389);
 * if next_norm_w != NULL also writes xn_out = RMSNorm(h) for the next layer / final norm. */
/* Fused top-2 router + token permute ("slot" layout): as vita_moe_router, but instead of xn / an offsets pass / a gather
 * pass the CTA of a token claims one row in each of its two experts' slot ranges (expert e owns rows [e * capacity,
 * (e + 1) * capacity) of x_slots; expert_counts[e], zero on entry, counts the claimed rows) and stores the normed
 * activations there; perm_row[t, k] = the claimed row, row_weight[row] = the renormalised routing weight.  topk_ids /
 * topk_w (optional) as vita_moe_router.  The grouped GEMMs *_slots walk the same layout; vita_moe_combine gathers by
 * perm_row.  Row order inside an expert is arrival order; results do not depend on it (rows are independent). */
int vita_moe_route_scatter(const void* h, const void* norm_w, const void* gate_w, void* x_slots, int32_t* expert_counts,
                           int32_t* perm_row, float* row_weight, int32_t* topk_ids, float* topk_w, int64_t n_tok,
                           int64_t H, int64_t E, int64_t capacity, float eps, void* stream);
int vita_moe_gemm_gate_up_silu_slots(const void* X_slots, const void* W_gate_up, void* Act_slots,
                                     const int32_t* expert_counts, int64_t capacity, int64_t rows_hint,
                                     int64_t num_experts, int64_t H, int64_t I, void* stream);
int vita_moe_gemm_down_slots(const void* Act_slots, const void* W_down, void* Y_slots, const int32_t* expert_counts,
                             const float* row_weight, int64_t capacity, int64_t rows_hint, int64_t num_experts, int64_t H,
                             int64_t I, void* stream);
int vita_moe_combine(void* h, const void* y_perm, const int32_t* perm_row, const void* next_norm_w, void* xn_out,
                     int64_t n_tok, int64_t H, float eps, void* stream);

/* ---- expert-parallel MoE over NVLink peer memory (fused compute + collective) -----------------------------
 * vita_moe_gemm_down_ep: the down-projection GEMM whose epilogue stores each (token, k) output row directly into the
 * receive buffer of the rank that owns the token (peer_out[rank] -> [chunk, 2, H] bf16 in symmetric memory).
 * vita_ep_signal / vita_ep_wait: epoch flags in symmetric memory (flags [2][n_ranks] per rank; which = 0 "rows
 * landed", 1 "h/xn gathered").  vita_ep_reduce_norm_gather: the owner sums its two slots per token into the residual
 * stream, applies the next RMSNorm and writes both rows into every rank's h / xn (all-gather by P2P stores). */
int vita_moe_gemm_down_ep(const void* Act, const void* W_down, const int32_t* expert_offsets, const float* row_weight,
                          const int32_t* row_assign, void* const* peer_out, int64_t rows, int64_t num_local_experts,
                          int64_t H, int64_t I, int64_t chunk, void* stream);
int vita_ep_signal(void* const* peer_flags, int64_t which, int64_t n_ranks, int64_t my_rank, int64_t epoch, void* stream);
/* waits for flags[which][src] >= epoch of the sources src < n_wait (n_wait = n_ranks: everybody) */
int vita_ep_wait(const int32_t* my_flags, int64_t which, int64_t n_ranks, int64_t n_wait, int64_t epoch, void* stream);
/* gather = 1: the reduced rows go to every rank's h / xn; gather = 0: to this rank's only (sequence-sharded stream) */
int vita_ep_reduce_norm_gather(const void* rs_buf, const int32_t* my_flags, void* const* peer_h, void* const* peer_xn,
                               const void* next_norm_w, int64_t tok0, int64_t n_owned, int64_t n_ranks, int64_t my_rank,
                               int64_t epoch, int64_t H, float eps, int64_t gather, void* stream);
/* all-gather by P2P stores: up to 4 byte ranges [offset, offset + bytes) of this rank's symmetric buffer
 * (peer_base[my_rank]) are copied to the same offsets of every other rank's buffer.  Offsets are multiples of 16,
 * sizes of 4.  Used for the K/V rows and the routed activations of a sequence shard. */
int vita_ep_push(void* const* peer_base, const int64_t* offsets, const int64_t* bytes, int64_t n_ranges,
                 int64_t n_ranks, int64_t my_rank, void* stream);

/* ---- InternViT front / back end --------------------------------------------------------------------------- */
/* im2col for Conv2d(3,1024,k=14,s=14) (modeling_intern_vit.py:80-85,109): out [n_img*(HW/P)^2, k_pad]. */
int vita_vit_im2col(const void* images, void* out, int64_t n_img, int64_t C, int64_t HW, int64_t P, int64_t k_pad,
                    void* stream);
/* cat([cls, patches]) + position_embedding (modeling_intern_vit.py:112-121). */
int vita_vit_assemble(const void* patches, const void* cls, const void* pos, void* out, int64_t n_img, int64_t n_patch,
                      int64_t H, void* stream);
/* drop CLS, x scale, pixel_shuffle(0.5) (internvit_encoder.py:35-53,71-77): [n,1+g*g,C] -> [n,(g/2)^2,4C]. */
int vita_vit_pixel_shuffle(const void* h, void* out, int64_t n_img, int64_t grid, int64_t C, float scale,
                           void* stream);

/* ---- image front end ---------------------------------------------------------------------------------------- */
/* One separable pass of Pillow's 8-bit resampler (what `image.resize(...)` runs inside the reference's
 * dynamic_preprocess, data_utils_video_audio_neg_patch.py:1239,1253; Pillow src/libImaging/Resample.c):
 *   out[o, p, c] = clip8((2^21 + sum_k in[bounds[o][0] + k, p, c] * kk[o][k]) >> 22),  k < bounds[o][1]
 * along `axis` (1 = horizontal pass: [H, W, C] -> [H, out_size, C]; 0 = vertical pass: [H, W, C] -> [out_size, W, C])
 * of an interleaved uint8 image.  kk [out_size, ksize] int32 fixed-point coefficients and bounds [out_size, 2] come
 * from the host (vita_b200/image_frontend.py::resample_tables = Resample.c precompute_coeffs + normalize_coeffs_8bpc).
 * Pillow's order for a 2-D resize: horizontal pass first, then vertical. */
int vita_image_resample_u8(const uint8_t* in, uint8_t* out, int64_t H, int64_t W, int64_t C, int axis,
                           int64_t out_size, const int32_t* kk, const int32_t* bounds, int64_t ksize, void* stream);
/* Tiling (dynamic_preprocess :1241-1250, row-major T x T tiles of a [gj*T, gi*T, 3] image) fused with
 * CLIPImageProcessor's rescale + normalise through a [3, 256] bf16 table (mm_utils.py:30-43):
 * out[tile0 + ty*gi + tx][c][y][x] = lut[c][img[ty*T + y][tx*T + x][c]];  out is [N, 3, T, T] bf16. */
int vita_image_tiles_lut(const uint8_t* img, const void* lut, void* out, int64_t gi, int64_t gj, int64_t T,
                         int64_t tile0, void* stream);

/* ---- Whale audio front end -------------------------------------------------------------------------------- */
/* Kaldi log-mel filterbank = torchaudio.compliance.kaldi.fbank as the reference calls it in
 * audioEncoderProcessor.process (whale/init_model.py:48-56: 25 ms povey window, 10 ms shift, snip_edges, DC removal,
 * pre-emphasis 0.97 with the first sample replicated, 512-point power spectrum, log floored at FLT_EPSILON; dither 0).
 * wave: [n_samples] fp32, already multiplied by 2^15 (init_model.py:47); window: [frame_len]; mel_weights_t:
 * [256, n_mel] (fft bin major) triangular filters; mel_span: [n_mel, 2] = [first, last) non-zero bin of each filter;
 * out: [n_frames, n_mel] fp32 with n_frames = 1 + (n_samples - frame_len) / frame_shift (0 frames: no launch).
 * Output feeds vita_whale_conv1 directly. */
int vita_fbank(const float* wave, int64_t n_samples, const float* window, const float* mel_weights_t,
               const int32_t* mel_span, float* out, int64_t frame_len, int64_t frame_shift, int64_t n_mel,
               float preemph, void* stream);
/* GlobalCMVN (cmvn.py:21-32, mean/istd may be NULL) + Conv2d(1,C,3,2) + ReLU (subsampling.py:28-29); feat fp32
 * [B,T,F]; out channels-last [B,T1,F1,C]. */
int vita_whale_conv1(const float* feat, const float* mean, const float* istd, const void* w, const void* bias,
                     void* out, int64_t B, int64_t T, int64_t F, int64_t C, void* stream);
/* im2col for Conv2d(C,C,3,2) on the channels-last map (subsampling.py:30): out [B*T2*F2, 9*C]. */
int vita_whale_im2col2(const void* in, void* out, int64_t B, int64_t T1, int64_t F1, int64_t C, void* stream);
/* rel-pos attention operands (attention.py:379-398): Q2 = [q+u | q+v], K2 = [k | p], each [B*T, heads, 2*dk]. */
int vita_whale_qk_prep(const void* qkv, const void* p, const void* bias_u, const void* bias_v, void* q2, void* k2,
                       int64_t B, int64_t T, int64_t heads, int64_t dk, void* stream);
/* adapter front (adapter.py:112-121): mask padded frames, right-pad k-1, im2col for Conv1d(C,2C,k,stride 2). */
int vita_whale_adapter_im2col(const void* x, const int32_t* lengths, void* out, int64_t B, int64_t T, int64_t C,
                              int64_t ksize, void* stream);

/* ---- greedy decode step: small kernels --------------------------------------------------------------------- */
/* consume the previous arg-max (best[b]), append it to token_log, advance cache_len, gather its embedding.
 * max_ctx = KV capacity per sequence (pages * page_size): cur_pos saturates at max_ctx - 1.
 * chain_serial (may be NULL): step serial of the completion-counter chain, bumped once per call. */
int vita_decode_embed(uint64_t* best, int32_t* token_log, int32_t* gen_count, int64_t max_log, int32_t* cache_len,
                      int32_t* cur_pos, const void* embed, void* h, int64_t B, int64_t H, int64_t vocab,
                      int64_t max_ctx, uint64_t* chain_serial, void* stream);
/* post_attention_layernorm + router (top-2 of 8) as a stand-alone kernel (the decode step uses the fused form below). */
int vita_decode_router(const void* h, const void* norm_w, const void* gate_w, void* xn, int32_t* topk_ids,
                       float* topk_w, int64_t B, int64_t H, int64_t E, float eps, void* stream);
/* batched decode through the GEMM path: per-sequence KV slots of the current positions, row-wise arg-max of bf16
 * logits into the packed `best` words the decode chain consumes. */
int vita_decode_slots(const int32_t* cur_pos, const int32_t* block_table, int32_t* slots, int64_t B, int64_t page_size,
                      int64_t max_pages, void* stream);
int vita_argmax_rows(const void* logits, uint64_t* best, int64_t B, int64_t V, void* stream);
/* Sampled next token per row (temperature, top-k, top-p, Gumbel-max draw; the contract is stated in
 * vita_b200/csrc/sample.cu and INTEGRATION.md section 2).  Replaces vLLM's Sampler at
 * web_demo/vllm_tools/vllm_file/mixtral.py:1180-1186 and the sampling loop of HF generate() as called from
 * video_audio_demo.py:257-270.  logits [B, ld] bf16 (first V columns); per-row device arrays temperature f32
 * (0 = greedy: the packed word of vita_argmax_rows), top_k i32 (<= 0 or >= V: off), top_p f32 (>= 1: off),
 * seed u64 (Philox key), counter i32 (index of the token being drawn within its request).  best [B]: packed
 * (logit, ~index) like vita_argmax_rows.  scores (may be NULL): [B, score_rows, score_ld] bf16; row counter[b] of
 * request b receives the warped row (x = l / T, -inf outside the kept set; the logits for greedy rows).
 * V <= 82288 on an H100 (the row is staged in shared memory next to 64 KB of histograms).  Launched as a programmatic
 * dependent: it waits for the preceding kernel before its first read of any input (the counter may be written by an
 * earlier kernel of the same step) and lets its dependents start only when it has completed. */
int vita_sample_rows(const void* logits, int64_t ld, int64_t B, int64_t V, const float* temperature,
                     const int32_t* top_k, const float* top_p, const uint64_t* seed, const int32_t* counter,
                     uint64_t* best, void* scores, int64_t score_ld, int64_t score_rows, void* stream);
/* vita_sample_rows plus log-probabilities over the processed row (the logits for greedy rows; x = l / T over the kept
 * set and -inf outside it otherwise; contract in vita_b200/sampling.py).  target (may be NULL): [B] i32; a row with
 * target[b] in [0, V) draws nothing, leaves the greedy word in best[b] and scores target[b] (prompt rows: the next
 * prompt token); other rows score the token they choose.  Per row: logprob f32 (log-sum-exp from u64 fixed-point
 * masses: independent of summation order and batch position), rank i32 (1 + kept tokens with a strictly greater
 * logit), and the n_top (0 .. 20, <= V) largest logits (lowest index first on ties) as top_ids i32 / top_logprobs f32
 * [.., top_ld].  Output row of request b: b when out_rows == 0, else b * out_rows + counter[b] (skipped outside
 * [0, out_rows)), so a device-resident log works under CUDA-graph replay. */
int vita_sample_rows_logprobs(const void* logits, int64_t ld, int64_t B, int64_t V, const float* temperature,
                              const int32_t* top_k, const float* top_p, const uint64_t* seed, const int32_t* counter,
                              const int32_t* target, uint64_t* best, void* scores, int64_t score_ld,
                              int64_t score_rows, float* logprob, int32_t* rank, int32_t* top_ids,
                              float* top_logprobs, int64_t n_top, int64_t top_ld, int64_t out_rows, void* stream);
/* vita_sample_rows_logprobs whose score rows receive the processed row's log-softmax instead: bf16(logprob(r)) of
 * every token, logprob(r) = x_r - x_max - log Z from the same Z as the logprob outputs (-inf outside the kept set).
 * HF beam search's per-step scores (the running beams' log-softmax rows). */
int vita_sample_rows_logsoftmax(const void* logits, int64_t ld, int64_t B, int64_t V, const float* temperature,
                                const int32_t* top_k, const float* top_p, const uint64_t* seed,
                                const int32_t* counter, const int32_t* target, uint64_t* best, void* scores,
                                int64_t score_ld, int64_t score_rows, float* logprob, int32_t* rank, int32_t* top_ids,
                                float* top_logprobs, int64_t n_top, int64_t top_ld, int64_t out_rows, void* stream);
/* The three sampler entry points above with a per-row stream index: streams (may be NULL: 0 everywhere) [B] i32, the
 * third Philox counter word of row b's draw, counter (r >> 2, counter[b], streams[b], 0).  The sequences of one
 * request share its key and draw from streams 0 .. N-1 (parallel sampling); stream 0 is bit for bit the entry points
 * above.  With logprob and rank both NULL this is vita_sample_rows (target must be NULL and log_softmax 0);
 * otherwise vita_sample_rows_logprobs, or vita_sample_rows_logsoftmax when log_softmax != 0.  Read after the
 * programmatic-dependency wait like every other input. */
int vita_sample_rows_streams(const void* logits, int64_t ld, int64_t B, int64_t V, const float* temperature,
                             const int32_t* top_k, const float* top_p, const uint64_t* seed, const int32_t* counter,
                             const int32_t* streams, const int32_t* target, uint64_t* best, void* scores,
                             int64_t score_ld, int64_t score_rows, float* logprob, int32_t* rank, int32_t* top_ids,
                             float* top_logprobs, int64_t n_top, int64_t top_ld, int64_t out_rows,
                             int64_t log_softmax, void* stream);
/* Copy-on-write of the paged KV cache (vLLM's copy_blocks): for every (src, dst) page pair of pairs [n_pairs, 2] i32
 * (device) and every cache of layer_base [n_bases] (device pointers: the K and the V cache of each layer, each
 * n_pages pages of page_bytes bytes, 16-byte aligned), copy page src over page dst.  One launch, 16-byte vector
 * copies, bit-exact; pairs with an index outside [0, n_pages) are skipped.  The pairs of one launch run concurrently:
 * no dst page may also be a src page of the launch, and no two pairs may share a dst page (beam search's PagePool
 * takes every dst fresh from its free list and copies only pages that are still referenced).  Beam search forks a
 * sequence's cache with it. */
int vita_kv_copy_pages(const uint64_t* layer_base, int64_t n_bases, const int32_t* pairs, int64_t n_pairs,
                       int64_t n_pages, int64_t page_bytes, void* stream);
/* Prefix caching in the continuous batcher: one 128-bit digest of every full page of prompt rows.  rows: bf16
 * [n_rows, H] with row stride ld (>= H, multiple of 8; 16-byte aligned base; H a multiple of 8); out: u64
 * [n_rows / page_size, 2] (a partial last page gets no digest).  Page p's words w_0 .. w_{n-1} are its rows' first
 * H values read as little-endian u64 (H / 4 per row), concatenated row by row; lane l of out[p] is
 *   sum_j splitmix64_finalizer(w_j + j * 0x9E3779B97F4A7C15 + seed_l)  mod 2^64,
 * seed_0 = 0x243F6A8885A308D3, seed_1 = 0x13198A2E03707344.  One CTA per page. */
int vita_page_digest(const void* rows, int64_t ld, int64_t n_rows, int64_t H, int64_t page_size, uint64_t* out,
                     void* stream);
/* ---- greedy decode step on the tensor cores (wgmma swap-AB GEMV, stream-K) ---------------------------------
 * Every linear of the decode step as a weight-streaming GEMV on the tensor cores: the weight tile is the M operand of
 * wgmma and the activation vector as row 0 of a 16-wide N operand; (row-block, k-block) units are split evenly
 * over all SMs and combined through `workspace` (vita_decode_tc_workspace_bytes, zero-initialised once, shared by all
 * five calls; ws_row_blocks = the max_row_blocks it was sized for): K-partials travel as 64-bit {value, tag} words,
 * the CTA that ends on a row block adds them in slot order (deterministic) and clears the tags.  K multiples of 64.
 * With programmatic dependent launch ("pdl") each kernel triggers its successor once its last weight tile is issued
 * and the successor fills its shared-memory ring before the dependency wait. */
int64_t vita_decode_tc_workspace_bytes(int64_t B, int64_t max_row_blocks);
int vita_decode_tc_qkv_rope(const void* h, const void* norm_w, const void* w_qkv, const float* cos_sin,
                            const int32_t* cur_pos, const int32_t* block_table, void* q_out, void* k_cache,
                            void* v_cache, void* workspace, int64_t ws_row_blocks, int64_t B, int64_t H,
                            int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim, int64_t page_size,
                            int64_t max_pages, float eps, void* stream);
/* the same over e4m3 caches (see vita_gemm_qkv_rope_fp8) */
int vita_decode_tc_qkv_rope_fp8(const void* h, const void* norm_w, const void* w_qkv, const float* cos_sin,
                                const int32_t* cur_pos, const int32_t* block_table, void* q_out, void* k_cache,
                                void* v_cache, void* workspace, int64_t ws_row_blocks, int64_t B, int64_t H,
                                int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim, int64_t page_size,
                                int64_t max_pages, float eps, float k_scale, float v_scale, void* stream);
int vita_decode_tc_oproj(const void* x, const void* w, void* h, void* workspace, int64_t ws_row_blocks, int64_t B,
                         int64_t N, int64_t K, void* stream);
/* route_word ([B] 64-bit words, or NULL) + route_tag (1 .. 2^32-1, different for neighbouring launches that share the
 * word, e.g. layer index + 1): the gate|up kernel publishes {tag, e0, e1} as one word as soon as its router is done and
 * triggers its dependent launch right then; the down projection given the same word and tag streams the rows of the
 * selected experts into its shared-memory ring while the gate|up kernel is still running (it still waits for the
 * activations).  NULL: the down projection reads topk_ids after its dependency wait. */
int vita_decode_tc_moe_gate_up(const void* h, const void* norm_w, const void* gate_w, const void* w13,
                               int32_t* topk_ids, float* topk_w, void* act, void* workspace, int64_t ws_row_blocks,
                               int64_t B, int64_t H, int64_t I, int64_t E, float eps, uint64_t* route_word,
                               int64_t route_tag, void* stream);
int vita_decode_tc_moe_down(const void* act, const void* w2, const int32_t* topk_ids, const float* topk_w, void* h,
                            void* workspace, int64_t ws_row_blocks, int64_t B, int64_t H, int64_t I, int64_t E,
                            const uint64_t* route_word, int64_t route_tag, void* stream);
int vita_tc_lm_head_argmax(const void* h, int64_t h_stride, const void* norm_w, const void* w, void* logits,
                           uint64_t* best, void* workspace, int64_t ws_row_blocks, int64_t B, int64_t H, int64_t V,
                           float eps, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VITA_B200_H */
