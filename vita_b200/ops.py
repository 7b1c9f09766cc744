"""torch.Tensor front-ends of the C ABI.  PyTorch is used for device memory and streams only: every function below
marshals pointers/sizes into one libvita_b200.so call on the current CUDA stream.  No arithmetic happens in torch.
"""
from __future__ import annotations

import ctypes
import math
from typing import Optional

import torch

from . import _lib

ACT_NONE, ACT_GELU, ACT_RELU = 0, 1, 2
BF16 = torch.bfloat16
FP8 = torch.float8_e4m3fn      # e4m3 KV cache (include/vita_b200.h, vita_gemm_qkv_rope_fp8)


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _chk(t: torch.Tensor, dtype, name: str, contiguous: bool = True):
    if not t.is_cuda:
        raise _lib.VitaB200Error(f"{name}: expected a CUDA tensor (vita_b200 has no CPU path)")
    if t.dtype != dtype:
        raise _lib.VitaB200Error(f"{name}: expected dtype {dtype}, got {t.dtype}")
    if contiguous and not t.is_contiguous():
        raise _lib.VitaB200Error(f"{name}: expected a contiguous tensor")


def _kv_fp8(k_cache, v_cache, name: str) -> bool:
    """True for an e4m3 cache pair, False for bf16; anything else (or a mixed pair) raises."""
    fp8 = k_cache is not None and k_cache.dtype == FP8
    dt = FP8 if fp8 else BF16
    _chk(k_cache, dt, f"{name}: k_cache"); _chk(v_cache, dt, f"{name}: v_cache")
    return fp8


def _scales(k_scale, v_scale):
    ks, vs = 1.0 if k_scale is None else float(k_scale), 1.0 if v_scale is None else float(v_scale)
    if not (math.isfinite(ks) and math.isfinite(vs) and ks > 0.0 and vs > 0.0):
        raise _lib.VitaB200Error(f"k_scale / v_scale must be finite and positive, got {ks} / {vs}")
    return ks, vs


def _i64arr(vals):
    return (ctypes.c_int64 * len(vals))(*[int(v) for v in vals])


# ------------------------------------------------------------------------------------------------ dense linear
def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: int = ACT_NONE,
           colscale: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
           out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = residual + colscale * act(x @ w.T + bias); x [..., K] (rows may be strided), w [N, K]."""
    _chk(w, BF16, "w")
    K = x.shape[-1]
    N = w.shape[0]
    x2 = x.reshape(-1, K)
    if x2.stride(-1) != 1:
        x2 = x2.contiguous()
    _chk(x2, BF16, "x", contiguous=False)
    M = x2.shape[0]
    if out is None:
        out = torch.empty((M, N), dtype=BF16, device=x.device)
    o2 = out.reshape(-1, N)
    r2 = None
    if residual is not None:
        r2 = residual.reshape(-1, N)
        _chk(r2, BF16, "residual", contiguous=False)
    for t, n in ((bias, "bias"), (colscale, "colscale")):
        if t is not None:
            _chk(t, BF16, n)
    _lib.call("vita_gemm_bf16", _p(x2), x2.stride(0), _p(w), _p(o2), o2.stride(0), M, N, K, _p(bias), act,
              _p(colscale), _p(r2), 0 if r2 is None else r2.stride(0), _stream())
    return out.reshape(*x.shape[:-1], N)


# ------------------------------------------------------------------------------------------------ row kernels
def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _chk(x, BF16, "x"); _chk(w, BF16, "w")
    H = x.shape[-1]
    if out is None:
        out = torch.empty_like(x)
    _lib.call("vita_rmsnorm", _p(x), _p(w), _p(out), x.numel() // H, H, float(eps), _stream())
    return out


def layernorm(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float, act: int = ACT_NONE,
              out_scale: float = 1.0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _chk(x, BF16, "x"); _chk(w, BF16, "w"); _chk(b, BF16, "b")
    H = x.shape[-1]
    if out is None:
        out = torch.empty_like(x)
    _lib.call("vita_layernorm", _p(x), _p(w), _p(b), _p(out), x.numel() // H, H, float(eps), act, float(out_scale),
              _stream())
    return out


def row_copy(table: torch.Tensor, src_index: Optional[torch.Tensor], dst_index: Optional[torch.Tensor],
             out: torch.Tensor, n_rows: int) -> torch.Tensor:
    _chk(table, BF16, "table"); _chk(out, BF16, "out")
    for t, n in ((src_index, "src_index"), (dst_index, "dst_index")):
        if t is not None:
            _chk(t, torch.int32, n)
    _lib.call("vita_row_copy", _p(table), _p(src_index), _p(dst_index), _p(out), n_rows, table.shape[-1], _stream())
    return out


def rope_kv_write(qkv: torch.Tensor, positions: torch.Tensor, slot_mapping: Optional[torch.Tensor],
                  cos_sin: torch.Tensor, k_cache: Optional[torch.Tensor], v_cache: Optional[torch.Tensor],
                  n_q: int, n_kv: int, head_dim: int) -> None:
    _chk(qkv, BF16, "qkv"); _chk(positions, torch.int32, "positions"); _chk(cos_sin, torch.float32, "cos_sin")
    if k_cache is not None and k_cache.dtype == FP8:
        raise _lib.VitaB200Error("rope_kv_write: e4m3 caches are not supported (linear_qkv_rope writes them)")
    if slot_mapping is not None:
        _chk(slot_mapping, torch.int32, "slot_mapping"); _chk(k_cache, BF16, "k_cache"); _chk(v_cache, BF16, "v_cache")
    _lib.call("vita_rope_kv_write", _p(qkv), _p(positions), _p(slot_mapping), _p(cos_sin), _p(k_cache), _p(v_cache),
              qkv.shape[0], n_q, n_kv, head_dim, _stream())


def linear_qkv_rope(x: torch.Tensor, w_qkv: torch.Tensor, out: torch.Tensor, positions: torch.Tensor,
                    slot_mapping: Optional[torch.Tensor], cos_sin: torch.Tensor, k_cache: Optional[torch.Tensor],
                    v_cache: Optional[torch.Tensor], n_q: int, n_kv: int, head_dim: int,
                    k_scale: Optional[float] = None, v_scale: Optional[float] = None) -> torch.Tensor:
    """qkv projection with RoPE + paged-KV append in the GEMM epilogue (== linear() then rope_kv_write(), one kernel).
    e4m3 caches (float8_e4m3fn) store each row as e4m3(bf16 row / scale) with the layer's k_scale / v_scale (default 1)."""
    _chk(x, BF16, "x", contiguous=False); _chk(w_qkv, BF16, "w_qkv"); _chk(out, BF16, "out")
    _chk(positions, torch.int32, "positions"); _chk(cos_sin, torch.float32, "cos_sin")
    M, K = x.shape
    if x.stride(1) != 1 or w_qkv.shape != ((n_q + 2 * n_kv) * head_dim, K) or out.shape != (M, w_qkv.shape[0]):
        raise _lib.VitaB200Error("linear_qkv_rope: shape mismatch")
    if positions.numel() < M or (slot_mapping is not None and slot_mapping.numel() < M):
        raise _lib.VitaB200Error("linear_qkv_rope: positions / slot_mapping shorter than the row count")
    fp8 = False
    if slot_mapping is not None:
        _chk(slot_mapping, torch.int32, "slot_mapping"); fp8 = _kv_fp8(k_cache, v_cache, "linear_qkv_rope")
    if fp8:
        ks, vs = _scales(k_scale, v_scale)
        _lib.call("vita_gemm_qkv_rope_fp8", _p(x), x.stride(0), _p(w_qkv), _p(out), M, K, n_q, n_kv, head_dim,
                  _p(positions), _p(slot_mapping), _p(cos_sin), _p(k_cache), _p(v_cache), ks, vs, _stream())
        return out
    _lib.call("vita_gemm_qkv_rope", _p(x), x.stride(0), _p(w_qkv), _p(out), M, K, n_q, n_kv, head_dim, _p(positions),
              _p(slot_mapping), _p(cos_sin), _p(k_cache), _p(v_cache), _stream())
    return out


# ------------------------------------------------------------------------------------------------ attention
def attention(q, k, v, out, q_strides, k_strides, v_strides, o_strides, B, n_q, n_kv, Sq, Skv, d_qk, d_v,
              kv_lens: Optional[torch.Tensor], causal: bool, scale: float, q_pos0: int = 0) -> torch.Tensor:
    """q/k/v/out: bf16 CUDA tensors (views allowed); *_strides = (batch, token, head) in elements.  causal: query
    row i attends keys <= q_pos0 + i."""
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        _chk(t, BF16, n, contiguous=False)
    if kv_lens is not None:
        _chk(kv_lens, torch.int32, "kv_lens")
    _lib.call("vita_attention_fwd", _p(q), _p(k), _p(v), _p(out), _i64arr(q_strides), _i64arr(k_strides),
              _i64arr(v_strides), _i64arr(o_strides), B, n_q, n_kv, Sq, Skv, d_qk, d_v, _p(kv_lens), int(causal),
              int(q_pos0), float(scale), _stream())
    return out


class PagedPrefill:
    """Work list of one step's prompt continuations for attention_prefill_paged, built once per step and reused by
    every layer.  query_start_loc (B + 1, host): sequence i owns the packed rows [qsl[i], qsl[i + 1]); ctx_lens[i]
    (host) counts its keys, cached prefix and new rows, all in the pages of block_table[i].  Only the sequences in
    `seqs` (default: all) are attended; one tile per (sequence, 128-row query block), longest causal rows first."""

    def __init__(self, query_start_loc, ctx_lens, block_table: torch.Tensor, page_size: int, seqs=None):
        qsl, ctx = [int(x) for x in query_start_loc], [int(x) for x in ctx_lens]
        B = len(ctx)
        seqs = list(range(B)) if seqs is None else [int(i) for i in seqs]
        if len(qsl) != B + 1 or block_table.dim() != 2 or block_table.shape[0] < B:
            raise _lib.VitaB200Error("PagedPrefill: query_start_loc, ctx_lens and block_table rows do not match")
        _chk(block_table, torch.int32, "block_table", contiguous=False)
        if block_table.stride(1) != 1:
            raise _lib.VitaB200Error("PagedPrefill: block_table rows must be contiguous")
        tiles = []
        for i in seqs:
            c, n = qsl[i + 1] - qsl[i], ctx[i]
            if not 0 < c <= n or qsl[i] < 0 or qsl[i + 1] > qsl[-1]:
                raise _lib.VitaB200Error(f"PagedPrefill: sequence {i} has {c} new rows and a context of {n}")
            if (n + page_size - 1) // page_size > block_table.shape[1]:
                raise _lib.VitaB200Error(f"PagedPrefill: a context of {n} needs more than {block_table.shape[1]} pages")
            tiles += [(n - c + 128 * b, i, b) for b in range((c + 127) // 128)]
        tiles.sort(key=lambda t: -t[0])
        self.T, self.page_size, self.block_table, self.n_tiles = qsl[-1], int(page_size), block_table, len(tiles)
        buf = torch.tensor([x for t in tiles for x in t[1:]] + qsl + ctx, dtype=torch.int32).to(block_table.device)
        n = 2 * len(tiles)
        self.tiles, self.qsl, self.ctx = buf[:n], buf[n:n + B + 1], buf[n + B + 1:]
        self._seqs, self._ctx_host, self._stage = seqs, ctx, None

    def fp8_stage(self, k_cache: torch.Tensor):
        """The e4m3 path's staging of this plan, built on first use and reused by every layer: (work [n, 3] int32
        device: (sequence, page index, scratch page) of every page a planned sequence reads, the remapped block table
        [B, pages] pointing at the scratch pages, k / v scratch [pages * page_size, n_kv, head_dim] bf16).  The scratch
        covers the whole context of every planned sequence (4 KiB per token for K and V together at 8 kv heads) and
        is allocated once per plan, i.e. once per step, from torch's caching allocator."""
        if self._stage is None:
            ps, work = self.page_size, []
            B = self.block_table.shape[0]
            width = max((c + ps - 1) // ps for c in self._ctx_host) if self._ctx_host else 1
            table = [[0] * width for _ in range(B)]
            for i in self._seqs:
                for pi in range((self._ctx_host[i] + ps - 1) // ps):
                    table[i][pi] = len(work)
                    work.append((i, pi, len(work)))
            dev = self.block_table.device
            n_pages = max(len(work), 1)
            shape = (n_pages * ps,) + tuple(k_cache.shape[1:])
            self._stage = (torch.tensor(work, dtype=torch.int32).reshape(-1, 3).to(dev),
                           torch.tensor(table, dtype=torch.int32).to(dev),
                           torch.empty(shape, dtype=BF16, device=dev), torch.empty(shape, dtype=BF16, device=dev))
        return self._stage


def attention_prefill_paged(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, plan: PagedPrefill,
                            out: torch.Tensor, n_q: int, n_kv: int, head_dim: int, scale: float,
                            k_scale: Optional[float] = None, v_scale: Optional[float] = None) -> torch.Tensor:
    """Causal attention of prompt continuations over the paged cache (include/vita_b200.h).  q [T, >= n_q * head_dim]
    (rows may be strided, e.g. the packed qkv), k/v_cache [slots, n_kv, head_dim], out [T, n_q * head_dim] (rows may
    be strided); row r of sequence i attends its keys <= ctx_lens[i] - (qsl[i + 1] - qsl[i]) + r.  Rows of sequences
    outside the plan are left as they are.  e4m3 caches: the plan's pages are dequantized into a bf16 scratch first
    (vita_kv_fp8_stage_pages, one launch) and the same kernel runs on it."""
    _chk(q, BF16, "q", contiguous=False); _chk(out, BF16, "out", contiguous=False)
    fp8 = _kv_fp8(k_cache, v_cache, "attention_prefill_paged")
    if q.shape[0] != plan.T or out.shape[0] != plan.T or q.stride(1) != 1 or out.stride(1) != 1 \
            or out.shape[1] < n_q * head_dim or k_cache.shape != v_cache.shape or k_cache.dim() != 3 \
            or tuple(k_cache.shape[1:]) != (n_kv, head_dim):
        raise _lib.VitaB200Error("attention_prefill_paged: shape mismatch")
    bt = plan.block_table
    if fp8:
        ks, vs = _scales(k_scale, v_scale)
        work, bt, k16, v16 = plan.fp8_stage(k_cache)
        _lib.call("vita_kv_fp8_stage_pages", _p(k_cache), _p(v_cache), _p(plan.block_table), plan.block_table.stride(0),
                  _p(plan.ctx), _p(work), work.shape[0], _p(k16), _p(v16), n_kv, head_dim, plan.page_size, ks, vs,
                  _stream())
        k_cache, v_cache = k16, v16
    _lib.call("vita_attention_prefill_paged", _p(q), q.stride(0), _p(k_cache), _p(v_cache), k_cache.shape[0], _p(bt),
              bt.stride(0), _p(plan.qsl), _p(plan.ctx), _p(plan.tiles), plan.n_tiles, _p(out), out.stride(0), plan.T,
              n_q, n_kv, head_dim, plan.page_size, float(scale), _stream())
    return out


def decode_attention_workspace(B: int, n_kv: int, splits: int, device) -> torch.Tensor:
    n = _lib.load().vita_decode_attention_workspace_bytes(B, n_kv, splits)
    return torch.zeros(n, dtype=torch.uint8, device=device)


def decode_attention_merge(B: int, n_kv: int, splits: int) -> str:
    """The split merge decode_attention takes for this shape under the current options: "tagged" or "ticket"."""
    return "tagged" if _lib.load().vita_decode_attention_merge(B, n_kv, splits) else "ticket"


def decode_attention(q, k_cache, v_cache, block_table, cur_pos, out, workspace, n_q, n_kv, head_dim, page_size,
                     splits, scale, q_stride: int = 0, k_scale: Optional[float] = None,
                     v_scale: Optional[float] = None) -> torch.Tensor:
    """e4m3 caches are read as bf16(c * scale) with the layer's k_scale / v_scale (default 1)."""
    _chk(q, BF16, "q", contiguous=False); fp8 = _kv_fp8(k_cache, v_cache, "decode_attention")
    _chk(out, BF16, "out")
    _chk(block_table, torch.int32, "block_table"); _chk(cur_pos, torch.int32, "cur_pos")
    B = cur_pos.shape[0]
    if fp8:
        ks, vs = _scales(k_scale, v_scale)
        _lib.call("vita_decode_attention_fp8", _p(q), _p(k_cache), _p(v_cache), _p(block_table), _p(cur_pos), _p(out),
                  _p(workspace), B, n_q, n_kv, head_dim, page_size, block_table.shape[1], splits, float(scale),
                  q_stride, ks, vs, _stream())
        return out
    _lib.call("vita_decode_attention", _p(q), _p(k_cache), _p(v_cache), _p(block_table), _p(cur_pos), _p(out),
              _p(workspace), B, n_q, n_kv, head_dim, page_size, block_table.shape[1], splits, float(scale), q_stride,
              _stream())
    return out


def decode_slots(cur_pos, block_table, slots, page_size):
    _lib.call("vita_decode_slots", _p(cur_pos), _p(block_table), _p(slots), cur_pos.shape[0], page_size,
              block_table.shape[1], _stream())


def argmax_rows(logits, best):
    _chk(logits, BF16, "logits"); _chk(best, torch.int64, "best")
    _lib.call("vita_argmax_rows", _p(logits), _p(best), logits.shape[0], logits.shape[1], _stream())


def _chk_streams(streams, B: int, name: str):
    if streams is not None:
        _chk(streams, torch.int32, "streams")
        if streams.numel() < B:
            raise _lib.VitaB200Error(f"{name}: streams has fewer than {B} rows")


def sample_rows(logits, temperature, top_k, top_p, seed, counter, best, scores: Optional[torch.Tensor] = None,
                streams: Optional[torch.Tensor] = None):
    """Sampled next token per row into the packed arg-max words `best` (contract: vita_b200/sampling.py).
    logits [B, V] bf16 (rows may be strided); temperature / top_p f32 [B], top_k / counter i32 [B], seed i64 [B]
    (the 64-bit Philox key, bit pattern); scores [B, rows, V] or [rows, V] (B = 1) bf16: row counter[b] receives
    the warped logits.  streams (i32 [B], optional; None = stream 0): the stream index of each row's draw."""
    _chk(logits, BF16, "logits", contiguous=False); _chk(best, torch.int64, "best")
    _chk(temperature, torch.float32, "temperature"); _chk(top_p, torch.float32, "top_p")
    _chk(top_k, torch.int32, "top_k"); _chk(counter, torch.int32, "counter"); _chk(seed, torch.int64, "seed")
    B, V = logits.shape
    if logits.stride(1) != 1:
        raise _lib.VitaB200Error("sample_rows: logits rows must be contiguous")
    for t, n in ((temperature, "temperature"), (top_k, "top_k"), (top_p, "top_p"), (seed, "seed"),
                 (counter, "counter"), (best, "best")):
        if t.numel() < B:
            raise _lib.VitaB200Error(f"sample_rows: {n} has fewer than {B} rows")
    rows = 0
    if scores is not None:
        _chk(scores, BF16, "scores")
        if scores.dim() == 2:
            scores = scores.unsqueeze(0)
        if scores.shape[0] < B or scores.shape[2] != V:
            raise _lib.VitaB200Error("sample_rows: scores must be [B, rows, V]")
        rows = scores.shape[1]
    _chk_streams(streams, B, "sample_rows")
    _lib.call("vita_sample_rows_streams", _p(logits), logits.stride(0), B, V, _p(temperature), _p(top_k), _p(top_p),
              _p(seed), _p(counter), _p(streams), None, _p(best), _p(scores), V, rows, None, None, None, None, 0, 0,
              0, 0, _stream())


def sample_logprobs(logits, temperature, top_k, top_p, seed, counter, best, logprob, rank, top_ids, top_logprobs,
                    n_top: int, target: Optional[torch.Tensor] = None, scores: Optional[torch.Tensor] = None,
                    log_softmax_scores: bool = False, streams: Optional[torch.Tensor] = None):
    """`sample_rows` plus log-probabilities over the processed row (contract: vita_b200/sampling.py).
    `target` (i32 [B], optional): rows with target[b] in [0, V) score that token and draw nothing (best[b] gets the
    greedy word); the other rows score the token they choose.  Outputs: logprob f32 / rank i32 of shape [B] (row b) or
    [B, rows] (row counter[b] of request b, a device-resident log); top_ids i32 / top_logprobs f32 of that shape plus
    a last dimension >= n_top (0 <= n_top <= 20): the n_top largest logits, lowest index first on ties.
    `log_softmax_scores`: the score rows receive bf16(logprob) of every token (HF beam search's scores) instead of the
    processed row.  `streams` as for `sample_rows`."""
    _chk(logits, BF16, "logits", contiguous=False); _chk(best, torch.int64, "best")
    _chk(temperature, torch.float32, "temperature"); _chk(top_p, torch.float32, "top_p")
    _chk(top_k, torch.int32, "top_k"); _chk(counter, torch.int32, "counter"); _chk(seed, torch.int64, "seed")
    _chk(logprob, torch.float32, "logprob"); _chk(rank, torch.int32, "rank")
    B, V = logits.shape
    if logits.stride(1) != 1:
        raise _lib.VitaB200Error("sample_logprobs: logits rows must be contiguous")
    for t, n in ((temperature, "temperature"), (top_k, "top_k"), (top_p, "top_p"), (seed, "seed"),
                 (counter, "counter"), (best, "best"), (logprob, "logprob"), (rank, "rank")):
        if t.shape[0] < B:
            raise _lib.VitaB200Error(f"sample_logprobs: {n} has fewer than {B} rows")
    if logprob.shape != rank.shape or logprob.dim() not in (1, 2):
        raise _lib.VitaB200Error("sample_logprobs: logprob and rank must both be [B] or [B, rows]")
    out_rows = logprob.shape[1] if logprob.dim() == 2 else 0
    top_ld = 0
    if n_top > 0:
        _chk(top_ids, torch.int32, "top_ids"); _chk(top_logprobs, torch.float32, "top_logprobs")
        if top_ids.shape != top_logprobs.shape or tuple(top_ids.shape[:-1]) != tuple(logprob.shape) \
                or top_ids.shape[-1] < n_top:
            raise _lib.VitaB200Error("sample_logprobs: top_ids / top_logprobs must be logprob's shape + [>= n_top]")
        top_ld = top_ids.shape[-1]
    if target is not None:
        _chk(target, torch.int32, "target")
        if target.numel() < B:
            raise _lib.VitaB200Error(f"sample_logprobs: target has fewer than {B} rows")
    rows = 0
    if scores is not None:
        _chk(scores, BF16, "scores")
        if scores.dim() == 2:
            scores = scores.unsqueeze(0)
        if scores.shape[0] < B or scores.shape[2] != V:
            raise _lib.VitaB200Error("sample_logprobs: scores must be [B, rows, V]")
        rows = scores.shape[1]
    _chk_streams(streams, B, "sample_logprobs")
    _lib.call("vita_sample_rows_streams", _p(logits), logits.stride(0), B, V, _p(temperature), _p(top_k), _p(top_p),
              _p(seed), _p(counter), _p(streams), _p(target), _p(best), _p(scores), V, rows, _p(logprob), _p(rank),
              _p(top_ids) if n_top > 0 else None, _p(top_logprobs) if n_top > 0 else None, int(n_top), top_ld,
              out_rows, int(log_softmax_scores), _stream())


def kv_copy_pages(layer_base: torch.Tensor, pairs: torch.Tensor, n_pages: int, page_bytes: int):
    """Copy page src over page dst for every (src, dst) row of pairs (i32 [n, 2]) in every cache whose base address
    is in layer_base (i64 [n_bases]: the K and V cache of each layer, n_pages pages of page_bytes each).  One launch."""
    _chk(layer_base, torch.int64, "layer_base"); _chk(pairs, torch.int32, "pairs")
    if pairs.dim() != 2 or pairs.shape[1] != 2:
        raise _lib.VitaB200Error("kv_copy_pages: pairs must be [n, 2]")
    _lib.call("vita_kv_copy_pages", _p(layer_base), layer_base.numel(), _p(pairs), pairs.shape[0], int(n_pages),
              int(page_bytes), _stream())


def page_digest(rows: torch.Tensor, page_size: int) -> torch.Tensor:
    """128-bit digest of every full page of prompt rows (include/vita_b200.h vita_page_digest): rows bf16 [n, H]
    (rows may be strided) -> int64 [n // page_size, 2], the bits of the two u64 lanes.  A partial last page gets none."""
    _chk(rows, BF16, "rows", contiguous=False)
    if rows.dim() != 2 or rows.stride(1) != 1:
        raise _lib.VitaB200Error("page_digest: rows must be [n, H] with contiguous rows")
    out = torch.empty(rows.shape[0] // page_size, 2, dtype=torch.int64, device=rows.device)
    _lib.call("vita_page_digest", _p(rows), rows.stride(0), rows.shape[0], rows.shape[1], int(page_size), _p(out),
              _stream())
    return out


# ------------------------------------------------------------------------------------------------ MoE (prefill)
def moe_router(h, norm_w, gate_w, xn, topk_ids, topk_w, eps):
    _chk(h, BF16, "h"); _chk(norm_w, BF16, "norm_w"); _chk(gate_w, BF16, "gate_w"); _chk(xn, BF16, "xn")
    _chk(topk_ids, torch.int32, "topk_ids"); _chk(topk_w, torch.float32, "topk_w")
    n_tok, H = h.shape
    _lib.call("vita_moe_router", _p(h), _p(norm_w), _p(gate_w), _p(xn), _p(topk_ids), _p(topk_w), n_tok, H,
              gate_w.shape[0], float(eps), _stream())


def moe_align(topk_ids, topk_w, expert_offsets, perm_row, row_token, row_weight, n_tok, E, row_assign=None):
    for t, n in ((topk_ids, "topk_ids"), (expert_offsets, "expert_offsets"), (perm_row, "perm_row"),
                 (row_token, "row_token")):
        _chk(t, torch.int32, n)
    _chk(topk_w, torch.float32, "topk_w"); _chk(row_weight, torch.float32, "row_weight")
    _lib.call("vita_moe_align", _p(topk_ids), _p(topk_w), _p(expert_offsets), _p(perm_row), _p(row_token),
              _p(row_weight), _p(row_assign), n_tok, E, _stream())


def moe_down_ep(act, w_down, expert_offsets, row_weight, row_assign, peer_out_ptrs, rows, chunk):
    """Down projection of the local experts; the epilogue pushes each row to its token's owner over NVLink."""
    _chk(act, BF16, "act"); _chk(w_down, BF16, "w_down"); _chk(peer_out_ptrs, torch.int64, "peer_out_ptrs")
    E, H, I = w_down.shape
    _lib.call("vita_moe_gemm_down_ep", _p(act), _p(w_down), _p(expert_offsets), _p(row_weight), _p(row_assign),
              _p(peer_out_ptrs), rows, E, H, I, chunk, _stream())


def ep_signal(peer_flag_ptrs, which, n_ranks, my_rank, epoch):
    _lib.call("vita_ep_signal", _p(peer_flag_ptrs), which, n_ranks, my_rank, epoch, _stream())


def ep_wait(my_flags, which, n_ranks, epoch, n_wait: Optional[int] = None):
    _lib.call("vita_ep_wait", _p(my_flags), which, n_ranks, n_ranks if n_wait is None else n_wait, epoch, _stream())


def ep_push(peer_base_ptrs, ranges, n_ranks, my_rank):
    """All-gather by P2P stores: `ranges` = [(byte offset, bytes), ...] (<= 4) of this rank's symmetric buffer."""
    offs = _i64arr([r[0] for r in ranges])
    nbytes = _i64arr([r[1] for r in ranges])
    _lib.call("vita_ep_push", _p(peer_base_ptrs), offs, nbytes, len(ranges), n_ranks, my_rank, _stream())


def ep_reduce_norm_gather(rs_buf, my_flags, peer_h_ptrs, peer_xn_ptrs, next_norm_w, tok0, n_owned, n_ranks, my_rank,
                          epoch, H, eps, gather: bool = True):
    _lib.call("vita_ep_reduce_norm_gather", _p(rs_buf), _p(my_flags), _p(peer_h_ptrs), _p(peer_xn_ptrs),
              _p(next_norm_w), tok0, n_owned, n_ranks, my_rank, epoch, H, float(eps), int(gather), _stream())


def moe_gate_up(x_perm, w_gate_up, act, expert_offsets, rows):
    _chk(x_perm, BF16, "x_perm"); _chk(w_gate_up, BF16, "w_gate_up"); _chk(act, BF16, "act")
    E, two_i, H = w_gate_up.shape
    _lib.call("vita_moe_gemm_gate_up_silu", _p(x_perm), _p(w_gate_up), _p(act), _p(expert_offsets), rows, E, H,
              two_i // 2, _stream())


def moe_down(act, w_down, y_perm, expert_offsets, row_weight, rows):
    _chk(act, BF16, "act"); _chk(w_down, BF16, "w_down"); _chk(y_perm, BF16, "y_perm")
    E, H, I = w_down.shape
    _lib.call("vita_moe_gemm_down", _p(act), _p(w_down), _p(y_perm), _p(expert_offsets), _p(row_weight), rows, E, H, I,
              _stream())


def moe_route_scatter(h, norm_w, gate_w, x_slots, expert_counts, perm_row, row_weight, eps, topk_ids=None, topk_w=None):
    """Fused router + permute: x_slots [E * capacity, H], expert_counts [E] (zero on entry)."""
    _chk(h, BF16, "h"); _chk(norm_w, BF16, "norm_w"); _chk(gate_w, BF16, "gate_w"); _chk(x_slots, BF16, "x_slots")
    _chk(expert_counts, torch.int32, "expert_counts"); _chk(perm_row, torch.int32, "perm_row")
    _chk(row_weight, torch.float32, "row_weight")
    n_tok, H = h.shape
    E = gate_w.shape[0]
    capacity = x_slots.shape[0] // E
    if row_weight.numel() < E * capacity or perm_row.numel() < 2 * n_tok or expert_counts.numel() < E:
        raise _lib.VitaB200Error("moe_route_scatter: output buffers too small")
    _lib.call("vita_moe_route_scatter", _p(h), _p(norm_w), _p(gate_w), _p(x_slots), _p(expert_counts), _p(perm_row),
              _p(row_weight), _p(topk_ids), _p(topk_w), n_tok, H, E, capacity, float(eps), _stream())


def moe_gate_up_slots(x_slots, w_gate_up, act_slots, expert_counts, rows_hint):
    _chk(x_slots, BF16, "x_slots"); _chk(w_gate_up, BF16, "w_gate_up"); _chk(act_slots, BF16, "act_slots")
    E, two_i, H = w_gate_up.shape
    _lib.call("vita_moe_gemm_gate_up_silu_slots", _p(x_slots), _p(w_gate_up), _p(act_slots), _p(expert_counts),
              x_slots.shape[0] // E, rows_hint, E, H, two_i // 2, _stream())


def moe_down_slots(act_slots, w_down, y_slots, expert_counts, row_weight, rows_hint):
    _chk(act_slots, BF16, "act_slots"); _chk(w_down, BF16, "w_down"); _chk(y_slots, BF16, "y_slots")
    E, H, I = w_down.shape
    _lib.call("vita_moe_gemm_down_slots", _p(act_slots), _p(w_down), _p(y_slots), _p(expert_counts), _p(row_weight),
              act_slots.shape[0] // E, rows_hint, E, H, I, _stream())


def moe_combine(h, y_perm, perm_row, next_norm_w, xn_out, eps):
    _chk(h, BF16, "h"); _chk(y_perm, BF16, "y_perm"); _chk(perm_row, torch.int32, "perm_row")
    n_tok, H = h.shape
    _lib.call("vita_moe_combine", _p(h), _p(y_perm), _p(perm_row), _p(next_norm_w), _p(xn_out), n_tok, H, float(eps),
              _stream())


# ------------------------------------------------------------------------------------------------ InternViT glue
def vit_im2col(images, out, P, k_pad):
    _chk(images, BF16, "images"); _chk(out, BF16, "out")
    n, C, HW, _ = images.shape
    _lib.call("vita_vit_im2col", _p(images), _p(out), n, C, HW, P, k_pad, _stream())


def vit_assemble(patches, cls, pos, out, n_img, n_patch, H):
    for t, nm in ((patches, "patches"), (cls, "cls"), (pos, "pos"), (out, "out")):
        _chk(t, BF16, nm)
    _lib.call("vita_vit_assemble", _p(patches), _p(cls), _p(pos), _p(out), n_img, n_patch, H, _stream())


def vit_pixel_shuffle(h, out, n_img, grid, C, scale):
    _chk(h, BF16, "h"); _chk(out, BF16, "out")
    _lib.call("vita_vit_pixel_shuffle", _p(h), _p(out), n_img, grid, C, float(scale), _stream())


# ------------------------------------------------------------------------------------------------ image front end
def image_resample_u8(img: torch.Tensor, axis: int, out_size: int, kk: torch.Tensor, bounds: torch.Tensor) -> torch.Tensor:
    """One Pillow-exact bicubic pass over `axis` of an interleaved [H, W, C] uint8 image."""
    _chk(img, torch.uint8, "img"); _chk(kk, torch.int32, "kk"); _chk(bounds, torch.int32, "bounds")
    H, W, C = img.shape
    out = torch.empty((H, out_size, C) if axis == 1 else (out_size, W, C), dtype=torch.uint8, device=img.device)
    _lib.call("vita_image_resample_u8", _p(img), _p(out), H, W, C, axis, out_size, _p(kk), _p(bounds), kk.shape[1],
              _stream())
    return out


def image_tiles_lut(img: torch.Tensor, lut: torch.Tensor, out: torch.Tensor, gi: int, gj: int, T: int, tile0: int) -> None:
    _chk(img, torch.uint8, "img"); _chk(lut, BF16, "lut"); _chk(out, BF16, "out")
    _lib.call("vita_image_tiles_lut", _p(img), _p(lut), _p(out), gi, gj, T, tile0, _stream())


# ------------------------------------------------------------------------------------------------ Whale glue
def fbank(wave, window, mel_weights_t, mel_span, frame_len: int, frame_shift: int, preemph: float) -> torch.Tensor:
    """wave: [n] fp32 on the device, already scaled by 2**15.  Returns [n_frames, n_mel] fp32 (kaldi log-mel)."""
    _chk(wave, torch.float32, "wave"); _chk(window, torch.float32, "window")
    _chk(mel_weights_t, torch.float32, "mel_weights_t"); _chk(mel_span, torch.int32, "mel_span")
    n = wave.numel()
    n_mel = mel_weights_t.shape[1]
    n_frames = 0 if n < frame_len else 1 + (n - frame_len) // frame_shift
    out = torch.empty(n_frames, n_mel, dtype=torch.float32, device=wave.device)
    if n_frames:
        _lib.call("vita_fbank", _p(wave), n, _p(window), _p(mel_weights_t), _p(mel_span), _p(out), frame_len,
                  frame_shift, n_mel, float(preemph), _stream())
    return out


def whale_conv1(feat, mean, istd, w, bias, out):
    _chk(feat, torch.float32, "feat"); _chk(w, BF16, "w"); _chk(bias, BF16, "bias"); _chk(out, BF16, "out")
    B, T, F = feat.shape
    _lib.call("vita_whale_conv1", _p(feat), _p(mean), _p(istd), _p(w), _p(bias), _p(out), B, T, F, w.shape[0],
              _stream())


def whale_im2col2(x, out, B, T1, F1, C):
    _chk(x, BF16, "x"); _chk(out, BF16, "out")
    _lib.call("vita_whale_im2col2", _p(x), _p(out), B, T1, F1, C, _stream())


def whale_qk_prep(qkv, p, bias_u, bias_v, q2, k2, B, T, heads, dk):
    for t, nm in ((qkv, "qkv"), (p, "p"), (bias_u, "bias_u"), (bias_v, "bias_v"), (q2, "q2"), (k2, "k2")):
        _chk(t, BF16, nm)
    _lib.call("vita_whale_qk_prep", _p(qkv), _p(p), _p(bias_u), _p(bias_v), _p(q2), _p(k2), B, T, heads, dk, _stream())


def whale_adapter_im2col(x, lengths, out, B, T, C, ksize):
    _chk(x, BF16, "x"); _chk(out, BF16, "out")
    if lengths is not None:
        _chk(lengths, torch.int32, "lengths")
    _lib.call("vita_whale_adapter_im2col", _p(x), _p(lengths), _p(out), B, T, C, ksize, _stream())


# ------------------------------------------------------------------------------------------------ decode step
def decode_embed(best, token_log, gen_count, cache_len, cur_pos, embed, h, max_ctx: int,
                 chain_mem: Optional[torch.Tensor] = None):
    _chk(best, torch.int64, "best"); _chk(token_log, torch.int32, "token_log"); _chk(embed, BF16, "embed")
    B, H = h.shape
    _lib.call("vita_decode_embed", _p(best), _p(token_log), _p(gen_count), token_log.shape[1], _p(cache_len),
              _p(cur_pos), _p(embed), _p(h), B, H, embed.shape[0], int(max_ctx), _p(chain_mem), _stream())


def chain_begin(chain_mem: torch.Tensor):
    """Open a completion-counter chain: chain_mem = int64 [1 + n_links] (serial + one counter per chain kernel)."""
    _chk(chain_mem, torch.int64, "chain_mem")
    _lib.call("vita_chain_begin", _p(chain_mem), chain_mem.numel() - 1)


def chain_end():
    _lib.call("vita_chain_end")


def decode_router(h, norm_w, gate_w, xn, topk_ids, topk_w, eps):
    B, H = h.shape
    _lib.call("vita_decode_router", _p(h), _p(norm_w), _p(gate_w), _p(xn), _p(topk_ids), _p(topk_w), B, H,
              gate_w.shape[0], float(eps), _stream())


# ------------------------------------------------------------------------------------------------ decode step (wgmma)
class TcWorkspace:
    """Cross-CTA reduction scratch of the tensor-core decode kernels (zero-initialised once, self-cleaning)."""

    def __init__(self, B: int, max_row_blocks: int, device):
        n = _lib.load().vita_decode_tc_workspace_bytes(B, max_row_blocks)
        self.buf = torch.zeros(n, dtype=torch.uint8, device=device)
        self.max_row_blocks = max_row_blocks


def decode_tc_qkv_rope(h, norm_w, w_qkv, cos_sin, cur_pos, block_table, q_out, k_cache, v_cache, ws, n_q, n_kv,
                       head_dim, page_size, eps, k_scale: Optional[float] = None, v_scale: Optional[float] = None):
    B, H = h.shape
    if k_cache.dtype == FP8:
        _kv_fp8(k_cache, v_cache, "decode_tc_qkv_rope")
        ks, vs = _scales(k_scale, v_scale)
        _lib.call("vita_decode_tc_qkv_rope_fp8", _p(h), _p(norm_w), _p(w_qkv), _p(cos_sin), _p(cur_pos),
                  _p(block_table), _p(q_out), _p(k_cache), _p(v_cache), _p(ws.buf), ws.max_row_blocks, B, H, n_q, n_kv,
                  head_dim, page_size, block_table.shape[1], float(eps), ks, vs, _stream())
        return
    _lib.call("vita_decode_tc_qkv_rope", _p(h), _p(norm_w), _p(w_qkv), _p(cos_sin), _p(cur_pos), _p(block_table),
              _p(q_out), _p(k_cache), _p(v_cache), _p(ws.buf), ws.max_row_blocks, B, H, n_q, n_kv, head_dim, page_size,
              block_table.shape[1], float(eps), _stream())


def decode_tc_oproj(x, w, h, ws):
    B, N = h.shape
    _lib.call("vita_decode_tc_oproj", _p(x), _p(w), _p(h), _p(ws.buf), ws.max_row_blocks, B, N, w.shape[1], _stream())


def decode_tc_moe_gate_up(h, norm_w, gate_w, w13, topk_ids, topk_w, act, ws, eps, route_word=None, route_tag=0):
    """`route_word` ([B] int64) + `route_tag` (>= 1): publish the routing early for decode_tc_moe_down (see the header)."""
    B, H = h.shape
    _lib.call("vita_decode_tc_moe_gate_up", _p(h), _p(norm_w), _p(gate_w), _p(w13), _p(topk_ids), _p(topk_w), _p(act),
              _p(ws.buf), ws.max_row_blocks, B, H, w13.shape[1] // 2, gate_w.shape[0], float(eps), _p(route_word),
              int(route_tag), _stream())


def decode_tc_moe_down(act, w2, topk_ids, topk_w, h, ws, route_word=None, route_tag=0):
    B, H = h.shape
    _lib.call("vita_decode_tc_moe_down", _p(act), _p(w2), _p(topk_ids), _p(topk_w), _p(h), _p(ws.buf),
              ws.max_row_blocks, B, H, w2.shape[2], w2.shape[0], _p(route_word), int(route_tag), _stream())


def tc_lm_head_argmax(h, h_stride, norm_w, w, logits, best, B, ws, eps):
    V, H = w.shape
    _lib.call("vita_tc_lm_head_argmax", _p(h), h_stride, _p(norm_w), _p(w), _p(logits), _p(best), _p(ws.buf),
              ws.max_row_blocks, B, H, V, float(eps), _stream())


# ------------------------------------------------------------------------------------------------ single-kernel decode
def launch_count(reset: bool = False) -> int:
    return int(_lib.load().vita_launch_count(1 if reset else 0))


def set_option(name: str, value: int) -> None:
    """Library tunable ("pdl", "attn_early", "chain_wait", "tc_prefetch_consts", "tc_wide_route", "tc_l2_ahead", "tc_trigger_lead"); affects launches issued afterwards."""
    _lib.call("vita_set_option", name.encode(), int(value))


def get_option(name: str) -> int:
    return int(_lib.load().vita_get_option(name.encode()))
