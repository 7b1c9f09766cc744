"""Mixtral-8x7B sparse-MoE decoder on the CUDA kernels: paged KV cache, prefill, CUDA-graphed greedy or sampled decode.

Replaces the third-party arithmetic the reference reaches through `self.model(...)` / `lm_head`
(vita/model/language_model/vita_mixtral.py:158-173 -> transformers MixtralModel; vLLM twin
web_demo/vllm_tools/vllm_file/mixtral.py:375-628).  Host code only sequences kernels; no arithmetic in torch.
"""
from __future__ import annotations

import gc
import hashlib
import os
from collections import OrderedDict
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import torch

from .. import ops
from ..config import LLMConfig
from ..sampling import MAX_LOGPROBS, SlotSampling, logprob_records

BF16 = torch.bfloat16
FP8 = torch.float8_e4m3fn

KV_CACHE_DTYPES = {"auto": "bf16", "bf16": "bf16", "bfloat16": "bf16", "fp8": "fp8", "fp8_e4m3": "fp8"}


def parse_kv_cache_dtype(name) -> str:
    """vLLM's kv_cache_dtype option -> "bf16" or "fp8" (e4m3, include/vita_b200.h vita_gemm_qkv_rope_fp8).  e5m2 and
    unknown names raise instead of being stored in a format nothing reads back."""
    key = str(name).lower()
    if key in KV_CACHE_DTYPES:
        return KV_CACHE_DTYPES[key]
    if key == "fp8_e5m2":
        raise NotImplementedError("kv_cache_dtype 'fp8_e5m2' is not supported: the fp8 KV cache is e4m3")
    raise ValueError(f"unknown kv_cache_dtype {name!r}; expected one of {sorted(KV_CACHE_DTYPES)}")


def kv_scales(scale, n_layers: int, name: str) -> List[float]:
    """A per-layer scale list from a float or a sequence of n_layers floats (vLLM's k_scale / v_scale)."""
    vals = [float(scale)] * n_layers if isinstance(scale, (int, float)) else [float(x) for x in scale]
    if len(vals) != n_layers or not all(v > 0.0 and v != float("inf") for v in vals):
        raise ValueError(f"{name}: expected a positive float or {n_layers} positive floats, got {scale!r}")
    return vals


def prefix_keys(digests) -> List[bytes]:
    """The prefix-cache keys of a prompt's full pages from their digests (ops.page_digest, [n, 2] int64 on the
    host): key_i = blake2b-128(key_{i-1} || digest_i), key_{-1} empty, so a page's key depends on every row before
    it as well as its own.  Collisions of 128-bit keys are treated as negligible: the cache belongs to one engine and
    is not a boundary between tenants."""
    keys, k = [], b""
    raw = digests.to("cpu", torch.int64).contiguous().numpy().tobytes()
    for i in range(0, len(raw), 16):
        k = hashlib.blake2b(k + raw[i:i + 16], digest_size=16).digest()
        keys.append(k)
    return keys


class PrefixIndex:
    """Host index of the prefix cache: key -> page of the full prompt pages whose KV rows are known, and its inverse.
    Pages without references that are indexed wait in `lru` (least recently released first) to be hit again or
    evicted."""

    def __init__(self):
        self.page: Dict[bytes, int] = {}
        self.key: Dict[int, bytes] = {}
        self.lru: "OrderedDict[int, None]" = OrderedDict()

    def add(self, key: bytes, pg: int) -> bool:
        if key in self.page or pg in self.key:
            return False
        self.page[key], self.key[pg] = pg, key
        return True

    def remove(self, pg: int):
        del self.page[self.key.pop(pg)]
        self.lru.pop(pg, None)


class PagePool:
    """Host page tables with reference counts: copy-on-write sharing of KV pages between sequences (beam search) and
    prompt-prefix sharing across requests (the continuous batcher's prefix cache).

    table[slot][i] is the page of positions [i * page_size, (i + 1) * page_size) of the slot, -1 for none.  At
    construction and after reset() every slot owns its row of `static`, the table at rest (rebase() takes a new one).  A forked or reordered slot holds the
    pages that cover its `length` tokens: full pages are shared (they are never written again), and the page its next
    row lands in (index length // page_size) is private to it.  refs[page] counts the table entries that point to the
    page; pages whose count drops to 0 go to `free` and are handed out again, or, when `index` holds them, to the
    index's LRU list of evictable pages.

    Prefix caching (admit / insert / release): a slot's row becomes the shared pages of its prompt's cached prefix,
    then private pages for everything else it can write, then -1.  reset() (every invalidation) clears the index and
    bumps `epoch`."""

    def __init__(self, static: torch.Tensor, page_size: int):
        self.static = static.to("cpu", torch.int32).clone()     # never a view of a device-side table
        self.page_size = page_size
        self.epoch = 0
        self.evictions = 0
        self.reset()

    def rebase(self, static: torch.Tensor):
        self.static = static.to("cpu", torch.int32).clone()
        self.reset()

    def reset(self):
        self.table: List[List[int]] = self.static.tolist()
        self.refs = [0] * self.static.numel()
        for row in self.table:
            for pg in row:
                self.refs[pg] += 1
        self.free: List[int] = []
        self.index = PrefixIndex()
        self.epoch += 1

    def _drop(self, pg: int):
        self.refs[pg] -= 1
        if self.refs[pg] == 0:
            if pg in self.index.key:
                self.index.lru[pg] = None
            else:
                self.free.append(pg)

    def _take(self) -> int:
        """A page nothing references: a free one, else the least recently released indexed one (evicted)."""
        if self.free:
            pg = self.free.pop()
        else:
            assert self.index.lru, "KV page pool exhausted"
            pg = next(iter(self.index.lru))
            self.index.remove(pg)
            self.evictions += 1
        self.refs[pg] += 1
        return pg

    def release(self, slot: int):
        """Drop the references of the slot's row, last page first (its earlier pages stay in the LRU list longer:
        a later page is useless once an earlier one of its chain is evicted)."""
        for i in reversed(range(len(self.table[slot]))):
            if self.table[slot][i] >= 0:
                self._drop(self.table[slot][i])
                self.table[slot][i] = -1

    def admit(self, slot: int, keys: Sequence[bytes], n_pages: int) -> int:
        """The released slot takes the indexed pages of the longest run of `keys` found (refcount + 1), then private
        pages up to `n_pages` in all.  Returns the number of hit pages.  Never fails while every slot row holds at
        most len(static row) pages: the pool has that many pages per slot, so at least n_pages - hits of them are
        free or evictable."""
        row = self.table[slot]
        assert all(pg < 0 for pg in row) and n_pages <= len(row), "admission into a slot that still holds pages"
        hits = 0
        for key in keys[:n_pages]:
            pg = self.index.page.get(key)
            if pg is None:
                break
            self.index.lru.pop(pg, None)
            self.refs[pg] += 1
            row[hits] = pg
            hits += 1
        assert len(self.free) + len(self.index.lru) >= n_pages - hits, "prefix-cache admission cannot fail"
        for i in range(hits, n_pages):
            row[i] = self._take()
        return hits

    def insert(self, slot: int, keys: Sequence[bytes]):
        """Index the slot's first len(keys) pages (its full prompt pages) under their keys; a key or page already
        indexed keeps its entry."""
        for key, pg in zip(keys, self.table[slot]):
            self.index.add(key, pg)

    def swap(self, i: int, j: int):
        self.table[i], self.table[j] = self.table[j], self.table[i]

    def _private_write_pages(self, slots: Sequence[int], length: int) -> List[Tuple[int, int]]:
        """Make page length // page_size of every slot private: a fresh page where there is none, a copy where it is
        shared (the last slot that shares it keeps the original).  Returns the (src, dst) pages to copy."""
        w, pairs = length // self.page_size, []
        for s in slots:
            pg = self.table[s][w]
            if pg >= 0 and self.refs[pg] == 1:
                continue
            if not self.free:
                raise RuntimeError("KV page pool exhausted")
            new = self.free.pop()
            self.refs[new] += 1
            if pg >= 0:
                pairs.append((pg, new))
                self._drop(pg)
            self.table[s][w] = new
        return pairs

    def fork(self, src: int, dsts: Sequence[int], length: int) -> List[Tuple[int, int]]:
        """dsts continue the `length` tokens of src: they share its full pages and get a copy of its partial last
        page.  The pages of the dst rows and src's pages past its tokens return to the pool."""
        n_cover = -(-length // self.page_size)
        assert src not in dsts and length < len(self.table[src]) * self.page_size
        for i, pg in enumerate(self.table[src]):
            if i >= n_cover and pg >= 0:
                self._drop(pg)
                self.table[src][i] = -1
        for d in dsts:
            for pg in self.table[d]:
                if pg >= 0:
                    self._drop(pg)
            self.table[d] = list(self.table[src])
            for pg in self.table[d]:
                if pg >= 0:
                    self.refs[pg] += 1
        return self._private_write_pages([*dsts, src], length)     # src keeps its page

    def fork_reserved(self, src: int, dsts: Sequence[int], length: int, n_pages: int) -> List[Tuple[int, int]]:
        """Parallel sampling: dsts continue the `length` tokens of src and then advance on their own, so each owns, from
        now on, private pages for everything it can write ([length, n_pages * page_size)), as admission guarantees a
        fresh request.  They share src's full pages, take fresh pages (free ones, else evicted indexed ones: `_take`)
        from page length // page_size up to n_pages, and the partial last page of src is copied into their first fresh
        page.  src's row is left as it is; the dst rows' previous pages are released first.  Returns the (src, dst)
        pages to copy.  Never fails: every row holds at most len(static row) pages, so the pages the dsts give up and
        the unreferenced ones cover what they take."""
        ps, full = self.page_size, length // self.page_size
        assert src not in dsts and length < n_pages * ps and n_pages <= len(self.table[src])
        for d in dsts:
            self.release(d)
        pairs = []
        for d in dsts:
            row = self.table[d]
            for i in range(full):
                row[i] = self.table[src][i]
                self.refs[row[i]] += 1
            for i in range(full, n_pages):
                row[i] = self._take()
            if length % ps:
                pairs.append((self.table[src][full], row[full]))
        return pairs

    def reorder(self, parents: Sequence[int], length: int) -> List[Tuple[int, int]]:
        """Slot i (i < len(parents)) continues slot parents[i], every slot holding `length` tokens: each takes its
        parent's row, then the page the next row lands in is made private (one child keeps the parent's page)."""
        rows = [list(self.table[p]) for p in parents]
        for row in rows:
            for pg in row:
                if pg >= 0:
                    self.refs[pg] += 1
        for i, row in enumerate(rows):
            for pg in self.table[i]:
                if pg >= 0:
                    self._drop(pg)
            self.table[i] = row
        return self._private_write_pages(range(len(parents)), length)

    def check(self):
        """Invariants: each count equals the number of table entries pointing to the page; the index maps keys and
        pages one to one; pages with count 0 are exactly the free ones (not indexed) and the evictable ones
        (indexed, in the LRU list)."""
        count = [0] * len(self.refs)
        for row in self.table:
            for pg in row:
                if pg >= 0:
                    count[pg] += 1
        assert count == self.refs, "reference counts do not match the tables"
        ix = self.index
        assert len(ix.page) == len(ix.key) and all(ix.key[pg] == k for k, pg in ix.page.items()), "index is not 1:1"
        unref = [pg for pg, c in enumerate(count) if c == 0]
        assert sorted(self.free) == [pg for pg in unref if pg not in ix.key], "free list does not match"
        assert sorted(ix.lru) == [pg for pg in unref if pg in ix.key], "evictable list does not match"


class PagedKVCache:
    """k/v per layer: [num_pages * page_size, n_kv_heads, head_dim] bf16, or float8_e4m3fn with kv_cache_dtype "fp8"
    (half the bytes; per-layer k_scale / v_scale, written e4m3(bf16 / scale), read bf16(e4m3 * scale));
    block_table [max_batch, pages_per_seq].
    slot_map is derived from block_table, and the serving engine swaps the rows of both together with their slots.
    fork / reorder change block_table rows only; unshare() (and reset()) gives every slot its row from before the
    first of them back, so the two agree again."""

    def __init__(self, cfg: LLMConfig, max_batch: int, max_seq_len: int, device, page_size: int = 16,
                 shuffle_pages: bool = False, storage=None, kv_cache_dtype: str = "auto", k_scale=1.0,
                 v_scale=1.0):
        """`storage(layer, "k" | "v", shape) -> tensor` lets the owner place the pages (e.g. in NVLink symmetric memory
        for the sequence-sharded expert-parallel prefill); default: ordinary device allocations.  `kv_cache_dtype`:
        "auto" / "bf16" or "fp8" / "fp8_e4m3"; `k_scale` / `v_scale`: a float or one per layer (fp8 only)."""
        self.kv_cache_dtype = parse_kv_cache_dtype(kv_cache_dtype)
        self.dtype = FP8 if self.kv_cache_dtype == "fp8" else BF16
        L = cfg.num_hidden_layers
        self.k_scale, self.v_scale = kv_scales(k_scale, L, "k_scale"), kv_scales(v_scale, L, "v_scale")
        if self.kv_cache_dtype == "bf16" and (set(self.k_scale) != {1.0} or set(self.v_scale) != {1.0}):
            raise ValueError("k_scale / v_scale apply to the fp8 KV cache only")
        self.page_size = page_size
        self.pages_per_seq = (max_seq_len + page_size - 1) // page_size
        self.max_seq_len = self.pages_per_seq * page_size
        self.max_batch = max_batch
        n_pages = max_batch * self.pages_per_seq
        slots = n_pages * page_size
        shape = (slots, cfg.num_key_value_heads, cfg.head_dim)
        if storage is None:
            storage = lambda layer, which, shp: torch.zeros(shp, dtype=self.dtype, device=device)
        self.k = [storage(l, "k", shape) for l in range(cfg.num_hidden_layers)]
        self.v = [storage(l, "v", shape) for l in range(cfg.num_hidden_layers)]
        order = torch.randperm(n_pages, generator=torch.Generator().manual_seed(0)) if shuffle_pages \
            else torch.arange(n_pages)
        table = order.view(max_batch, self.pages_per_seq).to(torch.int32)
        self.block_table = table.to(device)
        self.pool = PagePool(table, page_size)
        self.shared = False                  # fork / reorder / admit_prefix changed the tables since the pool's rebase
        self._layer_base = None
        self.slot_map = self._slot_map_rows(table).to(device)                # [max_batch, max_seq_len]
        self.cache_len = torch.zeros(max_batch, dtype=torch.int32, device=device)
        self.cur_pos = torch.zeros(max_batch, dtype=torch.int32, device=device)

    def reset(self):
        self.cache_len.zero_()
        self.cur_pos.zero_()
        self.unshare()

    def _share(self):
        """The first fork / reorder since the table was at rest: the pool starts from block_table's rows as they are
        now (they follow slot_map's rows, which the serving engine may have swapped)."""
        if not self.shared:
            self.pool.rebase(self.block_table.cpu())
            self.shared = True

    def _slot_map_rows(self, table: torch.Tensor) -> torch.Tensor:
        pos, ps = torch.arange(self.max_seq_len), self.page_size
        return (table[:, pos // ps].to(torch.int64) * ps + (pos % ps)[None, :]).to(torch.int32)

    def unshare(self):
        """Give every slot back the block_table (and slot_map) row it had before the first fork / reorder / prefix
        admission, and refill the pool; this also invalidates the prefix index."""
        if self.shared:
            self.pool.reset()
            self.block_table.copy_(self.pool.static)
            self.slot_map.copy_(self._slot_map_rows(self.pool.static))
            self.shared = False

    def admit_prefix(self, slot: int, keys: Sequence[bytes], prompt_len: int, n_pages: int) -> int:
        """Prefix caching: the slot gives up its pages, takes the cached pages of the longest run of its prompt's page
        keys and private pages up to n_pages in all (PagePool.admit); its block_table and slot_map rows are written
        here, once.  Returns the hit length P = page_size * min(pages found, (prompt_len - 1) // page_size): the last
        prompt row is always computed, because it yields the first token."""
        self._share()
        self.pool.release(slot)
        hits = self.pool.admit(slot, keys[:(prompt_len - 1) // self.page_size], n_pages)
        row = torch.tensor([self.pool.table[slot]], dtype=torch.int32)
        self.block_table[slot:slot + 1].copy_(row)
        self.slot_map[slot:slot + 1].copy_(self._slot_map_rows(row))
        return hits * self.page_size

    def fork(self, src: int, dsts: Sequence[int], length: int):
        """PagePool.fork on the device tables; the partial page is copied for the dsts in one kv_copy_pages launch."""
        self._share()
        self._apply(self.pool.fork(src, dsts, length))

    def fork_reserved(self, src: int, dsts: Sequence[int], length: int, n_pages: int):
        """PagePool.fork_reserved on the device tables: the dst rows of block_table and slot_map are written (a
        reused slot prefills through slot_map) and the partial page is copied in one kv_copy_pages launch."""
        self._share()
        pairs = self.pool.fork_reserved(src, dsts, length, n_pages)
        dsts = list(dsts)
        rows = torch.tensor([self.pool.table[d] for d in dsts], dtype=torch.int32)
        self.block_table[dsts] = rows.to(self.block_table.device)
        self.slot_map[dsts] = self._slot_map_rows(rows).to(self.slot_map.device)
        self._copy(pairs)

    def reorder(self, parents: Sequence[int], length: int):
        """PagePool.reorder on the device tables, with one kv_copy_pages launch for the pages it copies."""
        self._share()
        self._apply(self.pool.reorder(parents, length))

    def _apply(self, pairs):
        self.block_table.copy_(torch.tensor(self.pool.table, dtype=torch.int32))
        self._copy(pairs)

    def _copy(self, pairs):
        if not pairs:
            return
        if self._layer_base is None:
            self._layer_base = torch.tensor([t.data_ptr() for t in self.k + self.v], dtype=torch.int64,
                                            device=self.block_table.device)
        row_bytes = self.k[0][0].numel() * self.k[0].element_size()
        ops.kv_copy_pages(self._layer_base, torch.tensor(pairs, dtype=torch.int32).to(self.block_table.device),
                          self.k[0].shape[0] // self.page_size, self.page_size * row_bytes)


@dataclass
class LayerAttention:
    """The attention kernels every layer runs over the packed qkv rows of one call, chosen once per call.
    `whole`: (row0, n) prompts that attend only to themselves (causal FlashAttention over the qkv rows);
    `paged`: the continuations of cached pages (chunked-prefill chunks, prefix-cache hits);
    `decode`: (row0, n, block_table [n, pages], cur_pos [n], workspace) single-token rows over pages of `page_size`."""
    whole: Sequence[Tuple[int, int]] = ()
    paged: Optional[ops.PagedPrefill] = None
    decode: Optional[tuple] = None
    page_size: int = 16

    @staticmethod
    def of_batch(qsl: Sequence[int], seq_lens: Sequence[int], block_tables: torch.Tensor, page_size: int,
                 decode_workspace: Callable[[int], torch.Tensor]) -> "LayerAttention":
        """Flattened batch: sequence i owns rows [qsl[i], qsl[i + 1]) and has seq_lens[i] keys including them.  Rows
        that are the whole context are a prompt, one row is a decode, anything in between continues cached pages.
        The decode rows must be contiguous; decode_workspace(n) gives the decode-attention workspace of n rows."""
        whole, conts, decodes = [], [], []
        for i, sl in enumerate(seq_lens):
            n = qsl[i + 1] - qsl[i]
            if n == sl:
                whole.append((qsl[i], n))
            elif n == 1:
                decodes.append(i)
            elif 1 < n < sl:                                # chunked prefill / prefix caching: continues cached pages
                conts.append(i)
            else:
                raise ValueError(f"sequence {i}: {n} query tokens for a context of {sl}")
        paged = ops.PagedPrefill(qsl, seq_lens, block_tables, page_size, conts) if conts else None
        decode = None
        if decodes:
            d0, nd = qsl[decodes[0]], len(decodes)
            assert [qsl[i] for i in decodes] == list(range(d0, d0 + nd)), "decode tokens must be contiguous"
            cur = torch.tensor([seq_lens[i] - 1 for i in decodes], dtype=torch.int32).to(block_tables.device)
            decode = (d0, nd, block_tables[decodes].contiguous(), cur, decode_workspace(nd))
        return LayerAttention(whole, paged, decode, page_size)

    def __call__(self, qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, out: torch.Tensor,
                 c: LLMConfig, splits: int, k_scale: float = 1.0, v_scale: float = 1.0):
        """e4m3 caches (float8_e4m3fn) are read through bf16(c * scale): the paged FlashAttention over a dequantized
        scratch of the plan's pages, the decode kernel directly.  Whole prompts attend their own bf16 rows."""
        nq, nkv, D, W = c.num_attention_heads, c.num_key_value_heads, c.head_dim, c.qkv_rows
        for r0, n in self.whole:
            q = qkv[r0:r0 + n]
            ops.attention(q, q[:, nq * D:], q[:, (nq + nkv) * D:], out[r0:r0 + n], (0, W, D), (0, W, D), (0, W, D),
                          (0, nq * D, D), 1, nq, nkv, n, n, D, D, None, True, D ** -0.5)
        if self.paged is not None:
            ops.attention_prefill_paged(qkv, k_cache, v_cache, self.paged, out, nq, nkv, D, D ** -0.5, k_scale, v_scale)
        if self.decode is not None:
            r0, n, block_table, cur_pos, workspace = self.decode
            ops.decode_attention(qkv[r0:r0 + n], k_cache, v_cache, block_table, cur_pos, out[r0:r0 + n], workspace, nq,
                                 nkv, D, self.page_size, splits, D ** -0.5, q_stride=W, k_scale=k_scale,
                                 v_scale=v_scale)


class MixtralDecoder:
    def __init__(self, cfg: LLMConfig, weights: dict, device, max_batch: int = 1, max_seq_len: Optional[int] = None,
                 max_new_tokens: int = 1024, page_size: int = 16, decode_splits: int = 16, shuffle_pages: bool = False,
                 kv_cache_dtype: str = "auto", k_scale=1.0, v_scale=1.0,
                 ep_alloc: Optional[Callable[[int], Tuple[torch.Tensor, List[int]]]] = None):
        """`kv_cache_dtype`: "auto" / "bf16" (default) or "fp8" / "fp8_e4m3", an e4m3 paged KV cache at half the bytes
        with per-layer `k_scale` / `v_scale` (a float or one per layer; vLLM's defaults are 1.0).
        `ep_alloc(nbytes) -> (own zeroed uint8 buffer, [base address of every rank's buffer])`: where the
        sequence-sharded expert-parallel prefill gets its symmetric memory; default: NVLink symmetric memory over the
        default process group (`_symm_alloc`)."""
        self.cfg = cfg
        self.w = weights
        self.device = torch.device(device)
        self.max_batch = max_batch
        max_seq_len = max_seq_len or (cfg.tokenizer_model_max_length + max_new_tokens)
        if max_seq_len > cfg.max_position_embeddings:
            raise ValueError(f"max_seq_len {max_seq_len} exceeds max_position_embeddings {cfg.max_position_embeddings}")
        page_rounded = (max_seq_len + page_size - 1) // page_size * page_size
        if page_rounded > weights["rope"].shape[0]:      # cos/sin table sized from the KV capacity, not a constant
            from ..weights import rope_table
            weights["rope"] = rope_table(page_rounded, cfg.head_dim, cfg.rope_theta).to(self.device)
        # expert parallelism: this rank holds experts [e_lo, e_hi) of every layer; the residual stream is sequence
        # sharded: every rank owns S/N tokens for the dense part (qkv, causal attention over the all-gathered K/V,
        # o-proj, router); K/V rows and routed activations are all-gathered and the expert outputs pushed to the token
        # owners by P2P stores over NVLink symmetric memory
        self.ep_rank, self.ep_world = weights.get("ep", (0, 1))
        self.ep_mode = "seq" if self.ep_world > 1 else None
        self.ep_p2p = None
        if parse_kv_cache_dtype(kv_cache_dtype) == "fp8" and self.ep_world > 1:
            raise ValueError("the fp8 KV cache is single-GPU: the expert-parallel prefill all-gathers bf16 K/V rows")
        storage = None
        if self.ep_mode == "seq":
            assert max_batch == 1 and not shuffle_pages, "sequence-sharded EP serves one sequence with in-order pages"
            storage = self._init_ep_seq(page_rounded, ep_alloc or self._symm_alloc)
        self.cache = PagedKVCache(cfg, max_batch, max_seq_len, device, page_size, shuffle_pages, storage,
                                  kv_cache_dtype, k_scale, v_scale)
        self.max_new_tokens = max_new_tokens
        self.decode_splits = int(os.environ.get("VITA_B200_ATTN_SPLITS", decode_splits))
        H, I = cfg.hidden_size, cfg.intermediate_size
        B = max_batch
        dev = self.device
        # decode-step state (all device resident: a step needs no host input, so it can be replayed as a CUDA graph)
        self.best = torch.zeros(B, dtype=torch.int64, device=dev)         # packed (logit, ~index) arg-max
        self.token_log = torch.zeros(B, max_new_tokens + 8, dtype=torch.int32, device=dev)
        self.gen_count = torch.zeros(B, dtype=torch.int32, device=dev)
        self.sampling = SlotSampling(B, dev)                              # per-slot sampler parameters
        self.d_h = torch.zeros(B, H, dtype=BF16, device=dev)
        self.d_q = torch.zeros(B, cfg.num_attention_heads * cfg.head_dim, dtype=BF16, device=dev)
        self.d_attn = torch.zeros_like(self.d_q)
        self.d_xn = torch.zeros(B, H, dtype=BF16, device=dev)
        self.d_ids = torch.zeros(B, 2, dtype=torch.int32, device=dev)
        self.d_w = torch.zeros(B, 2, dtype=torch.float32, device=dev)
        self.d_route = torch.zeros(B, dtype=torch.int64, device=dev)      # early routing hand-over gate|up -> down
        self.d_act = torch.zeros(B, 2, I, dtype=BF16, device=dev)
        self.d_logits = torch.zeros(B, cfg.vocab_size, dtype=BF16, device=dev)
        self.attn_ws = ops.decode_attention_workspace(B, cfg.num_key_value_heads, self.decode_splits, dev)
        # decode linears: wgmma swap-AB GEMVs (decode_tc.cu); their stream-K partial sums meet in one workspace
        if H % 64 or I % 128:
            raise ValueError("the decode GEMVs need hidden_size % 64 == 0 and intermediate_size % 128 == 0")
        max_rb = max((cfg.vocab_size + 127) // 128, 2 * (I // 128), cfg.num_attention_heads
                     + 2 * cfg.num_key_value_heads, (H + 127) // 128)
        self.tc_ws = ops.TcWorkspace(B, max_rb, dev)
        # completion counters of the bs = 1 decode chain: [serial, one counter per chain kernel (5 per layer + LM head)]
        self.chain_mem = torch.zeros(2 + 5 * cfg.num_hidden_layers, dtype=torch.int64, device=dev)
        self._graphs = {}             # single-sequence decode step: captured CUDA graph per (B, want_logits[, sampled])
        self.scores_buf = None        # [max_new_tokens + 1, V] logits log of slot 0 (generate(output_scores=True))
        self.lp_log = None            # per-slot logprob log (enable_logprob_log)
        self.beam_scores = None       # per-slot log-softmax log of beam search (enable_beam_score_log)
        self._bgraphs = {}            # batched decode step: captured CUDA graph per (batch size, sampled)
        self.d_slots = torch.zeros(B, dtype=torch.int32, device=dev)
        self._prefill_ws = {}
        # router decisions of every layer (the reference returns them as `router_logits` when asked,
        # vita_mixtral.py:108,185-190): set to a list to have prefill() and the eager decode steps append one
        # (top-2 ids [T, 2] int32, renormalised weights [T, 2] fp32) pair per layer
        self.route_trace: Optional[list] = None
        # decode: the gate|up kernel can publish the expert pair as soon as its router is done so that the down projection
        # streams its weight rows while gate|up is still running.  Bit-identical; not measured on H100:
        # off unless VITA_B200_EARLY_ROUTE=1
        self.early_route = os.environ.get("VITA_B200_EARLY_ROUTE", "0") == "1"
        per = cfg.num_local_experts // self.ep_world
        self.e_lo, self.e_hi = self.ep_rank * per, (self.ep_rank + 1) * per
        assert weights["layers"][0]["w13"].shape[0] == per, "expert tensors do not match the EP layout"

    def _symm_alloc(self, nbytes: int):
        """NVLink symmetric memory over the default process group: (own zeroed uint8 buffer, base address of every
        rank's buffer), returned once every rank has zeroed its buffer."""
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm_mem
        sym = symm_mem.empty(nbytes, dtype=torch.uint8, device=self.device)
        sym.zero_()
        torch.cuda.synchronize()
        hdl = symm_mem.rendezvous(sym, dist.group.WORLD)
        delta = sym.data_ptr() - int(hdl.buffer_ptrs[hdl.rank])
        bases = [int(p) + delta for p in hdl.buffer_ptrs]
        assert hdl.world_size == self.ep_world and hdl.rank == self.ep_rank
        self._symm_hdl = hdl
        dist.barrier()
        return sym, bases

    def _init_ep_seq(self, S_max: int, alloc: Callable[[int], Tuple[torch.Tensor, List[int]]]):
        """One symmetric allocation (`alloc`, see __init__) for the sequence-sharded expert-parallel prefill: receive
        slots of the combine, residual stream / normed rows (own tokens), the all-gathered post-attention activations
        with their routing records, epoch flags, and the K/V pages of every layer.  Returns the page-storage callback."""
        c, N, dev = self.cfg, self.ep_world, self.device
        H, L = c.hidden_size, c.num_hidden_layers
        kv_row = c.num_key_value_heads * c.head_dim * 2                       # bytes of one K (or V) row
        chunk_max = self.ep_chunk(S_max)
        al = lambda n: (n + 255) // 256 * 256
        names = ["rs", "h", "xn", "xn2", "ids", "tw", "flags", "kv"]
        sizes = [al(chunk_max * 2 * H * 2), al(S_max * H * 2), al(S_max * H * 2), al(S_max * H * 2), al(S_max * 8),
                 al(S_max * 8), al(4 * N * 4), 2 * L * al(S_max * kv_row)]
        offs = [0]
        for z in sizes:
            offs.append(offs[-1] + z)
        sym, bases = alloc(offs[-1])
        assert sym.dtype == torch.uint8 and sym.numel() == offs[-1] and len(bases) == N
        off = dict(zip(names, offs))
        view = lambda n, dt: sym[off[n]:off[n] + sizes[names.index(n)]].view(dt)
        ptrs = lambda n: torch.tensor([b + off[n] for b in bases], dtype=torch.int64, device=dev)
        kv_layer = al(S_max * kv_row)
        self.ep_p2p = dict(
            sym=sym, chunk_max=chunk_max, off=off, kv_layer=kv_layer, kv_row=kv_row,
            base_ptrs=torch.tensor(bases, dtype=torch.int64, device=dev),
            rs=view("rs", BF16), h=view("h", BF16)[:S_max * H].view(S_max, H),
            xn=view("xn", BF16)[:S_max * H].view(S_max, H), xn2=view("xn2", BF16)[:S_max * H].view(S_max, H),
            ids=view("ids", torch.int32)[:S_max * 2].view(S_max, 2),      # (the regions are padded to 256 bytes)
            tw=view("tw", torch.float32)[:S_max * 2].view(S_max, 2), flags=view("flags", torch.int32),
            rs_ptrs=ptrs("rs"), h_ptrs=ptrs("h"), xn_ptrs=ptrs("xn"), flag_ptrs=ptrs("flags"), epoch=0)

        def storage(layer, which, shape):
            assert shape[0] == S_max, "K/V pages of the sequence-sharded prefill: one sequence, in-order pages"
            o = off["kv"] + (2 * layer + (which == "v")) * kv_layer
            return sym[o:o + S_max * kv_row].view(BF16).view(shape)
        return storage

    def ep_chunk(self, S: int) -> int:
        """Tokens per rank of the sequence-sharded stream (multiple of 8: 16-byte aligned routing records)."""
        from ..parallel import sequence_chunk
        return sequence_chunk(S, self.ep_world)

    # ------------------------------------------------------------------------------------------ prefill
    def _ws(self, S: int):
        """Prefill workspaces, grown geometrically and reused."""
        cap = self._prefill_ws.get("cap", 0)
        if S > cap:
            c = self.cfg
            cap = max(S, 2 * cap, 128)
            # the batched-step graphs reference the old workspaces; cleared in place because a _replay whose warm-up
            # grows them stores its new graph into this same dict
            self._bgraphs.clear()
            H, I, E, dev = c.hidden_size, c.intermediate_size, c.num_local_experts, self.device
            with torch.inference_mode(False):      # reused across calls: keep them ordinary tensors
                self._prefill_ws = self._alloc_ws(cap, H, I, E, dev)
        return self._prefill_ws

    def _alloc_ws(self, cap, H, I, E, dev):
        c = self.cfg
        e = lambda *shape, dt=BF16: torch.empty(*shape, dtype=dt, device=dev)
        # MoE activations in the "slot" layout of the fused router + permute: expert e owns rows [e * cap, (e + 1) * cap)
        # (any expert may receive every token).  The compact buffers of the align / gather flow of expert parallelism
        # are the first 2 * cap rows of the same storage.
        xs, acts, ys, rws = e(E * cap, H), e(E * cap, I), e(E * cap, H), e(E * cap, dt=torch.float32)
        return dict(
            cap=cap, xn=e(cap, H), qkv=e(cap, c.qkv_rows), attn=e(cap, c.num_attention_heads * c.head_dim),
            ids=e(cap, 2, dt=torch.int32), tw=e(cap, 2, dt=torch.float32),
            offs=e(E + 1, dt=torch.int32), perm=e(cap * 2, dt=torch.int32), rtok=e(cap * 2, dt=torch.int32),
            xs=xs, acts=acts, ys=ys, rws=rws,
            cnt=torch.zeros(c.num_hidden_layers, E, dtype=torch.int32, device=dev),
            rw=rws[:cap * 2], xp=xs[:cap * 2], act=acts[:cap * 2], rassign=e(cap * 2, dt=torch.int32),
            pos=torch.arange(cap, dtype=torch.int32, device=dev))

    def run_layers(self, h: torch.Tensor, pos: torch.Tensor, slots: torch.Tensor, k_cache: Sequence[torch.Tensor],
                   v_cache: Sequence[torch.Tensor], attention: LayerAttention, final_norm: bool) -> torch.Tensor:
        """Every layer over the T rows of the residual stream h [T, H] (updated in place): qkv projection + RoPE at
        `pos` + K/V append at `slots` of k_cache[l] / v_cache[l], `attention`, o-proj + residual, fused top-2 MoE.
        Returns xn [T, H] (workspace rows): the final RMSNorm(h) when `final_norm`, not written by the last layer
        otherwise."""
        c, w = self.cfg, self.w
        T = h.shape[0]
        nq, nkv, D = c.num_attention_heads, c.num_key_value_heads, c.head_dim
        ws = self._ws(T)
        xn, qkv, attn, perm = ws["xn"][:T], ws["qkv"][:T], ws["attn"][:T], ws["perm"][:2 * T]
        tracing = self.route_trace is not None and not torch.cuda.is_current_stream_capturing()
        ids, tw = (ws["ids"][:T], ws["tw"][:T]) if tracing else (None, None)
        layers = w["layers"]
        ws["cnt"].zero_()              # per-layer expert counters of the fused router + permute
        ops.rmsnorm(h, layers[0]["ln1"], c.rms_norm_eps, out=xn)
        for li, lw in enumerate(layers):
            # qkv projection, RoPE and the KV append in one kernel (GEMM epilogue)
            ks, vs = self.cache.k_scale[li], self.cache.v_scale[li]
            ops.linear_qkv_rope(xn, lw["wqkv"], qkv, pos, slots, w["rope"], k_cache[li], v_cache[li], nq, nkv, D, ks, vs)
            attention(qkv, k_cache[li], v_cache[li], attn, c, self.decode_splits, ks, vs)
            ops.linear(attn, lw["wo"], residual=h, out=h)
            # router + permute in one kernel (slot layout), grouped GEMMs over the slots, gather-combine
            cnt = ws["cnt"][li]
            ops.moe_route_scatter(h, lw["ln2"], lw["gate"], ws["xs"], cnt, perm, ws["rws"], c.rms_norm_eps, ids, tw)
            if tracing:
                self.route_trace.append((ids.clone(), tw.clone()))
            ops.moe_gate_up_slots(ws["xs"], lw["w13"], ws["acts"], cnt, 2 * T)
            ops.moe_down_slots(ws["acts"], lw["w2"], ws["ys"], cnt, ws["rws"], 2 * T)
            nxt = layers[li + 1]["ln1"] if li + 1 < len(layers) else (w["norm"] if final_norm else None)
            ops.moe_combine(h, ws["ys"], perm, nxt, xn if nxt is not None else None, c.rms_norm_eps)
        return xn

    @torch.no_grad()
    def prefill(self, inputs_embeds: torch.Tensor, slot: int = 0, all_logits: bool = False,
                want_last_logits: bool = False, sampled: bool = False, scores: Optional[torch.Tensor] = None,
                start: int = 0, final: bool = True, logprobs: Optional[int] = None, log_softmax_scores: bool = False):
        """One sequence: inputs_embeds [S, H] bf16 (consumed as the residual stream, modified in place).

        Appends S tokens to the KV cache of batch slot `slot` (which must be empty), leaves the arg-max of the last
        position in self.best[slot] (the first generated token) and returns logits [S, V] if `all_logits`.
        `sampled`: the first token is drawn instead (self.sampling's parameters of the slot, counter 0 =
        gen_count[slot] of the empty slot) from the last-row logits; `scores` [rows, V] receives the warped row at
        row 0.  `logprobs` (a log width, see `_sample`; None: none): the first token goes through the sampler (greedy
        slots get the LM head's arg-max word) and its logprobs land in row 0 of the slot's logprob log.

        Chunked prefill / prefix reuse: `start` is the number of tokens the slot already holds (rows get positions
        start + i and attend the cached ones through the paged-KV attention kernel).  With `final` False the rows are
        only appended: no LM head, and best / the sampler counter are left alone; the last chunk of a prompt passes
        `final` True and yields the first token as a whole-prompt prefill does.
        `log_softmax_scores` (with `logprobs` and `scores`): the score row is the log-softmax row (beam search)."""
        c, w = self.cfg, self.w
        S, H = inputs_embeds.shape
        assert inputs_embeds.dtype == BF16 and inputs_embeds.is_cuda and inputs_embeds.is_contiguous()
        if start < 0 or start + S > self.cache.max_seq_len:
            raise ValueError(f"prompt of {start} + {S} tokens exceeds the KV capacity of {self.cache.max_seq_len} "
                             f"per sequence")
        if sampled and self.ep_world > 1:
            raise ValueError("sampled decoding is single-GPU: the expert-parallel prefill serves greedy requests")
        if logprobs is not None and self.ep_world > 1:
            raise ValueError("logprobs are single-GPU: the expert-parallel prefill serves greedy requests")
        if (start > 0 or not final) and self.ep_world > 1:
            raise ValueError("chunked prefill is single-GPU: the expert-parallel prefill takes whole prompts")
        if self.ep_mode == "seq":
            return self._prefill_ep_seq(inputs_embeds, slot, all_logits, want_last_logits)
        h = inputs_embeds
        if start == 0:
            pos, attention = self._ws(S)["pos"][:S], LayerAttention(whole=[(0, S)])
        else:
            pos = torch.arange(start, start + S, dtype=torch.int32, device=self.device)
            plan = ops.PagedPrefill([0, S], [start + S], self.cache.block_table[slot:slot + 1], self.cache.page_size)
            attention = LayerAttention(paged=plan)
        xn = self.run_layers(h, pos, self.cache.slot_map[slot, start:start + S], self.cache.k, self.cache.v, attention,
                             final_norm=all_logits)
        self.cache.cache_len[slot:slot + 1] += S
        if not final:
            return ops.linear(xn, w["lm_head"]) if all_logits else None
        # first generated token: final norm + lm_head + arg-max on the last row only
        self.best[slot:slot + 1].zero_()
        last_logits = self.d_logits[slot:slot + 1] if (want_last_logits or all_logits or sampled
                                                             or logprobs is not None) else None
        ops.tc_lm_head_argmax(h[S - 1:], H, w["norm"], w["lm_head"], last_logits, self.best[slot:slot + 1], 1,
                              self.tc_ws, c.rms_norm_eps)
        if sampled or logprobs is not None:
            self._sample(slot, 1, scores, logprobs, log_softmax_scores)
        if all_logits:
            return ops.linear(xn, w["lm_head"])      # [S, V]; xn = final RMSNorm(h) written by the last combine
        return last_logits

    @torch.no_grad()
    def _prefill_ep_seq(self, inputs_embeds, slot, all_logits, want_last_logits):
        """Sequence-sharded expert-parallel prefill (BASELINE configs[3]; SURVEY.md section 8e).  Rank r owns tokens
        [t0, t1) for everything that is per-token (norms, qkv, o-proj, router, residual stream) and for their causal
        attention over keys [0, t1); per layer three exchanges over NVLink peer memory, all by direct stores:
          1. K/V rows of the own tokens -> every rank's pages (all-gather; a rank waits only for the ranks before it)
          2. post-attention normed rows + routing records -> every rank (all-gather), so every rank can run the
             grouped GEMMs of its local experts over the rows routed to them
          3. the down-projection epilogue pushes each (token, k) output row to the token's owner (fused combine);
             the owner sums its two slots into the residual stream and applies the next RMSNorm.
        No partial sums anywhere: logits are bit-identical to the single-GPU model.  Returns the logits of the OWN rows
        when `all_logits`, the last-row logits on the rank that owns the last token otherwise (None elsewhere)."""
        steps = self._prefill_ep_seq_steps(inputs_embeds, slot, all_logits, want_last_logits)
        while True:
            try:
                next(steps)
            except StopIteration as done:
                return done.value

    @torch.no_grad()
    def _prefill_ep_seq_steps(self, inputs_embeds, slot, all_logits, want_last_logits):
        """_prefill_ep_seq as a generator that yields right after each ep_signal (three times per layer, before the
        wait that needs the other ranks' flags), so that one process can step several ranks on one device in turn.
        Returns what _prefill_ep_seq returns."""
        assert slot == 0
        c, w, sy = self.cfg, self.w, self.ep_p2p
        S, H = inputs_embeds.shape
        N, r = self.ep_world, self.ep_rank
        from ..parallel import token_range
        chunk = self.ep_chunk(S)
        t0, t1 = token_range(S, r, N)
        n = t1 - t0
        ws = self._ws(S)
        nq, nkv, D, E = c.num_attention_heads, c.num_key_value_heads, c.head_dim, c.num_local_experts
        W = c.qkv_rows
        h_own, xn_own = sy["h"][t0:t1], sy["xn"][t0:t1]
        xn2, ids, tw = sy["xn2"][:S], sy["ids"][:S], sy["tw"][:S]
        qkv, attn = ws["qkv"][:n], ws["attn"][:n]
        perm, rtok, rw = ws["perm"][:2 * S], ws["rtok"][:2 * S], ws["rw"][:2 * S]
        xp, act = ws["xp"][:2 * S], ws["act"][:2 * S]
        pos, slots = ws["pos"][t0:t1], self.cache.slot_map[0, t0:t1]
        off, kvl, kvr = sy["off"], sy["kv_layer"], sy["kv_row"]
        offs_local = ws["offs"][self.e_lo:]
        layers = w["layers"]
        if n:
            h_own.copy_(inputs_embeds[t0:t1])
            ops.rmsnorm(h_own, layers[0]["ln1"], c.rms_norm_eps, out=xn_own)
        for li, lw in enumerate(layers):
            sy["epoch"] += 1
            ep = sy["epoch"]
            if n:
                ops.linear_qkv_rope(xn_own, lw["wqkv"], qkv, pos, slots, w["rope"], self.cache.k[li],
                                    self.cache.v[li], nq, nkv, D)
                ko = off["kv"] + 2 * li * kvl + t0 * kvr
                ops.ep_push(sy["base_ptrs"], [(ko, n * kvr), (ko + kvl, n * kvr)], N, r)
            ops.ep_signal(sy["flag_ptrs"], 2, N, r, ep)
            yield
            ops.ep_wait(sy["flags"], 2, N, ep, n_wait=r)          # K/V rows of the ranks before this one
            if n:
                ops.attention(qkv, self.cache.k[li], self.cache.v[li], attn, (0, W, D), (0, nkv * D, D),
                              (0, nkv * D, D), (0, nq * D, D), 1, nq, nkv, n, t1, D, D, None, True, D ** -0.5,
                              q_pos0=t0)
                ops.linear(attn, lw["wo"], residual=h_own, out=h_own)
                ops.moe_router(h_own, lw["ln2"], lw["gate"], xn2[t0:t1], ids[t0:t1], tw[t0:t1], c.rms_norm_eps)
                ops.ep_push(sy["base_ptrs"], [(off["xn2"] + t0 * H * 2, n * H * 2), (off["ids"] + t0 * 8, n * 8),
                                              (off["tw"] + t0 * 8, n * 8)], N, r)
            ops.ep_signal(sy["flag_ptrs"], 3, N, r, ep)
            yield
            ops.ep_wait(sy["flags"], 3, N, ep)
            ops.moe_align(ids, tw, ws["offs"], perm, rtok, rw, S, E, row_assign=ws["rassign"][:2 * S])
            ops.row_copy(xn2, rtok, None, xp, 2 * S)
            ops.moe_gate_up(xp, lw["w13"], act, offs_local, 2 * S)
            ops.moe_down_ep(act, lw["w2"], offs_local, rw, ws["rassign"][:2 * S], sy["rs_ptrs"], 2 * S, chunk)
            ops.ep_signal(sy["flag_ptrs"], 0, N, r, ep)
            yield
            nxt = layers[li + 1]["ln1"] if li + 1 < len(layers) else (w["norm"] if all_logits else None)
            # (waits for flags[0] of every rank: all expert rows of the own tokens have landed)
            ops.ep_reduce_norm_gather(sy["rs"], sy["flags"], sy["h_ptrs"], sy["xn_ptrs"], nxt, t0, n, N, r, ep, H,
                                      c.rms_norm_eps, gather=False)
            if n == 0:
                ops.ep_wait(sy["flags"], 0, N, ep)   # keep the epochs of a token-less rank in step with the others
        self.cache.cache_len[slot:slot + 1] += S
        self.best[slot:slot + 1].zero_()
        last_logits = None
        if t0 <= S - 1 < t1:     # this rank owns the last token: first generated token
            last_logits = self.d_logits[slot:slot + 1] if (want_last_logits or all_logits) else None
            ops.tc_lm_head_argmax(sy["h"][S - 1:S], H, w["norm"], w["lm_head"], last_logits,
                                  self.best[slot:slot + 1], 1, self.tc_ws, c.rms_norm_eps)
        if all_logits:
            return ops.linear(xn_own, w["lm_head"]) if n else torch.empty(0, c.vocab_size, dtype=BF16, device=self.device)
        return last_logits

    # ------------------------------------------------------------------------------------------ decode
    def _decode_step_kernels(self, B: int, want_logits: bool, sampled: bool = False,
                             logprobs: Optional[int] = None):
        """One greedy token for slots [0, B): embed + per layer (qkv+RoPE+KV append -> paged attention -> o-proj ->
        router+gate/up -> down) + LM head with arg-max, 2 + 5 L launches chained by programmatic dependent launch.
        For B = 1 the kernels are additionally linked by completion counters (include/vita_b200.h, vita_chain_begin).
        `sampled`: the LM head writes the logits and the sampler draws the token from them (one launch more, after the
        counter chain; with a score log it writes the warped row in place of the logits copy).  `logprobs`: the
        sampler path as well, writing the logprob log too (greedy rows keep the LM head's arg-max word)."""
        c, w, cache = self.cfg, self.w, self.cache
        nq, nkv, D = c.num_attention_heads, c.num_key_value_heads, c.head_dim
        h = self.d_h[:B]
        ws = self.tc_ws
        chained = B == 1
        ops.decode_embed(self.best[:B], self.token_log[:B], self.gen_count[:B], cache.cache_len[:B], cache.cur_pos[:B],
                         w["embed"], h, cache.max_seq_len, self.chain_mem if chained else None)
        if chained:
            ops.chain_begin(self.chain_mem)
        try:
            for li, lw in enumerate(w["layers"]):
                ops.decode_tc_qkv_rope(h, lw["ln1"], lw["wqkv"], w["rope"], cache.cur_pos[:B], cache.block_table[:B],
                                       self.d_q[:B], cache.k[li], cache.v[li], ws, nq, nkv, D, cache.page_size,
                                       c.rms_norm_eps, cache.k_scale[li], cache.v_scale[li])
                ops.decode_attention(self.d_q[:B], cache.k[li], cache.v[li], cache.block_table[:B], cache.cur_pos[:B],
                                     self.d_attn[:B], self.attn_ws, nq, nkv, D, cache.page_size, self.decode_splits,
                                     D ** -0.5, k_scale=cache.k_scale[li], v_scale=cache.v_scale[li])
                ops.decode_tc_oproj(self.d_attn[:B], lw["wo"], h, ws)
                tracing = self.route_trace is not None and not torch.cuda.is_current_stream_capturing()
                route = None if (tracing or not self.early_route) else self.d_route[:B]
                ops.decode_tc_moe_gate_up(h, lw["ln2"], lw["gate"], lw["w13"], self.d_ids[:B], self.d_w[:B],
                                          self.d_act[:B], ws, c.rms_norm_eps, route, li + 1)
                if tracing:
                    self.route_trace.append((self.d_ids[:B].clone(), self.d_w[:B].clone()))
                ops.decode_tc_moe_down(self.d_act[:B], lw["w2"], self.d_ids[:B], self.d_w[:B], h, ws, route, li + 1)
            lg = self.d_logits[:B] if (want_logits or sampled or logprobs is not None) else None
            ops.tc_lm_head_argmax(h, c.hidden_size, w["norm"], w["lm_head"], lg, self.best[:B], B, ws, c.rms_norm_eps)
        finally:
            if chained:
                ops.chain_end()
        if sampled or logprobs is not None:
            self._sample(0, B, self.scores_buf if (want_logits and B == 1) else None, logprobs)
        else:
            self._log_scores(B, want_logits)

    def _sample(self, s0: int, n: int, scores: Optional[torch.Tensor], logprobs: Optional[int] = None,
                log_softmax_scores: bool = False):
        """Draw the next token of slots [s0, s0 + n) from d_logits into best (counter = gen_count of the slot).
        `logprobs` (the log width, SlotSampling.log_width: 0 or 20): also write the token's logprob, rank and that
        many top entries at row gen_count of each slot's logprob log; `log_softmax_scores`: the score rows get the
        log-softmax of the processed row."""
        sp, rows = self.sampling, slice(s0, s0 + n)
        if logprobs is None:
            ops.sample_rows(self.d_logits[rows], sp.temperature[rows], sp.top_k[rows], sp.top_p[rows], sp.seed[rows],
                            self.gen_count[rows], self.best[rows], scores, streams=sp.stream[rows])
            return
        lg = self.enable_logprob_log()
        ops.sample_logprobs(self.d_logits[rows], sp.temperature[rows], sp.top_k[rows], sp.top_p[rows], sp.seed[rows],
                            self.gen_count[rows], self.best[rows], lg[0][rows], lg[1][rows], lg[2][rows], lg[3][rows],
                            logprobs, scores=scores, log_softmax_scores=log_softmax_scores, streams=sp.stream[rows])

    def enable_logprob_log(self):
        """Allocate the per-slot logprob log: (logprob f32 [B, R], rank i32 [B, R], top ids i32 [B, R, 20], top
        logprobs f32 [B, R, 20]), R = the token log's length.  Row i of a slot belongs to its generated token i (row
        index = gen_count, written on the device, so it works under CUDA-graph replay).  A step records the top 20 when
        any of its requests asks for top entries (readers keep the N a request asked for), none otherwise."""
        if self.lp_log is None:
            B, R, dev = self.max_batch, self.token_log.shape[1], self.device
            with torch.inference_mode(False):
                self.lp_log = (torch.zeros(B, R, dtype=torch.float32, device=dev),
                               torch.zeros(B, R, dtype=torch.int32, device=dev),
                               torch.zeros(B, R, MAX_LOGPROBS, dtype=torch.int32, device=dev),
                               torch.zeros(B, R, MAX_LOGPROBS, dtype=torch.float32, device=dev))
        return self.lp_log

    def read_logprobs(self, slot: int, tokens: Sequence[int], n_top: int):
        """TokenLogprobs of the generated tokens of `slot` (`tokens`: the first len(tokens) of them, as the caller
        holds them; the token log only receives a token when the next step consumes it), top-n_top each."""
        lp, rk, ti, tl = (t[slot, :len(tokens)].cpu() for t in self.lp_log)
        return logprob_records(tokens, lp, rk, ti, tl, n_top)

    def enable_beam_score_log(self, n: int, rows: int) -> torch.Tensor:
        """The per-slot log-softmax log of beam search's `output_scores`: [>= n, >= rows, V] bf16, row i of slot b
        written by the step that produced token i (row index = gen_count).  Sized to the largest call so far (n beams,
        `rows` = its max_new_tokens) and kept with the decoder; the batched-step graphs that write it are re-captured
        when it grows."""
        old = self.beam_scores
        if old is None or old.shape[0] < n or old.shape[1] < rows:
            n, rows = (n, rows) if old is None else (max(n, old.shape[0]), max(rows, old.shape[1]))
            self.beam_scores = None
            with torch.inference_mode(False):
                self.beam_scores = torch.zeros(n, rows, self.cfg.vocab_size, dtype=BF16, device=self.device)
            self._bgraphs = {k: g for k, g in self._bgraphs.items() if "scores" not in k}
        return self.beam_scores

    def fork(self, src: int, dsts: Sequence[int], length: int):
        """Slots dsts continue slot src, which holds `length` tokens: its KV pages are shared copy-on-write
        (PagedKVCache.fork) and its decode state (cache_len, cur_pos, gen_count, token log, next token) is copied."""
        c = self.cache
        idx = torch.tensor(list(dsts), dtype=torch.int64, device=self.device)
        for t in (c.cache_len, c.cur_pos, self.gen_count, self.token_log, self.best):
            t[idx] = t[src].clone()
        c.fork(src, dsts, length)

    def fork_sampled(self, src: int, count: int, length: int, n_pages: int, scores: Optional[torch.Tensor] = None):
        """Parallel sampling: slot src has just prefilled its `length` prompt rows with a sampled first token; slots
        src + 1 .. src + count - 1 become further sampled sequences of the same request.  They share src's full KV
        pages, get a copy of its partial page and private pages up to n_pages (PagedKVCache.fork_reserved), take its
        sampler parameters with streams 1 .. count - 1 (SlotSampling.fork) and its decode state, and each draws its own
        first token at counter 0 from src's last-row logits (with its logprob record when src's request asks).
        `scores` (a per-slot score log [>= src + count, rows, V]): their warped rows land in row 0 of their slots."""
        if count < 2:
            return
        c, dst = self.cache, slice(src + 1, src + count)
        for t in (c.cache_len, c.cur_pos, self.gen_count, self.token_log, self.d_logits):
            t[dst] = t[src].clone()
        self.sampling.fork(src, count)
        c.fork_reserved(src, range(src + 1, src + count), length, n_pages)
        self._sample(src + 1, count - 1, scores[dst] if scores is not None else None,
                     self.sampling.log_width(src, 1))

    def enable_score_log(self):
        """Allocate the per-step logits log (HF `output_scores=True`): row i holds the logits token i was chosen from.
        The decode step appends to it on the device (row index = gen_count), so it works under CUDA-graph replay."""
        if self.scores_buf is None:
            with torch.inference_mode(False):   # persistent state must not become an inference tensor when the first
                #                                 call happens under torch.inference_mode() (video_audio_demo.py:256)
                self.scores_buf = torch.zeros(self.max_new_tokens + 1, self.cfg.vocab_size, dtype=BF16,
                                              device=self.device)
            self._graphs = {k: g for k, g in self._graphs.items() if not k[1]}   # re-capture the logits variants
        return self.scores_buf

    def _log_scores(self, B: int, want_logits: bool):
        if want_logits and B == 1 and self.scores_buf is not None:
            ops.row_copy(self.d_logits[:1], None, self.gen_count[:1], self.scores_buf, 1)

    @property
    def launches_per_decode_step(self) -> int:
        return 2 + 5 * self.cfg.num_hidden_layers

    def launches_per_decode_step_with_scores(self) -> int:
        return self.launches_per_decode_step + 1

    @property
    def launches_per_decode_step_sampled(self) -> int:
        """A sampled bs = 1 step, with or without the score log: the sampler replaces the logits copy."""
        return self.launches_per_decode_step + 1

    @torch.no_grad()
    def decode_step(self, B: int = 1, use_graph: bool = True, want_logits: bool = False, sampled: bool = False,
                    logprobs: Optional[int] = None):
        """Generate one token for batch slots [0, B): consumes self.best, appends to token_log, leaves the next
        arg-max (or, `sampled`, the drawn token) in self.best.  With use_graph the whole step (2 + 5 * layers kernels,
        one more when sampled) replays as one CUDA graph."""
        assert self.ep_world == 1, "expert-parallel mode covers the prefill (BASELINE configs[3]); decode is replicated"
        step = lambda: self._decode_step_kernels(B, want_logits, sampled, logprobs)
        if not use_graph:
            step()
            return
        key = (B, want_logits, True) if sampled else (B, want_logits)    # greedy keys keep their (B, want_logits) form
        if logprobs is not None:
            key = (B, want_logits, sampled, "logprobs", logprobs)
        self._replay(self._graphs, key, step)

    # ------------------------------------------------------------------------------------------ batched decode
    def _batched_step_kernels(self, B: int, sampled: bool = False, logprobs: Optional[int] = None,
                              scores: bool = False, warped_scores: bool = False):
        """One token for each of B sequences through the GEMM path (weights of every touched expert are streamed once
        for the whole batch; BASELINE configs[4]).  The prefill's layer loop with M = B rows at B different
        positions and the paged decode attention.  `scores` (with `logprobs`): the sampler also writes each slot's
        log-softmax row to the beam score log; `warped_scores` (sampled): each slot's warped row to the same per-slot
        log (parallel sampling's output_scores)."""
        c, w, cache = self.cfg, self.w, self.cache
        h = self.d_h[:B]
        ops.decode_embed(self.best[:B], self.token_log[:B], self.gen_count[:B], cache.cache_len[:B], cache.cur_pos[:B],
                         w["embed"], h, cache.max_seq_len)
        slots = self.d_slots[:B]
        ops.decode_slots(cache.cur_pos[:B], cache.block_table[:B], slots, cache.page_size)
        attention = LayerAttention(decode=(0, B, cache.block_table[:B], cache.cur_pos[:B], self.attn_ws),
                                   page_size=cache.page_size)
        xn = self.run_layers(h, cache.cur_pos[:B], slots, cache.k, cache.v, attention, final_norm=True)
        logits = ops.linear(xn, w["lm_head"], out=self.d_logits[:B])
        if sampled or logprobs is not None:   # greedy rows (temperature 0) get argmax_rows' word: a mixed batch keeps their tokens
            self._sample(0, B, self.beam_scores if (scores or warped_scores) else None, logprobs, scores)
        else:
            ops.argmax_rows(logits, self.best[:B])

    @property
    def launches_per_batched_step(self) -> int:
        return 6 + 8 * self.cfg.num_hidden_layers

    @torch.no_grad()
    def decode_step_batched(self, B: int, use_graph: bool = True, sampled: bool = False,
                            logprobs: Optional[int] = None, scores: bool = False, warped_scores: bool = False):
        """`scores`: write the log-softmax rows to the beam score log (enable_beam_score_log; needs `logprobs`).
        `warped_scores`: write the warped rows to that log instead (needs `sampled`)."""
        assert self.ep_world == 1 and 1 <= B <= self.max_batch
        assert not scores or (logprobs is not None and self.beam_scores is not None and self.beam_scores.shape[0] >= B)
        assert not warped_scores or (sampled and not scores and self.beam_scores is not None
                                     and self.beam_scores.shape[0] >= B)
        step = lambda: self._batched_step_kernels(B, sampled, logprobs, scores, warped_scores)
        if not use_graph:
            step()
            return
        key = (B, sampled, "logprobs", logprobs) if logprobs is not None else (B, sampled)
        if scores:
            key += ("scores",)
        if warped_scores:
            key += ("scores", "warped")     # "scores": re-captured when the log grows (enable_beam_score_log)
        self._replay(self._bgraphs, key, step)   # one graph per batch size (continuous batching changes B)

    def _replay(self, graphs: dict, key, step):
        """Replay graphs[key], capturing `step` (a decode step that takes no host input) into it first: an eager
        warm-up runs every cudaFuncSetAttribute outside the capture, and the decode state it advanced is restored."""
        if key not in graphs:
            snap = self._save_state()
            step()
            torch.cuda.synchronize()
            self._restore_state(snap)
            g = torch.cuda.CUDAGraph()
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            # no garbage collection inside the capture: collecting an unreachable model destroys its CUDA graphs, and
            # destroying a graph while a stream captures invalidates the capture
            gc_enabled = gc.isenabled()
            gc.disable()
            try:
                with torch.cuda.stream(side):
                    with torch.cuda.graph(g, stream=side):
                        step()
            finally:
                if gc_enabled:
                    gc.enable()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            self._restore_state(snap)   # capture does not execute, but keep the invariant explicit
            graphs[key] = g
        graphs[key].replay()

    def _save_state(self):
        c = self.cache
        return (self.best.clone(), self.gen_count.clone(), c.cache_len.clone(), c.cur_pos.clone(), self.d_h.clone(),
                self.token_log.clone())

    def _restore_state(self, s):
        c = self.cache
        self.best.copy_(s[0]); self.gen_count.copy_(s[1]); c.cache_len.copy_(s[2]); c.cur_pos.copy_(s[3])
        self.d_h.copy_(s[4]); self.token_log.copy_(s[5])
        # the KV slot written by the warm-up step is rewritten by the real step (same position): nothing to undo

    def check_capacity(self, prompt_len: int, new_tokens: int):
        """Every decode entry point calls this: prompt + reply must fit the paged KV cache of one sequence (the
        kernels index block_table[pos / page_size] and the rope table without a bound of their own)."""
        if prompt_len + new_tokens > self.cache.max_seq_len:
            raise ValueError(f"prompt ({prompt_len}) + max_new_tokens ({new_tokens}) exceeds the KV capacity "
                             f"({self.cache.max_seq_len} positions per sequence); build the model with a larger "
                             f"max_seq_len")
        if new_tokens > self.max_new_tokens:
            raise ValueError(f"max_new_tokens {new_tokens} exceeds the token log ({self.max_new_tokens}); build the "
                             f"model with a larger max_new_tokens")

    def reset(self):
        self.cache.reset()
        self.chain_mem.zero_()     # completion counters restart with the request (also heals an aborted step)
        self.best.zero_()
        self.gen_count.zero_()
        self.token_log.zero_()

    def generated_tokens(self, slot: int = 0) -> List[int]:
        n = int(self.gen_count[slot])
        return self.token_log[slot, :n].tolist()
