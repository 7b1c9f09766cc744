"""Prefix caching in the continuous batcher on the CPU: the page digest's numpy reference, the key chain, the hit-length
rule, PagePool / PrefixIndex bookkeeping (admit, retire, swap, evict, invalidate) and the batcher / DecoderEngine
admission policy over a stand-in decoder."""
import random

import numpy as np
import pytest
import torch

from tests.test_engine_chunked import ChunkEngine
from vita_b200.config import VitaConfig
from vita_b200.engine import ContinuousBatcher, DecoderEngine, Request
from vita_b200.model.mixtral import PagedKVCache, PagePool, prefix_keys

M64 = (1 << 64) - 1
GAMMA, SEEDS = 0x9E3779B97F4A7C15, (0x243F6A8885A308D3, 0x13198A2E03707344)


def mix64_np(z):
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def digest_ref(rows: torch.Tensor, page_size: int) -> np.ndarray:
    """include/vita_b200.h vita_page_digest in numpy: rows bf16 [n, H] -> uint64 [n // page_size, 2]."""
    n, H = rows.shape
    n_pages = n // page_size
    bits = rows[: n_pages * page_size].contiguous().view(torch.int16).numpy().view(np.uint16)
    words = bits.reshape(n_pages, page_size * H).view("<u8")              # [pages, page_size * H / 4]
    j = np.arange(words.shape[1], dtype=np.uint64) * np.uint64(GAMMA)
    out = np.zeros((n_pages, 2), dtype=np.uint64)
    with np.errstate(over="ignore"):
        for lane, seed in enumerate(SEEDS):
            out[:, lane] = mix64_np(words + j + np.uint64(seed)).sum(axis=1, dtype=np.uint64)
    return out


def digest_scalar(words, seed):
    """The same function on Python integers, one word at a time."""
    def mix(z):
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
        return z ^ (z >> 31)
    return sum(mix((w + j * GAMMA + seed) & M64) for j, w in enumerate(words)) & M64


def digests(rows, page_size):
    return torch.from_numpy(digest_ref(rows, page_size).view(np.int64))


def test_mix64_is_splitmix64():
    # the first output of splitmix64 seeded with 0: mix64(0 + gamma)
    assert int(mix64_np(np.array([GAMMA], dtype=np.uint64))[0]) == 0xE220A8397B1DCDAF


def test_digest_reference_known_answers():
    zero = torch.zeros(4, 8, dtype=torch.bfloat16)                 # one page of 4 rows x 8 values: 8 zero words
    d = digest_ref(zero, 4)
    assert d.shape == (1, 2)
    assert [int(x) for x in d[0]] == [digest_scalar([0] * 8, s) for s in SEEDS]
    assert [int(x) for x in d[0]] == [0xDF9DCA7C15F4CE41, 0xAA507FEA49086BDE]
    g = torch.Generator().manual_seed(0)
    rows = torch.randn(37, 16, generator=g).bfloat16()
    d = digest_ref(rows, 16)
    assert d.shape == (2, 2)                                          # the partial last page gets no digest
    for p in range(2):
        words = rows[16 * p:16 * (p + 1)].contiguous().view(torch.int16).numpy().view("<u8").ravel().tolist()
        assert [int(x) for x in d[p]] == [digest_scalar(words, s) for s in SEEDS]


def test_digest_depends_on_word_position():
    rows = torch.zeros(4, 8, dtype=torch.bfloat16)
    a, b = rows.clone(), rows.clone()
    a[0, 0], b[3, 7] = 1.0, 1.0
    assert not np.array_equal(digest_ref(a, 4), digest_ref(b, 4))


def test_key_chain_changes_with_any_earlier_page():
    g = torch.Generator().manual_seed(1)
    rows = torch.randn(16 * 6, 8, generator=g).bfloat16()
    base = prefix_keys(digests(rows, 16))
    assert len(base) == 6 and len(set(base)) == 6 and all(len(k) == 16 for k in base)
    for p in range(6):
        other = rows.clone()
        other[16 * p + 5, 3] += 1.0
        keys = prefix_keys(digests(other, 16))
        assert keys[:p] == base[:p]                                   # pages before the change keep their keys
        assert all(k != b for k, b in zip(keys[p:], base[p:]))        # it and every later page change


# ------------------------------------------------------------------------------------------------ hit length
def _cache(B=2, max_seq_len=256, ps=16):
    return PagedKVCache(VitaConfig.tiny().llm, B, max_seq_len, "cpu", ps, shuffle_pages=True)


@pytest.mark.parametrize("ps", [16, 32])
def test_hit_length_is_page_aligned_and_capped(ps):
    c = _cache(ps=ps)
    g = torch.Generator().manual_seed(2)
    rows = torch.randn(5 * ps + 3, 8, generator=g).bfloat16()
    keys = prefix_keys(digests(rows, ps))
    assert c.admit_prefix(0, keys, rows.shape[0], 8) == 0
    c.pool.insert(0, keys)
    c.pool.check()
    for S in (1, ps - 1, ps, ps + 1, 2 * ps, 3 * ps + 7, 5 * ps, 5 * ps + 1, 5 * ps + 3):
        P = c.admit_prefix(1, keys[:S // ps], S, 8)
        assert P % ps == 0 and P == ps * min(5, (S - 1) // ps) and P < S, (S, P)
        assert c.pool.table[1][: P // ps] == c.pool.table[0][: P // ps]
        c.pool.check()
    other = rows.clone()
    other[0, 0] += 1.0                                                # a different first page: no hit at all
    assert c.admit_prefix(1, prefix_keys(digests(other, ps)), rows.shape[0], 8) == 0
    # the device rows follow the pool's table: block_table and the slot_map derived from it
    row = torch.tensor(c.pool.table[1], dtype=torch.int32)
    assert torch.equal(c.block_table[1], row)
    pos = torch.arange(8 * ps)
    assert torch.equal(c.slot_map[1, :8 * ps], (row[pos // ps] * ps + pos % ps).int())


# ------------------------------------------------------------------------------------------------ pool invariants
def _pool(B, pps, ps, seed=0):
    return PagePool(torch.randperm(B * pps, generator=torch.Generator().manual_seed(seed)).view(B, pps), ps)


def _keys(prefix_id, n, tail_id):
    """n page keys: a shared prefix of pages from `prefix_id` for its first half, then pages unique to `tail_id`."""
    return prefix_keys(torch.tensor([[prefix_id, i] if i < n // 2 else [tail_id, i] for i in range(n)],
                                    dtype=torch.int64))


@pytest.mark.parametrize("ps", [16, 32])
@pytest.mark.parametrize("trial", range(4))
def test_pool_invariants_under_random_admit_retire_swap_evict(ps, trial):
    rng = random.Random(1000 * ps + trial)
    B, pps = rng.choice([(1, 6), (2, 5), (4, 8)])
    pool = _pool(B, pps, ps, trial)
    content = {}                         # page -> the key whose rows it holds (written by the request that indexed it)
    evictions = 0
    for it in range(300):
        slot = rng.randrange(B)
        op = rng.random()
        if op < 0.6:                     # admit a new request into the slot (releases whatever it held)
            n_prompt = rng.randint(0, pps)
            keys = _keys(rng.randrange(3), n_prompt, rng.randrange(10 ** 6))
            n_pages = rng.randint(max(n_prompt, 1), pps)
            pool.release(slot)
            hits = pool.admit(slot, keys[:max(n_prompt - 1, 0)], n_pages)
            row = pool.table[slot]
            assert sum(pg >= 0 for pg in row) == n_pages and len(set(row[:n_pages])) == n_pages
            for i in range(hits):
                assert content[row[i]] == keys[i], "a hit page holds another prefix"
            for i in range(hits, n_pages):
                content.pop(row[i], None)                           # private: rewritten by this request
            pool.insert(slot, keys)
            for i, key in enumerate(keys):
                if pool.index.page.get(key) == row[i]:
                    content[row[i]] = key
        elif op < 0.8:                   # retire
            pool.release(slot)
        else:                            # swap two slots
            j = rng.randrange(B)
            pool.swap(slot, j)
        assert pool.evictions >= evictions
        evictions = pool.evictions
        pool.check()
    assert pool.evictions > 0                                        # the sequences do reach eviction


def test_admission_never_fails_with_max_batch_maximal_requests():
    B, pps, ps = 4, 6, 16
    pool = _pool(B, pps, ps)
    rid = 0
    for rnd in range(25):
        for slot in range(B):            # every slot holds a maximal request, all indexed
            rid += 1
            keys = _keys(rnd % 2, pps, rid)
            pool.release(slot)
            pool.admit(slot, keys[:pps - 1], pps)
            pool.insert(slot, keys)
            pool.check()
            assert all(pg >= 0 for pg in pool.table[slot])
    assert pool.evictions > 0


def test_lru_eviction_order():
    ps = 16
    pool = _pool(2, 4, ps)
    a, b = _keys(10, 4, 11), _keys(20, 4, 21)
    for slot, keys in ((0, a), (1, b)):
        pool.release(slot)
        pool.admit(slot, [], 4)
        pool.insert(slot, keys)
    pa, pb = list(pool.table[0]), list(pool.table[1])
    pool.release(0)                      # a's pages become evictable first, its last page first of all
    pool.release(1)
    assert list(pool.index.lru) == pa[::-1] + pb[::-1] and not pool.free
    pool.admit(0, [], 3)                 # three unrelated pages: evicts a's pages 3, 2, 1
    assert pool.evictions == 3 and set(pool.table[0][:3]) == set(pa[1:])
    assert pool.index.page.get(a[0]) == pa[0] and all(k not in pool.index.page for k in a[1:])
    pool.check()
    pool.release(1)
    assert pool.admit(1, b[:3], 4) == 3 and pool.table[1][:3] == pb[:3]    # b is untouched: it still hits
    pool.check()


def test_invalidation_on_reset():
    c = _cache(B=2, max_seq_len=128, ps=16)
    static_bt, static_sm = c.block_table.clone(), c.slot_map.clone()
    keys = _keys(1, 4, 2)
    c.admit_prefix(0, keys, 70, 6)
    c.pool.insert(0, keys)
    assert c.admit_prefix(1, keys, 70, 6) == 64
    epoch = c.pool.epoch
    c.reset()
    assert c.pool.epoch > epoch and not c.pool.index.page and not c.pool.index.lru
    assert torch.equal(c.block_table, static_bt) and torch.equal(c.slot_map, static_sm)
    c.pool.check()
    assert c.admit_prefix(1, keys, 70, 6) == 0                            # no stale hit after the reset
    c.unshare()
    assert torch.equal(c.block_table, static_bt) and torch.equal(c.slot_map, static_sm)


# ------------------------------------------------------------------------------------------------ DecoderEngine policy
class StubLLM:
    """What DecoderEngine touches of MixtralDecoder, on the CPU: a real PagedKVCache (tables only) and a prefill that
    records its calls; every prompt's first token is FIRST, every decode step appends token 1."""
    FIRST = 5

    def __init__(self, B=3, max_seq_len=256, ps=16):
        from vita_b200.sampling import SlotSampling
        self.cache = PagedKVCache(VitaConfig.tiny().llm, B, max_seq_len, "cpu", ps, shuffle_pages=True)
        self.ep_world, self.max_new_tokens, self.lp_log = 1, 32, None
        self.best = torch.zeros(B, dtype=torch.int64)
        self.token_log = torch.zeros(B, 40, dtype=torch.int32)
        self.gen_count = torch.zeros(B, dtype=torch.int32)
        self.sampling = SlotSampling(B, "cpu")
        self.calls = []                                  # (slot, start, rows, final)

    def prefill(self, rows, slot, sampled=False, start=0, final=True, logprobs=None):
        assert int(self.cache.cache_len[slot]) == start, "the slot holds exactly the rows before `start`"
        self.calls.append((slot, start, rows.shape[0], final))
        self.cache.cache_len[slot] += rows.shape[0]
        if final:
            self.best[slot] = 0xFFFFFFFF - self.FIRST

    def decode_step_batched(self, n, use_graph=True, sampled=False, logprobs=None):
        for s in range(n):
            self.token_log[s, int(self.gen_count[s])] = 0xFFFFFFFF - int(self.best[s])
            self.gen_count[s] += 1
            self.best[s] = 0xFFFFFFFF - 1

    def generated_tokens(self, slot):
        return self.token_log[slot, :int(self.gen_count[slot])].tolist()


class StubModel:
    def __init__(self, **kw):
        self.llm = StubLLM(**kw)
        self.table = torch.randn(1000, 16, generator=torch.Generator().manual_seed(3)).bfloat16()

    def _embeds_for(self, ids, images, audios):
        return self.table[ids], torch.tensor([ids.shape[1]])


@pytest.fixture
def stub_digest(monkeypatch):
    from vita_b200 import ops
    monkeypatch.setattr(ops, "page_digest", lambda rows, ps: digests(rows, ps))


def _req(rid, ids, n=3, arrival=0, **kw):
    return Request(rid, {"input_ids": torch.tensor([ids])}, n, None, arrival_step=arrival, **kw)


def test_engine_prefill_starts_at_the_hit_length(stub_digest):
    model = StubModel()
    eng = DecoderEngine(model, use_graph=False, prefix_cache=True)
    shared = list(range(100, 150))                       # 3 full pages + 2 rows
    reqs = [_req(0, shared + [1, 2, 3]), _req(1, shared + [7, 8], arrival=1), _req(2, shared[:32], arrival=2),
            _req(3, [9] + shared[1:], arrival=3)]
    ContinuousBatcher(eng, 3).run(reqs)
    starts = [c[1] for c in model.llm.calls]
    # 0: cold; 1: three full pages; 2: exactly two pages long, so its last page is computed; 3: first page differs
    assert starts == [0, 48, 16, 0]
    assert [r.cached_tokens for r in reqs] == starts
    assert [c[2] for c in model.llm.calls] == [53 - 0, 52 - 48, 32 - 16, 50]
    assert eng.prefix_stats == {"hit_pages": 4, "missed_pages": 3 + 3 + 2 + 3 - 4}
    model.llm.cache.pool.check()


def test_engine_chunked_admission_starts_at_the_hit_length(stub_digest):
    model = StubModel()
    eng = DecoderEngine(model, use_graph=False, prefix_cache=True)
    shared = list(range(200, 300))
    reqs = [_req(0, shared, n=12), _req(1, shared + [5] * 30, n=4, arrival=2)]
    ContinuousBatcher(eng, 3, prefill_chunk=16).run(reqs)
    calls = [c for c in model.llm.calls if c[1] >= 0]
    second = [c for c in calls if c[1] >= 96]
    assert reqs[1].cached_tokens == 96 and second[0][1] == 96       # its chunks begin at P = 6 pages
    assert sum(c[2] for c in second) == 130 - 96 and second[-1][3]
    model.llm.cache.pool.check()


def test_batcher_reports_cached_tokens_from_begin_prefill():
    """A stand-in engine whose begin_prefill returns (S, P): the chunks start at P, cached_tokens is P."""
    class HitEngine(ChunkEngine):
        def begin_prefill(self, slot, request):
            S = super().begin_prefill(slot, request)
            P = request.payload.get("hit", 0)
            self.filled[slot] = P
            return S, P
    eng = HitEngine(2, cap=16)
    reqs = [Request(0, {"seed": 3, "len": 50, "hit": 32}, 4), Request(1, {"seed": 4, "len": 20}, 3, arrival_step=1)]
    ContinuousBatcher(eng, 2, prefill_chunk=8).run(reqs)
    assert [r.cached_tokens for r in reqs] == [32, 0]
    assert eng.chunks[0][2] == 18                       # nothing running: the rest of request 0 at once


def test_negative_query_leaves_its_pages_indexed(stub_digest):
    model = StubModel()
    eng = DecoderEngine(model, use_graph=False, prefix_cache=True)
    history = list(range(300, 340))                      # 2 full pages + 8
    reqs = [_req(0, history, negative_token_id=StubLLM.FIRST, session=1),
            _req(1, history + [4, 4, 4], arrival=1, session=1)]
    out = ContinuousBatcher(eng, 2).run(reqs)
    assert reqs[0].outcome == "negative" and out[0] == [StubLLM.FIRST]
    assert reqs[1].cached_tokens == 32 and reqs[1].outcome == "finished"
    model.llm.cache.pool.check()


def test_generate_style_reset_invalidates_the_engine_index(stub_digest):
    model = StubModel()
    eng = DecoderEngine(model, use_graph=False, prefix_cache=True)
    ids = list(range(400, 440))
    ContinuousBatcher(eng, 2).run([_req(0, ids)])
    model.llm.cache.reset()                              # what MixtralDecoder.reset() does for generate() & co.
    r = _req(1, ids)
    ContinuousBatcher(eng, 2).run([r])
    assert r.cached_tokens == 0
    r = _req(2, ids)
    ContinuousBatcher(eng, 2).run([r])
    assert r.cached_tokens == 32


def test_prefix_cache_is_off_by_default(stub_digest):
    model = StubModel()
    eng = DecoderEngine(model, use_graph=False)
    ids = list(range(500, 540))
    reqs = [_req(0, ids), _req(1, ids, arrival=1)]
    ContinuousBatcher(eng, 2).run(reqs)
    assert [c[1] for c in model.llm.calls] == [0, 0] and [r.cached_tokens for r in reqs] == [0, 0]
    assert not model.llm.cache.shared


def test_expert_parallel_is_refused():
    model = StubModel()
    model.llm.ep_world = 2
    with pytest.raises(ValueError):
        DecoderEngine(model, prefix_cache=True)
