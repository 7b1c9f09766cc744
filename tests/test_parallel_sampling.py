"""Parallel sampling on the CPU: the stream index of the sampling oracle, PagePool.fork_reserved, and the batcher's
n / best_of groups with a deterministic stand-in engine whose token streams depend only on (request, stream)."""
import random
import types

import numpy as np
import pytest
import torch

from oracle import sampling_oracle as SO
from tests import stream_oracle as SSO
from vita_b200.engine import ContinuousBatcher, Request, check_request, swap_rows
from vita_b200.model.mixtral import PagePool
from vita_b200.sampling import SamplingParams, TokenLogprobs

SP = SamplingParams(0.8, 0, 1.0, 5)


# ------------------------------------------------------------------------------------------------ oracle
def test_stream_zero_is_the_oracle_draw():
    for seed, n in ((0, 0), (0xDEADBEEF12345678, 7), (2**64 - 1, 4095)):
        assert np.array_equal(SSO.gumbel(1001, seed, n, 0), SO.gumbel(1001, seed, n))
    rng = np.random.default_rng(0)
    l = rng.normal(0, 2, 500)
    for n in range(20):
        assert SSO.choose(l, 0.9, 40, 0.9, 77, n, 0) == SO.choose(l, 0.9, 40, 0.9, 77, n)


def test_streams_differ():
    g = [SSO.gumbel(4096, 123, 3, s) for s in range(4)]
    for a in range(4):
        for b in range(a + 1, 4):
            assert not np.any(g[a] == g[b])
            assert abs(np.corrcoef(g[a], g[b])[0, 1]) < 0.06
    l = np.zeros(64)                                     # flat row: the token is the noise's arg-max
    toks = [[SSO.choose(l, 1.0, 0, 1.0, 9, n, s)[0] for n in range(32)] for s in range(3)]
    assert toks[0] != toks[1] and toks[1] != toks[2]


# ------------------------------------------------------------------------------------------------ PagePool
def _pool(B, pps, ps, shuffle=0):
    order = torch.randperm(B * pps, generator=torch.Generator().manual_seed(shuffle)) if shuffle \
        else torch.arange(B * pps)
    return PagePool(order.view(B, pps).to(torch.int32), ps)


@pytest.mark.parametrize("ps", [16, 32])
@pytest.mark.parametrize("length", [1, 15, 16, 17, 100, 128])
def test_fork_reserved_gives_private_pages(ps, length):
    B, pps, new = 4, 12, 40
    pool = _pool(B, pps, ps, shuffle=ps + length)
    n_pages = -(-(length + new) // ps)
    src_row = list(pool.table[1])
    pairs = pool.fork_reserved(1, [2, 3], length, n_pages)
    pool.check()
    full = length // ps
    assert pool.table[1] == src_row                      # src keeps its row
    for d in (2, 3):
        row = pool.table[d]
        assert row[:full] == src_row[:full]                # full prompt pages shared
        assert all(pg >= 0 for pg in row[:n_pages]) and all(pg < 0 for pg in row[n_pages:])
        for pg in row[full:n_pages]:                       # everything it can write is its own
            assert pool.refs[pg] == 1 and pg not in src_row
    for pg in src_row[:full]:
        assert pool.refs[pg] == 3
    mine = [pool.table[d][full] for d in (2, 3)]
    assert pairs == ([(src_row[full], m) for m in mine] if length % ps else [])
    assert len({pg for d in (2, 3) for pg in pool.table[d][full:n_pages]}) == 2 * (n_pages - full)
    # retiring the forks returns every page they held alone
    for d in (2, 3):
        pool.release(d)
    pool.check()
    assert [pool.refs[pg] for pg in src_row[:full]] == [1] * full
    assert len(pool.free) == 2 * pps


def test_fork_reserved_with_indexed_prefix_pages_and_eviction():
    """Admission through the prefix index, every free page indexed: the forks' pages come from eviction."""
    B, pps, ps = 3, 8, 16
    pool = _pool(B, pps, ps, shuffle=3)
    keys = [bytes([i]) * 16 for i in range(5)]
    pool.release(0)
    assert pool.admit(0, keys, pps) == 0
    pool.insert(0, keys)
    for s in (1, 2):                                     # release the other slots: their pages are free
        pool.release(s)
    # a second request over the same prefix takes the hits; the free pages are indexed under other keys
    pool.release(0)
    pool.check()
    spare = list(pool.free)
    for i, pg in enumerate(spare):
        pool.free.remove(pg)
        pool.index.add(b"x" + bytes([i]) * 15, pg)
        pool.index.lru[pg] = None
    pool.check()
    assert not pool.free
    hits = pool.admit(0, keys, 6)
    assert hits == 5
    before = pool.evictions
    pairs = pool.fork_reserved(0, [1, 2], 5 * ps + 3, 6)
    pool.check()
    assert pool.evictions > before and len(pairs) == 2
    for d in (1, 2):
        assert pool.table[d][:5] == pool.table[0][:5]
        assert pool.refs[pool.table[d][5]] == 1
    for pg in pool.table[0][:5]:
        assert pool.refs[pg] == 3 and pg in pool.index.key
    for s in (0, 1, 2):
        pool.release(s)
    pool.check()
    assert len(pool.free) + len(pool.index.lru) == B * pps


def test_fork_reserved_random_schedule_keeps_invariants():
    rng = random.Random(4)
    B, pps, ps = 6, 10, 16
    pool = _pool(B, pps, ps, shuffle=9)
    for s in range(B):
        pool.release(s)
    for _ in range(200):
        src = rng.randrange(B)
        count = rng.randint(1, B - src)
        length = rng.randint(1, 60)
        n_pages = rng.randint(length // ps + 1, pps)
        pool.release(src)
        pool.admit(src, [], n_pages)
        pool.fork_reserved(src, range(src + 1, src + count), length, n_pages)
        pool.check()
        i, j = rng.randrange(B), rng.randrange(B)
        pool.swap(i, j)
        pool.check()
        for s in rng.sample(range(B), rng.randint(0, 3)):
            pool.release(s)
        pool.check()


# ------------------------------------------------------------------------------------------------ batcher
def tok(seed, s, i):
    return (seed * 7919 + s * 15485863 + i * 104729 + (i * i) % 13) % 1000


def lp(seed, s, i):
    return -float((seed * 31 + s * 17 + i * 7) % 97) / 8.0


class GroupEngine:
    """Stand-in engine with `fork`: slot state in swapped tensors; a slot's token i is tok(seed, stream, i)."""

    def __init__(self, max_batch: int, cap: int):
        self.seed = torch.zeros(max_batch, dtype=torch.int64)
        self.strm = torch.zeros(max_batch, dtype=torch.int64)
        self.count = torch.zeros(max_batch, dtype=torch.int64)
        self.log = torch.full((max_batch, cap), -1, dtype=torch.int64)
        self.forks, self.admitted = [], []

    def reset_slot(self, slot):
        self.seed[slot] = 0; self.strm[slot] = 0; self.count[slot] = 0; self.log[slot] = -1

    def prefill(self, slot, r):
        assert int(self.count[slot]) == 0
        self.seed[slot], self.strm[slot] = r.payload["seed"], 0
        self.admitted.append(r.rid)

    def begin_prefill(self, slot, r):
        self.prefill(slot, r)
        return r.payload.get("len", 40)

    def prefill_rows(self, slot, start, n, final):
        pass

    def fork(self, slot, count, max_new_tokens):
        self.forks.append((slot, count))
        for j in range(1, count):
            self.seed[slot + j], self.strm[slot + j] = self.seed[slot], j
            self.count[slot + j] = 0
            self.log[slot + j] = -1

    def step(self, n_active):
        for s in range(n_active):
            i = int(self.count[s])
            self.log[s, i] = tok(int(self.seed[s]), int(self.strm[s]), i)
            self.count[s] += 1

    def swap(self, i, j):
        swap_rows([self.seed, self.strm, self.count, self.log], i, j)

    def read_tokens(self, slot):
        return self.log[slot, : int(self.count[slot])].tolist()

    def read_logprobs(self, slot, tokens, n_top):
        seed, s = int(self.seed[slot]), int(self.strm[slot])
        return [TokenLogprobs(t, lp(seed, s, i), 1) for i, t in enumerate(tokens)]

    def first_token(self, slot):
        return tok(int(self.seed[slot]), int(self.strm[slot]), 0)


def _expected(r: Request):
    k = r.best_of or r.n
    seqs = []
    for j in range(k):
        toks = [tok(r.payload["seed"], j, i) for i in range(r.max_new_tokens)]
        if r.eos_token_id is not None and r.eos_token_id in toks:
            toks = toks[: toks.index(r.eos_token_id) + 1]
        seqs.append((j, toks, sum(lp(r.payload["seed"], j, i) for i in range(len(toks)))))
    if k > r.n:
        seqs = sorted(seqs, key=lambda q: (-q[2], q[0]))[: r.n]
    return seqs


def _req(rid, seed, new, arrival=0, n=1, best_of=None, eos=None, logprobs=None, sampled=True, plen=40):
    return Request(rid, {"seed": seed, "len": plen}, new, eos, arrival_step=arrival,
                   sampling=SP if sampled else None, logprobs=logprobs, n=n, best_of=best_of)


@pytest.mark.parametrize("chunk", [None, 16])
@pytest.mark.parametrize("sync_every", [1, 3])
@pytest.mark.parametrize("trial", range(5))
def test_groups_get_their_own_streams(trial, sync_every, chunk):
    rng = random.Random(trial)
    max_batch = rng.choice([4, 6, 8])
    reqs = []
    for rid in range(rng.randint(3, 20)):
        k = rng.choice([1, 1, 2, 3, max_batch])
        n = rng.randint(1, k)
        best_of = k if (k > n or rng.random() < 0.5) else None
        new = rng.randint(1, 15)
        seed = rng.randint(1, 10 ** 6)
        eos = tok(seed, rng.randrange(k), rng.randrange(new)) if rng.random() < 0.4 else None
        reqs.append(_req(rid, seed, new, rng.randint(0, 25), n, best_of, eos,
                         rng.choice([None, 0, 2]), plen=rng.randint(2, 60)))
    eng = GroupEngine(max_batch, 64)
    done = ContinuousBatcher(eng, max_batch, sync_every=sync_every, prefill_chunk=chunk).run(reqs)
    for r in reqs:
        want = _expected(r)
        assert [(q.index, q.tokens) for q in r.sequences] == [(j, t) for j, t, _ in want], r.rid
        assert done[r.rid] == r.tokens == want[0][1]
        assert r.outcome == "finished" and all(q.outcome == "finished" for q in r.sequences)
        for q, (_, toks, cum) in zip(r.sequences, want):
            if r.logprobs is not None or (r.best_of or r.n) > r.n:
                assert q.cumulative_logprob == pytest.approx(cum)
            else:
                assert q.cumulative_logprob is None
            assert [t.token for t in q.token_logprobs] == (toks if r.logprobs is not None else [])
        assert r.token_logprobs == r.sequences[0].token_logprobs
    assert [s for s, c in eng.forks] and all(c > 1 for s, c in eng.forks)


def test_group_waits_for_its_slots_first_come_first_served():
    reqs = [_req(0, 11, 10, 0), _req(1, 12, 10, 0), _req(2, 13, 4, 1, n=3), _req(3, 14, 2, 2)]
    eng = GroupEngine(4, 32)
    ContinuousBatcher(eng, 4).run(reqs)
    # the group needs 3 free slots: it waits for both running requests; request 3 arrives later and waits behind it
    assert eng.admitted == [0, 1, 2, 3]
    assert reqs[2].admitted_step == 10 and reqs[3].admitted_step >= reqs[2].admitted_step
    assert eng.forks == [(0, 3)]


def test_forks_sit_right_behind_the_prefix():
    """A group admitted behind running requests forks into the slots right after its own; retirements swap them."""
    reqs = [_req(0, 21, 3, 0), _req(1, 22, 9, 0), _req(2, 23, 6, 1, n=2, best_of=3), _req(3, 24, 5, 2)]
    eng = GroupEngine(6, 32)
    ContinuousBatcher(eng, 6, sync_every=2, prefill_chunk=8).run(reqs)
    assert eng.forks == [(1, 3)]             # request 0 retired during the chunked admission: the group moved down
    for r in reqs:
        assert [(q.index, q.tokens) for q in r.sequences] == [(j, t) for j, t, _ in _expected(r)]


def test_best_of_ranking_breaks_ties_by_index(monkeypatch):
    import tests.test_parallel_sampling as me
    monkeypatch.setattr(me, "lp", lambda seed, s, i: -1.0 if s in (1, 2) else -2.0)
    r = _req(0, 5, 4, n=2, best_of=4)
    ContinuousBatcher(GroupEngine(4, 16), 4).run([r])
    assert [q.index for q in r.sequences] == [1, 2]
    assert [q.cumulative_logprob for q in r.sequences] == [-4.0, -4.0]
    assert r.tokens == r.sequences[0].tokens == [tok(5, 1, i) for i in range(4)]


def test_single_sequence_requests_are_unchanged():
    r = _req(0, 9, 5)
    done = ContinuousBatcher(GroupEngine(2, 16), 2).run([r])
    assert done == {0: [tok(9, 0, i) for i in range(5)]}
    assert [(q.index, q.tokens, q.cumulative_logprob) for q in r.sequences] == [(0, done[0], None)]


@pytest.mark.parametrize("kw,match", [
    (dict(n=2, sampled=False), "greedy"),
    (dict(n=1, best_of=2, sampled=False), "greedy"),
    (dict(n=3, best_of=2), "best_of"),
    (dict(n=5), "max_batch"),
    (dict(n=2, best_of=5), "max_batch"),
    (dict(n=0), "positive"),
    (dict(n=2, best_of=0), "positive"),
])
def test_refusals(kw, match):
    r = _req(0, 1, 4, **kw)
    with pytest.raises(ValueError, match=match):
        ContinuousBatcher(GroupEngine(4, 16), 4).run([r])
    with pytest.raises(ValueError, match=match):
        check_request(r, 4)


@pytest.mark.parametrize("field,value", [("session", 1), ("negative_token_id", 7)])
def test_duplex_fields_are_refused_with_groups(field, value):
    r = _req(0, 1, 4, n=2)
    setattr(r, field, value)
    with pytest.raises(ValueError, match="duplex"):
        ContinuousBatcher(GroupEngine(4, 16), 4).run([r])
    r.n = 1
    ContinuousBatcher(GroupEngine(4, 16), 4).run([r])      # a single sequence keeps the duplex fields


def test_positional_construction_keeps_working():
    r = Request(3, {}, 8, 2, 1, None, None, SP, 4)
    assert (r.n, r.best_of, r.sequences, r.logprobs) == (1, None, [], 4)


# ------------------------------------------------------------------------------------------------ generate()
def _stub_model(max_batch=4, ep_world=1):
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    m = object.__new__(VITAMixtralForCausalLM)
    m.llm = types.SimpleNamespace(max_batch=max_batch, ep_world=ep_world)
    return m


@pytest.mark.parametrize("kw,match", [
    (dict(num_return_sequences=2), "num_return_sequences"),                  # greedy
    (dict(do_sample=True, num_return_sequences=5), "max_batch"),
    (dict(do_sample=True, num_return_sequences=0), "positive"),
    (dict(num_return_sequences=0), "positive"),
    (dict(do_sample=True, num_return_sequences=2, max_new_tokens=0), "max_new_tokens"),
])
def test_generate_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        _stub_model().generate(torch.zeros(1, 4, dtype=torch.long), **kw)


def test_generate_refuses_expert_parallel():
    with pytest.raises(ValueError, match="expert-parallel"):
        _stub_model(ep_world=2).generate(torch.zeros(1, 4, dtype=torch.long), do_sample=True, num_return_sequences=2)
