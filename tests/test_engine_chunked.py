"""Chunked admission of the continuous batcher (vita_b200/engine.py, `prefill_chunk`) on the CPU.

The stand-in engine extends the one of test_engine.py with prompts of a given length that are prefilled row range by
row range.  Its per-slot state (prompt length, rows prefilled) moves with the slot on swaps, and it asserts the
protocol as it goes: chunks continue exactly where the slot stopped, the decode step never sees a half-prefilled slot,
the first token is read only after the final chunk."""
import random

import pytest
import torch

from tests.test_engine import FakeEngine, expected, stream
from vita_b200.engine import ContinuousBatcher, Request, swap_rows


class ChunkEngine(FakeEngine):
    def __init__(self, max_batch: int, cap: int):
        super().__init__(max_batch, cap)
        self.plen = torch.zeros(max_batch, dtype=torch.int64)
        self.filled = torch.zeros(max_batch, dtype=torch.int64)
        self.chunks = []                  # (engine step index, slot, rows) of every prefill call
        self.admitting = None             # seed of the request whose chunks are in flight

    def reset_slot(self, slot):
        super().reset_slot(slot)
        self.plen[slot] = 0; self.filled[slot] = 0

    def prefill(self, slot, request):
        raise AssertionError("a budgeted batcher admits through begin_prefill / prefill_rows")

    def begin_prefill(self, slot, request):
        assert self.admitting is None, "one request at a time is admitted"
        assert int(self.count[slot]) == 0 and int(self.filled[slot]) == 0, "slot must be empty"
        self.seed[slot] = request.payload["seed"]
        self.plen[slot] = request.payload["len"]
        self.admitting = request.payload["seed"]
        return request.payload["len"]

    def prefill_rows(self, slot, start, n, final):
        assert int(self.seed[slot]) == self.admitting, "the admitting request must sit in slot n_active"
        assert int(self.filled[slot]) == start and n >= 1
        self.filled[slot] += n
        assert final == (int(self.filled[slot]) == int(self.plen[slot]))
        self.chunks.append((self.steps, slot, n))
        if final:
            self.admitting = None

    def step(self, n_active):
        for s in range(n_active):
            assert int(self.filled[s]) == int(self.plen[s]) > 0, "decode step over a half-prefilled slot"
        super().step(n_active)

    def swap(self, i, j):
        super().swap(i, j)
        swap_rows([self.plen, self.filled], i, j)

    def first_token(self, slot):
        assert int(self.filled[slot]) == int(self.plen[slot]), "first token read before the final chunk"
        return super().first_token(slot)


def req(rid, seed, n, plen, arrival, **kw):
    return Request(rid, {"seed": seed, "len": plen}, n, None, arrival, **kw)


def per_step_prefill(eng):
    """{step index: prefilled rows} over the chunks issued while other requests were running (slot > 0)."""
    out = {}
    for st, slot, n in eng.chunks:
        if slot > 0:
            out[st] = out.get(st, 0) + n
    return out


@pytest.mark.parametrize("chunk", [1, 16, 64])
@pytest.mark.parametrize("trial", range(6))
def test_every_request_gets_its_own_stream_and_the_budget_holds(trial, chunk):
    rng = random.Random(1000 + trial)
    max_batch = rng.choice([1, 2, 4, 16])
    reqs = []
    for rid in range(rng.randint(1, 30)):
        n, seed = rng.randint(1, 24), rng.randint(1, 10 ** 6)
        eos = stream(seed, n)[rng.randrange(n)] if rng.random() < 0.5 else None
        reqs.append(Request(rid, {"seed": seed, "len": rng.randint(1, 300)}, n, eos, rng.randint(0, 60)))
    eng = ChunkEngine(max_batch, cap=32)
    out = ContinuousBatcher(eng, max_batch, rng.choice([1, 3]), prefill_chunk=chunk).run(reqs)
    assert set(out) == {r.rid for r in reqs}
    for r in reqs:
        assert out[r.rid] == expected(r), r.rid
        assert r.admitted_step >= r.arrival_step and r.finished_step > r.admitted_step
    assert all(v <= chunk for v in per_step_prefill(eng).values())
    assert eng.admitting is None and eng.max_active <= max_batch


def test_running_requests_advance_one_token_per_step_during_admission():
    reqs = [req(0, 11, 20, 8, 0), req(1, 12, 20, 8, 0), req(2, 13, 4, 200, 3)]
    eng = ChunkEngine(4, cap=32)
    seen = []
    out = ContinuousBatcher(eng, 4, prefill_chunk=64).run(reqs, on_step=lambda s, n: seen.append((s, n)))
    # request 0 goes in whole (nobody running), request 1 in one chunk; request 2 takes 64 + 64 + 64 + 8 rows
    assert [c[2] for c in eng.chunks] == [8, 8, 64, 64, 64, 8]
    assert reqs[2].admitted_step == 3 + 3
    # one decode step per chunk, the prefix of two keeps decoding; request 2 joins after its final chunk
    assert seen[:9] == [(0, 1), (1, 2), (2, 2), (3, 2), (4, 2), (5, 2), (6, 3), (7, 3), (8, 3)]
    assert out[0] == stream(11, 20) and out[1] == stream(12, 20) and out[2] == stream(13, 4)


def test_nothing_running_takes_the_whole_prompt_at_once():
    eng = ChunkEngine(2, cap=16)
    out = ContinuousBatcher(eng, 2, prefill_chunk=16).run([req(0, 5, 3, 500, 0)])
    assert eng.chunks == [(0, 0, 500)] and out[0] == stream(5, 3)


def test_duplex_events_fire_after_the_final_chunk():
    neg = stream(77, 1)[0]
    reqs = [req(0, 5, 30, 10, 0, session=1, negative_token_id=neg),
            req(1, 77, 6, 100, 2, session=1, negative_token_id=neg),      # noise: dropped after its last chunk
            req(2, 7, 5, 100, 4, session=1, negative_token_id=neg)]       # barge-in: interrupts request 0
    eng = ChunkEngine(4, cap=40)
    out = ContinuousBatcher(eng, 4, prefill_chunk=32).run(reqs)
    # request 1: chunks at steps 2, 3, 4, 5 (32 + 32 + 32 + 4); dropped at step 5 without taking a decode slot
    assert reqs[1].outcome == "negative" and out[1] == [neg] and reqs[1].finished_step == 5
    # request 2 starts at step 6 and finishes its prompt at step 9: request 0 produced 9 tokens before it was stopped
    assert reqs[2].admitted_step == 9 and reqs[0].finished_step == 9
    assert reqs[0].outcome == "interrupted" and out[0] == stream(5, 9)
    assert out[2] == stream(7, 5) and eng.max_active == 1


def test_retirement_during_admission_keeps_the_admitting_request_behind_the_prefix():
    # request 3 is admitted over steps 3..12; requests 0 and 1 finish meanwhile, request 2 keeps running
    reqs = [req(0, 21, 5, 4, 0), req(1, 22, 8, 4, 0), req(2, 23, 30, 4, 0), req(3, 24, 5, 160, 1)]
    eng = ChunkEngine(4, cap=40)
    out = ContinuousBatcher(eng, 4, prefill_chunk=16).run(reqs)
    for r in reqs:
        assert out[r.rid] == stream(r.payload["seed"], r.max_new_tokens), r.rid
    # (ChunkEngine checks on every chunk that request 3 sits in slot n_active, right behind the prefix)
    slots = [slot for st, slot, n in eng.chunks if 3 <= st <= 12]
    assert slots == [3, 3, 2, 2, 2, 2, 1, 1, 1, 1]
    assert reqs[3].admitted_step == 12
