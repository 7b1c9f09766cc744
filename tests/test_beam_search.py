"""Beam search on the CPU: the oracle (tests/beam_oracle.py) against the installed transformers' own
generate(num_beams=N), the library's bookkeeping (vita_b200/beam.py) against the oracle, the copy-on-write page pool
and the parameter refusals of generate()."""
import itertools
import random
import types

import numpy as np
import pytest
import torch

from tests.beam_oracle import beam_search as oracle_beam_search
from vita_b200.beam import MAX_BEAMS, BeamSearch, check_beam_args, pack_outputs
from vita_b200.model.mixtral import PagePool

V, L, T = 40, 5, 7
EOS = 3


def _table(seed: int, eos_case: str) -> torch.Tensor:
    """logits[step, last token] [T, V, V]: a seeded table; EOS wins early, late or never."""
    g = torch.Generator().manual_seed(seed)
    tab = torch.randn(T, V, V, generator=g) * 2.0
    if eos_case == "early":
        tab[1, :, EOS] += 3.0
    elif eos_case == "late":
        tab[T - 2, :, EOS] += 3.0
    else:
        tab[:, :, EOS] = -30.0
    return tab


def _rows(tab, prompt, tokens, step):
    """fp32 log-softmax rows of the running beams (tokens [n, step]), as the stub model's logits give them."""
    last = [prompt[-1] if step == 0 else int(t[-1]) for t in tokens]
    return torch.log_softmax(tab[step, last].float(), dim=-1)


def _hf_model(tab):
    import torch.nn as nn
    from transformers import GenerationMixin, PretrainedConfig, PreTrainedModel
    from transformers.modeling_outputs import CausalLMOutputWithPast

    class StubConfig(PretrainedConfig):
        model_type = "vita-beam-stub"

    class StubLM(PreTrainedModel, GenerationMixin):
        config_class = StubConfig

        def __init__(self, config):
            super().__init__(config)
            self.anchor = nn.Parameter(torch.zeros(1))

        def forward(self, input_ids=None, **kw):
            B, S = input_ids.shape
            logits = torch.zeros(B, S, V)
            logits[:, -1] = tab[S - L, input_ids[:, -1]]
            return CausalLMOutputWithPast(logits=logits)

    return StubLM(StubConfig(vocab_size=V)).eval()


GRID = list(itertools.product([2, 3, 4, 8], [1.0, 0.0, -0.5, 2.0], [False, True, "never"], ["one", "all"],
                              ["early", "late", "never"]))


@pytest.mark.parametrize("N,lp,es,R,eos_case", GRID)
def test_oracle_matches_transformers(N, lp, es, R, eos_case):
    seed = GRID.index((N, lp, es, R, eos_case))
    R = 1 if R == "one" else N
    tab = _table(seed, eos_case)
    prompt = torch.randint(4, V, (L,), generator=torch.Generator().manual_seed(seed)).tolist()
    model = _hf_model(tab)
    with torch.no_grad():
        out = model.generate(torch.tensor([prompt]), num_beams=N, max_new_tokens=T, eos_token_id=EOS,
                             pad_token_id=EOS, length_penalty=lp, early_stopping=es, num_return_sequences=R,
                             do_sample=False, output_scores=True, return_dict_in_generate=True, use_cache=False)
    seqs, scores, idx, steps = oracle_beam_search(lambda toks, step: _rows(tab, prompt, toks.tolist(), step), N, T,
                                                  EOS, lp, es, R)
    hf_new = out.sequences[:, L:]
    assert torch.equal(out.sequences[:, :L], torch.tensor([prompt] * R))
    assert torch.equal(hf_new, seqs)
    assert torch.equal(out.beam_indices.to(torch.int64), idx)
    assert torch.allclose(out.sequences_scores.float(), scores, rtol=0, atol=1e-6)
    assert len(out.scores) == steps


def _library(tab, prompt, N, lp, es, R):
    """vita_b200.beam over each running beam's top 2N of the same rows (row order: value descending, index
    ascending, as the kernel's top-N)."""
    bs = BeamSearch(N, T, EOS, lp, es)
    steps = 0
    while not bs.done:
        rows = _rows(tab, prompt, [b.tokens for b in bs.running], steps).numpy()
        order = np.lexsort((np.arange(V)[None, :].repeat(len(rows), 0), -rows), axis=1)[:, :2 * N]
        bs.step(order.tolist(), np.take_along_axis(rows, order, axis=1))
        steps += 1
    return bs.best(R), steps


@pytest.mark.parametrize("N,lp,es,R,eos_case", GRID[::5])
def test_library_matches_oracle(N, lp, es, R, eos_case):
    seed = 1000 + GRID.index((N, lp, es, R, eos_case))
    R = 1 if R == "one" else N
    tab = _table(seed, eos_case)
    prompt = torch.randint(4, V, (L,), generator=torch.Generator().manual_seed(seed)).tolist()
    seqs, scores, idx, steps = oracle_beam_search(lambda toks, step: _rows(tab, prompt, toks.tolist(), step), N, T,
                                                  EOS, lp, es, R)
    hyps, lib_steps = _library(tab, prompt, N, lp, es, R)
    seq, sc, bi = pack_outputs(hyps, prompt, EOS)
    assert lib_steps == steps
    assert np.array_equal(seq[:, L:], seqs.numpy()) and np.array_equal(seq[:, :L], np.array([prompt] * R))
    assert np.array_equal(bi, idx.numpy())
    assert np.array_equal(sc, scores.numpy())          # same fp32 operations: bit-equal


def test_finalize_adds_running_beams():
    bs = BeamSearch(2, 10, eos_token_id=None)
    bs.step([[5, 6, 7, 8]], [[-0.5, -1.0, -2.0, -3.0]])
    assert [b.tokens for b in bs.running] == [[5], [6]]
    bs.finalize()
    assert bs.done and [h.tokens for h in bs.best(2)] == [[5], [6]]
    assert [float(h.score) for h in bs.best(2)] == [-0.5, -1.0]


# ------------------------------------------------------------------------------------------------ page pool
def _check_pool(pool, rows, lineage, mem, length, ps):
    pool.check()
    w = length // ps
    write_pages = [pool.table[b][w] for b in range(rows)]
    assert len(set(write_pages)) == rows and min(write_pages) >= 0, "write pages must be private"
    for b in range(rows):
        assert all(pg == -1 for pg in pool.table[b][w + 1:]), "no pages past the write page"
        got = [mem[pool.table[b][p // ps]][p % ps] for p in range(length)]
        assert got == lineage[b], "a beam reads another beam's rows"


@pytest.mark.parametrize("ps", [16, 32])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_page_pool_invariants(ps, seed):
    rng = random.Random(seed)
    max_batch, pps, N = 6, 5, 4
    static = torch.randperm(max_batch * pps, generator=torch.Generator().manual_seed(seed)).view(max_batch, pps)
    pool = PagePool(static.to(torch.int32), ps)
    mem = {pg: [None] * ps for pg in range(max_batch * pps)}
    prompt = ps + 7 + seed
    for p in range(prompt):                                   # the prompt in slot 0's static pages
        mem[pool.table[0][p // ps]][p % ps] = ("prompt", p)
    lineage = [[("prompt", p) for p in range(prompt)]]

    def apply(pairs):
        for src, dst in pairs:
            mem[dst] = list(mem[src])

    apply(pool.fork(0, [1, 2, 3], prompt))
    lineage = [list(lineage[0]) for _ in range(N)]
    length = prompt
    _check_pool(pool, N, lineage, mem, length, ps)
    while length < pps * ps - 1:
        for b in range(N):                                    # the step writes each beam's row at `length`
            tok = (b, length, rng.random())
            mem[pool.table[b][length // ps]][length % ps] = tok
            lineage[b].append(tok)
        length += 1
        parents = [rng.randrange(N) for _ in range(N)]
        apply(pool.reorder(parents, length))
        lineage = [list(lineage[p]) for p in parents]
        _check_pool(pool, N, lineage, mem, length, ps)
    pool.reset()
    pool.check()
    assert pool.table == static.tolist() and pool.free == [] and all(r == 1 for r in pool.refs)


def test_page_pool_keeps_one_original():
    pool = PagePool(torch.arange(8, dtype=torch.int32).view(2, 4), 16)
    pairs = pool.fork(0, [1], 20)                             # partial page 1 of slot 0: copied once
    assert len(pairs) == 1 and pairs[0][0] == 1 and pool.table[0][1] == 1
    assert pool.table[1][0] == 0 and pool.refs[0] == 2
    assert pool.reorder([0, 0], 21) == [(1, pool.table[0][1])] and pool.table[1][1] == 1
    pool.check()


# ------------------------------------------------------------------------------------------------ refusals
def _stub_model(max_batch=4, ep_world=1):
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    m = object.__new__(VITAMixtralForCausalLM)
    m.llm = types.SimpleNamespace(max_batch=max_batch, ep_world=ep_world)
    return m


@pytest.mark.parametrize("kw,match", [
    (dict(num_beams=2, do_sample=True), "beam-sample"),
    (dict(num_beams=2, logprobs=3), "logprobs"),
    (dict(num_beams=8), "max_batch"),
    (dict(num_beams=11), "MAX_LOGPROBS"),
    (dict(num_beams=0), "positive"),
    (dict(num_beams=2, num_return_sequences=3), "num_return_sequences"),
    (dict(num_beams=2, num_return_sequences=0), "num_return_sequences"),
    (dict(num_beams=2, early_stopping="sometimes"), "early_stopping"),
])
def test_generate_refusals(kw, match):
    with pytest.raises(ValueError, match=match):
        _stub_model().generate(torch.zeros(1, 4, dtype=torch.long), **kw)


def test_generate_refuses_expert_parallel():
    with pytest.raises(ValueError, match="expert-parallel"):
        _stub_model(ep_world=2).generate(torch.zeros(1, 4, dtype=torch.long), num_beams=2)


def test_max_beams_follows_logprob_width():
    assert MAX_BEAMS == 10
    check_beam_args(10, 10, "never")
    with pytest.raises(ValueError):
        check_beam_args(True, 1, False)


def test_last_step_keeps_running_beams_for_the_criteria():
    bs = BeamSearch(2, 1, eos_token_id=5)
    assert bs.step([[5, 6, 7, 8]], [[-0.5, -1.0, -2.0, -3.0]]) == [] and bs.done
    assert [b.tokens for b in bs.running] == [[6], [7]]           # 4.41's running beams of the last step
    assert [h.tokens for h in bs.best(2)] == [[5], [6]]           # 5.5.0: the top-N candidates are finalized
    bs.finalize()                                                  # a criterion firing on the last step adds nothing
    assert [h.tokens for h in bs.best(2)] == [[5], [6]]


def test_cache_unshare_restores_the_table():
    from vita_b200.config import VitaConfig
    from vita_b200.model.mixtral import PagedKVCache
    cache = PagedKVCache(VitaConfig.tiny().llm, 3, 64, "cpu", shuffle_pages=True)
    static = cache.block_table.clone()
    cache.fork(0, [1, 2], 32)                  # at a page boundary: fresh pages only, nothing to copy
    assert not torch.equal(cache.block_table, static) and cache.shared
    cache.unshare()
    assert torch.equal(cache.block_table, static) and not cache.shared and cache.pool.free == []
