"""Sampling contract on the CPU: Philox4x32-10 known answers, the oracle's warping against the installed transformers'
warpers, and the parameter normalisation of vita_b200/sampling.py (HF kwargs and vLLM-style params)."""
import types

import numpy as np
import pytest
import torch

from oracle import sampling_oracle as SO
from vita_b200 import sampling as S


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
     (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
])
def test_philox_known_answers(ctr, key, want):
    got = tuple(int(w) for w in SO.philox4x32_10(ctr, key))
    assert got == want


def test_gumbel_noise_layout():
    """word r & 3 of the call with counter (r >> 2, n): four consecutive tokens share one Philox call"""
    seed, n = 0x0123456789ABCDEF, 7
    g = SO.gumbel(8, seed, n)
    w = SO.philox4x32_10((1, n, 0, 0), (seed & 0xFFFFFFFF, seed >> 32))
    u = ((int(w[2]) >> 8) + 0.5) * 2.0 ** -24
    assert g[6] == -np.log(-np.log(u))
    assert not np.array_equal(SO.gumbel(8, seed, n + 1), g)


def _hf_warp(logits, T, k, p):
    from transformers.generation.logits_process import (TemperatureLogitsWarper, TopKLogitsWarper,
                                                        TopPLogitsWarper)
    s = torch.tensor(logits, dtype=torch.float64)[None]
    ids = torch.zeros(1, 1, dtype=torch.long)
    s = TemperatureLogitsWarper(T)(ids, s)
    if k:
        s = TopKLogitsWarper(k)(ids, s)
    if p < 1.0:
        s = TopPLogitsWarper(p)(ids, s)
    return torch.softmax(s, -1)[0].numpy()


def _has_boundary_tie(l, k, p):
    """a value tie at the top-k or top-p boundary: HF breaks it by sort order, the contract keeps / drops ties together"""
    sv = np.sort(l)[::-1]
    if 0 < k < l.size and sv[k - 1] == sv[k]:
        return True
    return bool(np.any(np.diff(sv[: (k or l.size) + 1]) == 0)) if p < 1.0 else False


def test_warping_matches_transformers():
    rng = np.random.default_rng(3)
    checked = 0
    for trial in range(300):
        V = int(rng.choice([7, 64, 500]))
        l = rng.normal(0, rng.choice([0.5, 2.0, 6.0]), V)
        T = float(rng.choice([0.3, 0.7, 1.0, 1.5]))
        k = int(rng.choice([0, 1, 5, 50]))
        p = float(rng.choice([1.0, 0.5, 0.9, 0.95]))
        if _has_boundary_tie(l, k, p):
            continue
        want = _hf_warp(l, T, k, p)
        got = SO.probs(l, T, k, p)
        assert np.array_equal(got > 0, want > 0), (trial, V, T, k, p)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-15)
        checked += 1
    assert checked > 200


def test_oracle_choose_is_a_gumbel_max_over_the_kept_set():
    rng = np.random.default_rng(0)
    l = rng.normal(0, 2, 300)
    x, kept, _ = SO.warp(l, 0.7, 20, 0.9)
    for n in range(20):
        tok, gap, _ = SO.choose(l, 0.7, 20, 0.9, 1234, n)
        assert kept[tok] and gap >= 0
    assert SO.choose(l, 0, 0, 1.0, 0, 0)[0] == int(np.argmax(l))


# ------------------------------------------------------------------------------------------------ normalisation
def test_hf_defaults_and_greedy():
    assert S.from_hf(False, temperature=0.3, top_p=0.5, typical_p=0.2) is None      # greedy: warpers not applied
    p = S.from_hf(True, seed=5)
    assert (p.temperature, p.top_k, p.top_p, p.seed) == (1.0, 50, 1.0, 5)
    p = S.from_hf(True, temperature=None, top_k=None, top_p=None, seed=1)
    assert (p.temperature, p.top_k, p.top_p) == (1.0, 50, 1.0)
    p = S.from_hf(True, temperature=0.7, top_k=0, top_p=0.9, seed=2**64 - 1)
    assert (p.temperature, p.top_k, p.top_p, p.seed) == (0.7, 0, 0.9, 2**64 - 1)


@pytest.mark.parametrize("kw", [dict(temperature=0.0), dict(temperature=-1.0), dict(top_k=-1), dict(top_k=2.5),
                                dict(top_p=1.5), dict(top_p=-0.1), dict(typical_p=0.9), dict(min_p=0.1),
                                dict(epsilon_cutoff=3e-4), dict(eta_cutoff=1e-3), dict(repetition_penalty=1.2),
                                dict(no_repeat_ngram_size=3)])
def test_hf_errors(kw):
    with pytest.raises(ValueError):
        S.from_hf(True, seed=0, **kw)


def test_hf_neutral_unsupported_values_pass():
    assert S.from_hf(True, seed=0, repetition_penalty=1.0, typical_p=1.0, min_p=None, no_repeat_ngram_size=0)


def test_unseeded_key_follows_torch_manual_seed():
    torch.manual_seed(123)
    a = S.from_hf(True).seed
    torch.manual_seed(123)
    b = S.from_hf(True).seed
    assert a == b and 0 <= a < 2**64
    assert S.from_hf(True).seed != a
    torch.manual_seed(123)
    w = torch.randint(0, 2**32, (2,), dtype=torch.int64).tolist()
    assert a == w[0] | (w[1] << 32)


def _sp(**kw):
    base = dict(n=1, best_of=None, use_beam_search=False, presence_penalty=0.0, frequency_penalty=0.0,
                repetition_penalty=1.0, min_p=0.0, temperature=1.0, top_k=-1, top_p=1.0, seed=None)
    base.update(kw)
    return types.SimpleNamespace(**base)


def test_vllm_params():
    assert S.from_vllm(_sp(temperature=0.0)) is None
    assert S.from_vllm(_sp(temperature=0.999e-5)) is None
    p = S.from_vllm(_sp(temperature=1e-5, seed=9))
    assert p.temperature == 1e-5 and p.seed == 9
    assert S.from_vllm(_sp(temperature=0.001, top_k=-1, seed=1)).top_k == 0
    assert S.from_vllm(_sp(temperature=0.001, top_k=0, seed=1)).top_k == 0
    assert S.from_vllm(_sp(temperature=0.5, top_k=40, top_p=0.8, seed=1)).top_k == 40
    torch.manual_seed(7)
    a = S.from_vllm(_sp(temperature=0.5)).seed
    torch.manual_seed(7)
    assert S.from_vllm(_sp(temperature=0.5)).seed == a


@pytest.mark.parametrize("kw", [dict(n=2), dict(best_of=2), dict(use_beam_search=True), dict(presence_penalty=0.5),
                                dict(frequency_penalty=0.5), dict(repetition_penalty=1.1), dict(min_p=0.05)])
def test_vllm_unsupported(kw):
    with pytest.raises(NotImplementedError):
        S.from_vllm(_sp(temperature=0.7, **kw))


def test_slot_params_host_mirror():
    """SlotSampling on the CPU: device rows and the host flags follow set / swap"""
    sl = S.SlotSampling(3, "cpu")
    sl.set(1, S.SamplingParams(0.5, 7, 0.9, 2**64 - 2))
    assert sl.any_sampled(2) and not sl.any_sampled(1)
    assert sl.temperature.tolist()[:2] == [0.0, 0.5] and sl.seed[1].item() == -2 and sl.top_k[1].item() == 7
    sl.swap(0, 1)
    assert sl.any_sampled(1)
    sl.set(0, None)
    assert not sl.any_sampled(3) and sl.temperature[0].item() == 0.0
