"""PR1 / BASELINE configs[0]: text-only Mixtral-8x7B geometry, 128-token prompt, bs = 1, 32 free-running greedy tokens.

TEST INFRASTRUCTURE (only tests/ and the golden scripts import this).

Full layer width (H = 4096, I = 14336, 8 experts top-2, V = 51760) at depth L = 4 -- what fits the host as fp32
(SURVEY.md section 8c/8d).  Random-init weights give flat next-token distributions: the top-1 / top-2 logit gap is
below the bf16 noise floor at ~40 % of the steps, so no bf16 implementation (the reference's own bf16 mode included)
reproduces an fp32 greedy trajectory.  SURVEY.md section 8(c) therefore asks for weights scaled so that margins are
non-degenerate and a seed chosen once and recorded:

* the lm_head rows get log-normal gains (sigma 2.5): heavy-tailed logits, the top-1 / top-2 gap is tens of percent of
  the top logit at most steps instead of 4 %;
* the router weights are scaled x8 (a power of two: exact in bf16).  Two bf16 effects compete: a rank-2 / rank-3
  near-tie flips an expert (frequency ~3 % of all decisions whatever the scale; harm = the second expert's weight, large
  for soft routers), and the noise of the top-1 / top-2 logit difference moves the mixing weights (harm ~ scale).  Round 2
  measured both ends on the GPU: x1 and x128 reproduce an fp32 trajectory less often
  than x8 / x16, where a flipped second expert mostly carries a few percent of weight and the weight noise stays ~1.5 %;
* everything else is `vita_b200.weights.synthetic_state` (std 0.02 matrices, 1 +- 0.1 norm gains), seed 0;
* the prompt seed: `make_golden_pr1.py search` walks the seeds, keeps those whose 33 logit rows are clear of near-ties
  (top-1 / top-2 gap >= 5 % of the top logit) and runs the CUDA path on them -- as shipped and in four numerically
  distinct variants of itself (exp2 without the polynomial chunk, the narrow router summation order, a cos/sin table
  from another libm, all three).  A random-init MoE is chaotic at bf16 precision: a flipped expert on a PROMPT token
  changes that token's keys and values for every later query, an ulp in the rope table is enough to move a trajectory,
  and at x16 only 4 of 21 qualified seeds reproduce the fp32 tokens.  The fixture uses a seed that every variant
  reproduces (x8: the first three qualified seeds all do; seed 33 has the most distinct tokens), i.e. one whose
  decisions have real margins; tests/test_pr1_gpu.py additionally checks arbitrary seeds against the routing-aligned
  oracle, which holds for any seed.  The chosen seed, the tokens and the observed margins are recorded in
  tests/golden/pr1_l4.npz.
"""
from __future__ import annotations

import zlib

import torch

from vita_b200 import weights as W
from vita_b200.config import VitaConfig

LAYERS = 4
PROMPT_LEN = 128
NEW_TOKENS = 32
WEIGHT_SEED = 0
HEAD_GAIN_SIGMA = 2.5
GATE_SCALE = 8.0


def config() -> VitaConfig:
    return VitaConfig.full(num_hidden_layers=LAYERS)


def head_gains(vocab: int) -> torch.Tensor:
    with torch.device("cpu"):
        g = torch.Generator(device="cpu").manual_seed(zlib.crc32(b"pr1.lm_head.row_gain"))
        return torch.exp(HEAD_GAIN_SIGMA * torch.randn(vocab, generator=g))


def build_state(cfg: VitaConfig | None = None, gate_scale: float | None = None):
    """Reference-named bf16 state dict of the PR1 model (LLM part only)."""
    cfg = cfg or config()
    gate_scale = GATE_SCALE if gate_scale is None else gate_scale
    state = W.synthetic_state(cfg, WEIGHT_SEED, parts=("llm",))
    gains = head_gains(cfg.llm.vocab_size)
    state["lm_head.weight"] = (state["lm_head.weight"].float() * gains[:, None]).to(torch.bfloat16)
    for l in range(cfg.llm.num_hidden_layers):
        k = f"model.layers.{l}.block_sparse_moe.gate.weight"
        state[k] = (state[k].float() * gate_scale).to(torch.bfloat16)
    return state


def prompt(seed: int, vocab: int) -> torch.Tensor:
    with torch.device("cpu"):      # the search runs under a cuda default device; the prompt is host data
        return torch.randint(0, vocab, (1, PROMPT_LEN), generator=torch.Generator(device="cpu").manual_seed(1000 + seed))


def margins(rows: torch.Tensor, router_probs, gate_norms=None, hidden: int = 4096) -> dict:
    """rows [n, V]: the logits the tokens were chosen from; router_probs: per step, per layer, the [E] routing
    probabilities of that token; gate_norms: per layer [E] row norms of the router weight.
    -> the smallest top-1 / top-2 logit gap relative to the top logit, and the worst router decision: for every
    decision either the rank-2 / rank-3 logit gap in units of the two logits' spread (|g_e| * rms(x): the standard
    deviation of such a logit, which its bf16 noise -- ~0.2-0.5 % of it -- is proportional to) or, when the second renormalised weight is <= 2 %, "harmless" (reported as 1.0)."""
    top = rows.float().topk(2, dim=-1).values
    rel = ((top[:, 0] - top[:, 1]) / top[:, 0].abs().clamp_min(1e-9))
    gaps, wnoise = [], 0.0
    for step in router_probs:
        for l, p in enumerate(step):
            lp = p.double().clamp_min(1e-300).log()
            srt, idx = lp.sort(descending=True)
            w2 = float(1.0 / (1.0 + torch.exp(srt[0] - srt[1])))          # renormalised weight of the second expert
            if gate_norms is not None:
                # expected bf16 noise of the mixing weights: d w2 = w2 (1 - w2) d(logit_1 - logit_2), with the noise of
                # a router logit ~0.4 % of its spread |g_e| * rms(x)
                sp12 = float(0.5 * (gate_norms[l][idx[0]] + gate_norms[l][idx[1]]))
                wnoise = max(wnoise, 0.006 * sp12 * w2 * (1.0 - w2))
            if w2 <= 0.02:
                gaps.append(1.0)
                continue
            spread = 1.0
            if gate_norms is not None:
                spread = float(0.5 * (gate_norms[l][idx[1]] + gate_norms[l][idx[2]]))   # |g_e| * rms(x), rms(x) ~ 1 after RMSNorm
            gaps.append(float(srt[1] - srt[2]) / spread)
    return {"logit_rel_gap_min": float(rel.min()), "logit_rel_gaps": rel.tolist(),
            "router_gap_min": min(gaps), "router_gaps": gaps, "weight_noise_max": wnoise}


def gate_norms(state, cfg):
    return [state[f"model.layers.{l}.block_sparse_moe.gate.weight"].float().norm(dim=-1).cpu()
            for l in range(cfg.llm.num_hidden_layers)]
