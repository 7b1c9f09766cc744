"""PR1 / BASELINE configs[0]: text-only Mixtral-8x7B geometry (full layer width, depth 4), 128-token prompt, bs = 1,
32 FREE-RUNNING greedy tokens.

(1) Against the fixture minted from the reference's own classes (oracle/make_golden_pr1.py mint --reference): every token
    id must equal the reference's -- no margin gating, no teacher forcing.  The weight scaling and the prompt seed that
    make an fp32 trajectory reproducible in bf16 are described in oracle/pr1.py (the seed came from a search over prompts).
(2) For other prompt seeds, against the fp32 oracle run on the same GPU with the routing aligned (tests/full_depth.py):
    every one of the 32 logits rows within tolerance and every id the oracle decides beyond that row's error equal.
    This form holds for ANY seed: a random-init MoE turns a rank-2 / rank-3 router near-tie on a prompt token into a
    different trajectory, which no bf16 implementation (the reference's own included) can avoid."""
from pathlib import Path

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden" / "pr1_l4.npz"


def _build(gate_scale=None):
    from oracle import pr1
    from vita_b200 import weights as W
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = pr1.config()
    state = pr1.build_state(cfg, gate_scale)
    model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(state, cfg, "cuda")}, "cuda", max_seq_len=256,
                                   max_new_tokens=pr1.NEW_TOKENS + 1)
    del state
    return cfg, model


@pytest.fixture(scope="module")
def pr1_model():
    return _build()


@pytest.fixture(scope="module")
def pr1_model_unit_router():
    # the routing-aligned comparison takes the discrete decisions out, so the routers stay at their natural scale: the
    # mixing weights are then smooth in the logits (sharpened x16 a near-tied pair turns 1 % of logit noise into 10 % of
    # weight noise: measured row errors 0.1-1.0 at depth 4, against 0.01-0.02 at scale 1)
    return _build(1.0)


@pytest.mark.skipif(not GOLDEN.exists(), reason="tests/golden/pr1_l4.npz not minted yet")
def test_pr1_free_running_greedy_token_ids_exact(pr1_model):
    from oracle import pr1
    cfg, model = pr1_model
    g = np.load(GOLDEN)
    assert float(g["gate_scale"]) == pr1.GATE_SCALE, "fixture minted with another router scale"
    ids = pr1.prompt(int(g["prompt_seed"]), cfg.llm.vocab_size)
    assert np.array_equal(ids.numpy(), g["input_ids"]), "prompt generator drifted from the fixture"
    want = g["tokens"].tolist()
    out = model.generate(ids.cuda(), max_new_tokens=pr1.NEW_TOKENS, output_scores=True)
    got = out.sequences[0, pr1.PROMPT_LEN:].tolist()
    print("oracle margins: logit gap min %.3f, router gap min %.3f" % (g["logit_rel_gaps"].min(), g["router_gaps"].min()))
    assert got == want, (got, want)
    # the logits the tokens were chosen from: top-2 values of every step within bf16 tolerance of the oracle's
    rows = torch.cat(list(out.scores)).float().cpu()
    idx = torch.from_numpy(g["top2_indices"])
    ref = torch.from_numpy(g["top2_values"])
    per_row = ((rows.gather(1, idx) - ref).abs() / ref[:, :1].abs())
    rel = per_row.max().item()
    print(f"top-2 logit values: max rel err {rel:.3e}; per row (top-1, top-2): {[[round(float(x), 3) for x in r] for r in per_row]}")
    print("cuda top-2 values of the first rows:", rows.gather(1, idx)[:4].tolist(), "oracle:", ref[:4].tolist())
    # The ids are the bar.  The VALUES agree to a few percent at most steps; at a step where an expert flipped upstream (a
    # rank-2 / rank-3 router near-tie resolved differently in bf16, see oracle/pr1.py) the hidden state differs visibly
    # although the token survives on its margin.  Measured on the fixture: 29 of 32 rows below 0.06, three at 0.12-0.88.
    worst = per_row.max(dim=1).values
    assert float(worst.median()) < 3e-2 and int((worst < 0.1).sum()) >= 27, per_row
    # CUDA-graph replay, eager launches and a different read-back cadence give the same ids
    again = model.generate(ids.cuda(), max_new_tokens=pr1.NEW_TOKENS, use_graph=False, sync_every=5)
    assert again.sequences[0, pr1.PROMPT_LEN:].tolist() == want


@pytest.mark.parametrize("prompt_seed", [0, 1, 2])
def test_pr1_any_seed_against_the_routing_aligned_oracle(pr1_model_unit_router, prompt_seed):
    from oracle import pr1
    from tests.full_depth import check_mixtral
    cfg, model = pr1_model_unit_router
    ids = pr1.prompt(prompt_seed, cfg.llm.vocab_size)
    emb = model.packed["llm"]["embed"][ids[0].cuda()].contiguous()
    r = check_mixtral(model, emb, n_tokens=pr1.NEW_TOKENS)
    print({k: v for k, v in r.items() if k not in ("oracle_top2_rel_gap",)})
    # measured (round 2, three seeds): rows 0.005-0.084, median ~0.025 (the log-normal lm_head gains put the largest
    # logits on a few rows); without the alignment the FIRST row is already off by 0.02 / 0.71 / 0.16
    rows = sorted(r["row_rel_err"])
    assert rows[len(rows) // 2] < 3.5e-2 and rows[-1] < 0.1, r   # all 32 logits rows, depth 4
    assert r["ids_equal_where_decided"] == r["ids_decided"] and r["ids_decided"] >= 16, r
    assert r["ids_equal"] >= 30, r
    assert r["routing_differ_frac"] < 0.04 and r["routing_weight_err_p99"] < 0.03, r
