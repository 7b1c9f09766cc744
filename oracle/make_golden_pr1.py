"""Golden vectors for PR1 / BASELINE configs[0] (see oracle/pr1.py).  TEST INFRASTRUCTURE.

    python -m oracle.make_golden_pr1 search [--max 400]        # on a GPU box: prompt-seed search with the fp32 oracle
                                                               # on cuda (TF32 off); writes gpurun_out/pr1_search.json
    python -m oracle.make_golden_pr1 mint --prompt-seed N      # build container: fp32 oracle on the CPU, and the
                                                               # REFERENCE's own classes (needs /root/reference);
                                                               # writes tests/golden/pr1_l4.npz

`search` also runs the CUDA path (vita_b200) on every candidate that passes the margin criteria and reports whether the
32 free-running tokens agree -- information only: the seed is chosen by the margin criteria, the verdict is the test's.
"""
from __future__ import annotations

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import pr1, vita_oracle as O  # noqa: E402

GOLDEN = ROOT / "tests" / "golden" / "pr1_l4.npz"
LOGIT_GAP_MIN = 0.05      # top-1/top-2 gap >= 5 % of the top logit at every step (bf16 noise floor ~1 %)
ROUTER_GAP_MIN = 0.02     # rank-2 vs rank-3 router logit gap >= 2 % of the logits' spread (noise ~0.5 %), or harmless


def oracle_greedy(state, cfg, ids, n_new):
    """Free-running greedy decode with the oracle; returns tokens, the logits rows and the router probabilities of
    the last prompt token + every generated token (per step, per layer)."""
    lcfg = cfg.llm
    emb = O._f(state["model.embed_tokens.weight"])[ids]
    tr = []
    logits, past, _ = O.mixtral_forward(state, lcfg, emb, last_only=True, trace=tr)
    toks, rows, probs = [], [], [[t["router_probs"][-1] for t in tr]]
    for step in range(n_new):
        row = logits[0, -1]
        rows.append(row)
        nxt = int(row.argmax())
        toks.append(nxt)
        if step + 1 < n_new:
            tr = []
            e = O._f(state["model.embed_tokens.weight"])[torch.tensor([[nxt]], device=ids.device)]
            logits, past, _ = O.mixtral_forward(state, lcfg, e, past=past, last_only=True, trace=tr)
            probs.append([t["router_probs"][-1] for t in tr])
    return toks, torch.stack(rows), probs


def cmd_search(args):
    """For every router scale in --scales (powers of two: exact in bf16) walk the prompt seeds, compute the oracle's
    trajectory and margins, and run the CUDA path on every seed whose logit margins qualify -- first as shipped, then
    (if that reproduces the 32 tokens) in numerically distinct variants of itself: exp2 without the polynomial chunk,
    the narrow router summation order, a cos/sin table computed by another libm.  A seed that survives all of them is
    reproducible at bf16 precision for a reason (its decisions have real margins), not by a coin flip: a random-init MoE
    turns an ulp into another trajectory at most seeds."""
    on_gpu = torch.cuda.is_available()      # a GPU makes a candidate cost ~0.2 s instead of ~35 s; the CPU works too
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = pr1.config()
    t0 = time.time()
    state_bf16 = pr1.build_state(cfg, gate_scale=1.0)
    print(f"[pr1] state built in {time.time() - t0:.0f}s", flush=True)
    dev = "cuda" if on_gpu else "cpu"
    model = ops = None
    variants = []
    if on_gpu:
        # the CUDA path exactly as tests/test_pr1_gpu.py builds it (host-computed rope table, default options)
        from vita_b200 import ops, weights as W
        from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
        model = VITAMixtralForCausalLM(cfg, {"llm": W.pack_llm(state_bf16, cfg, "cuda")}, "cuda", max_seq_len=256,
                                       max_new_tokens=pr1.NEW_TOKENS + 1)
        rope_host = model.llm.w["rope"].clone()
        with torch.device("cuda"):
            rope_dev = W.rope_table(rope_host.shape[0], cfg.llm.head_dim, cfg.llm.rope_theta)
        print(f"[pr1] rope table host vs device libm: max |diff| {(rope_host - rope_dev).abs().max().item():.2e}", flush=True)

        def variant(name, opts=None, rope=None):
            def run(ids_cpu):
                for k, v in (opts or {}).items():
                    ops.set_option(k, v)
                if rope is not None:
                    model.llm.w["rope"].copy_(rope)
                model.llm._graphs = {}
                try:
                    return model.generate(ids_cpu.cuda(), max_new_tokens=pr1.NEW_TOKENS, output_scores=True) \
                        .sequences[0, pr1.PROMPT_LEN:].tolist()
                finally:
                    for k in (opts or {}):
                        ops.set_option(k, DEFAULTS[k])
                    model.llm.w["rope"].copy_(rope_host)
                    model.llm._graphs = {}
            return name, run
        DEFAULTS = {k: ops.get_option(k) for k in ("fa_poly", "tc_wide_route")}
        variants = [variant("as_shipped"), variant("exp2_mufu_only", {"fa_poly": 0}),
                    variant("narrow_router", {"tc_wide_route": 0}), variant("device_rope_table", rope=rope_dev),
                    variant("all_three", {"fa_poly": 0, "tc_wide_route": 0}, rope_dev)]
        state = {k: v.to("cuda").float() for k, v in state_bf16.items()}
    else:
        state = {k: v.clone() for k, v in state_bf16.items()}
    gkeys = [f"model.layers.{l}.block_sparse_moe.gate.weight" for l in range(cfg.llm.num_hidden_layers)]
    out = {"criteria": {"logit_rel_gap_min": LOGIT_GAP_MIN, "router_gap_min": ROUTER_GAP_MIN},
           "variants": [v[0] for v in variants], "scales": {}}
    cur = 1.0
    for scale in [float(x) for x in args.scales.split(",")]:
        f = scale / cur
        for l, k in enumerate(gkeys):                      # rescale the routers of both sides in place
            state[k] = state[k] * f
            state_bf16[k] = (state_bf16[k].float() * f).to(torch.bfloat16)
            if model is not None:
                model.packed["llm"]["layers"][l]["gate"].mul_(f)
        cur = scale
        gnorms = pr1.gate_norms(state_bf16, cfg)
        cands, n_ok, n_run, n_eq, n_robust = [], 0, 0, 0, 0
        for seed in range(args.first, args.max):
            ids_cpu = pr1.prompt(seed, cfg.llm.vocab_size)
            with torch.device(dev):
                toks, rows, probs = oracle_greedy(state, cfg, ids_cpu.to(dev), pr1.NEW_TOKENS)
            m = pr1.margins(rows.cpu(), [[p.cpu() for p in s] for s in probs], gnorms, cfg.llm.hidden_size)
            logit_ok = m["logit_rel_gap_min"] >= LOGIT_GAP_MIN
            ok = logit_ok and m["router_gap_min"] >= ROUTER_GAP_MIN
            rec = {"prompt_seed": seed, "logit_rel_gap_min": m["logit_rel_gap_min"],
                   "router_gap_min": m["router_gap_min"], "weight_noise_max": m["weight_noise_max"], "ok": ok,
                   "tokens": toks, "distinct_tokens": len(set(toks))}
            if model is not None and logit_ok:
                res = {}
                for name, run in variants:
                    got = run(ids_cpu)
                    res[name] = next((i for i, (a, b) in enumerate(zip(got, toks)) if a != b), None)
                    if name == "as_shipped" and res[name] is not None:
                        break                                   # not reproducible as shipped: no need for the variants
                rec["first_diff_by_variant"] = res
                rec["cuda_tokens_equal"] = res["as_shipped"] is None
                rec["robust"] = len(res) == len(variants) and all(v is None for v in res.values())
                n_run += 1
                n_eq += rec["cuda_tokens_equal"]
                n_robust += rec["robust"]
            if logit_ok or not on_gpu:
                cands.append(rec)
                print(f"[pr1] scale {scale:g}", json.dumps({k: v for k, v in rec.items() if k != "tokens"}), flush=True)
            n_ok += ok
            if n_robust >= args.want:
                break
        out["scales"][f"{scale:g}"] = {"candidates": cands, "seeds_tried": seed + 1 - args.first,
                                       "cuda_runs": n_run, "cuda_equal": n_eq, "cuda_robust": n_robust}
        print(f"[pr1] scale {scale:g}: {n_ok} margin-qualified seed(s) in {seed + 1 - args.first}; CUDA path equal on "
              f"{n_eq} of {n_run} logit-qualified seeds, in every variant on {n_robust}, {time.time() - t0:.0f}s", flush=True)
    Path("gpurun_out").mkdir(exist_ok=True)
    Path(f"gpurun_out/pr1_search{'' if on_gpu else '_cpu'}.json").write_text(json.dumps(out, indent=1))


def reference_greedy(state_bf16, cfg, ids, n_new):
    """The reference's own VITAMixtralForCausalLM (installed transformers, fp32, CPU) through the manual greedy loop of
    SURVEY.md Appendix C (HF generate() cannot run on transformers 5.x)."""
    from oracle import ref_shim
    from oracle.make_golden import to_hf5_llm_names
    ref_shim.install()
    from vita.model.language_model.vita_mixtral import VITAMixtralConfig, VITAMixtralForCausalLM
    c = cfg.llm
    hf = VITAMixtralConfig(vocab_size=c.vocab_size, hidden_size=c.hidden_size, intermediate_size=c.intermediate_size,
                           num_hidden_layers=c.num_hidden_layers, num_attention_heads=c.num_attention_heads,
                           num_key_value_heads=c.num_key_value_heads, num_local_experts=c.num_local_experts,
                           num_experts_per_tok=c.num_experts_per_tok, rms_norm_eps=c.rms_norm_eps,
                           rope_theta=c.rope_theta, max_position_embeddings=c.max_position_embeddings,
                           attn_implementation="eager", tie_word_embeddings=False)
    with torch.device("meta"):
        m = VITAMixtralForCausalLM(hf)
    sd = to_hf5_llm_names(state_bf16, c)
    missing, unexpected = m.load_state_dict(sd, strict=False, assign=True)
    missing = [k for k in missing if "rotary" not in k and "inv_freq" not in k]
    assert not missing, missing
    # buffers created on meta (rotary inv_freq) have to be materialised
    for name, buf in list(m.named_buffers()):
        if buf.is_meta:
            mod = m.get_submodule(name.rsplit(".", 1)[0]) if "." in name else m
            if "inv_freq" in name:
                D = c.head_dim
                inv = 1.0 / (c.rope_theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
                setattr(mod, name.rsplit(".", 1)[-1], inv)
    m.eval()
    toks, rows = [], []
    with torch.no_grad():
        out = m(input_ids=ids, use_cache=True)
        pkv = out.past_key_values
        for step in range(n_new):
            row = out.logits[0, -1].float()
            rows.append(row)
            nxt = int(row.argmax())
            toks.append(nxt)
            if step + 1 < n_new:
                out = m(input_ids=torch.tensor([[nxt]]), past_key_values=pkv, use_cache=True)
                pkv = out.past_key_values
    return toks, torch.stack(rows)


def cmd_mint(args):
    cfg = pr1.config()
    t0 = time.time()
    state = pr1.build_state(cfg)                     # bf16 resident; the oracle converts what it touches to fp32
    print(f"[pr1] state built in {time.time() - t0:.0f}s", flush=True)
    ids = pr1.prompt(args.prompt_seed, cfg.llm.vocab_size)
    toks, rows, probs = oracle_greedy(state, cfg, ids, pr1.NEW_TOKENS)
    m = pr1.margins(rows, probs, pr1.gate_norms(state, cfg), cfg.llm.hidden_size)
    print(f"[pr1] oracle done in {time.time() - t0:.0f}s: logit gap min {m['logit_rel_gap_min']:.4f}, router gap min "
          f"{m['router_gap_min']:.4f}", flush=True)
    ref_note = "reference not run"
    if args.reference:
        r_toks, r_rows = reference_greedy(state, cfg, ids, pr1.NEW_TOKENS)
        d = (r_rows - rows).abs().max().item()
        assert r_toks == toks, (r_toks, toks)
        assert d <= 2e-3 * rows.abs().max().item(), d
        ref_note = f"reference classes (transformers {__import__('transformers').__version__}, fp32 CPU): tokens equal, " \
                   f"max |logit diff| {d:.3e}"
        print("[pr1]", ref_note, flush=True)
    top2 = rows.topk(2, dim=-1)
    np.savez_compressed(
        GOLDEN, prompt_seed=np.int64(args.prompt_seed), input_ids=ids.numpy(), tokens=np.array(toks, dtype=np.int64),
        top2_values=top2.values.numpy().astype(np.float32), top2_indices=top2.indices.numpy(),
        logit_rel_gaps=np.array(m["logit_rel_gaps"], dtype=np.float32),
        router_gaps=np.array(m["router_gaps"], dtype=np.float32),
        first_row_head=rows[0, :4096].numpy().astype(np.float32), note=np.array(ref_note),
        gate_scale=np.float64(pr1.GATE_SCALE), head_gain_sigma=np.float64(pr1.HEAD_GAIN_SIGMA))
    print("[pr1] wrote", GOLDEN)


def main():
    ap = argparse.ArgumentParser()
    sub = ap.add_subparsers(dest="cmd", required=True)
    s = sub.add_parser("search"); s.add_argument("--max", type=int, default=400); s.add_argument("--want", type=int, default=3)
    s.add_argument("--first", type=int, default=0); s.add_argument("--scales", default=str(pr1.GATE_SCALE))
    m = sub.add_parser("mint"); m.add_argument("--prompt-seed", type=int, required=True)
    m.add_argument("--reference", action="store_true")
    args = ap.parse_args()
    {"search": cmd_search, "mint": cmd_mint}[args.cmd](args)


if __name__ == "__main__":
    main()
