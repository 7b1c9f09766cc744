"""Full-depth check of the benchmarked configuration (BASELINE configs[2]): full-size InternViT + Whale + projector
+ splice, then the 24 Mixtral layers one 80 GB H100 holds, against the fp32 oracle run layer-streamed on the same GPU (tests/full_depth.py).
Needs ~78 GB of device memory (70 GB of bf16 weights + one fp32 layer)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_configs2_full_depth_prefill_and_greedy_vs_streamed_fp32_oracle():
    torch.cuda.empty_cache()   # what earlier tests of this process still cache counts as free
    if torch.cuda.mem_get_info(0)[0] < 78e9:
        pytest.skip("needs 78 GB of free device memory (an 80 GB card with nothing else on it)")
    from oracle import vita_oracle as O
    from tests.full_depth import check_mixtral
    from tests.util import assert_close
    from vita_b200 import weights as W
    from vita_b200.config import VitaConfig, IMAGE_TOKEN_INDEX, AUDIO_TOKEN_INDEX
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    cfg = VitaConfig.full(24)
    dev = torch.device("cuda")
    enc_state = W.synthetic_state(cfg, 0, parts=("vision", "projector", "audio"))
    packed = W.random_packed(cfg, dev, seed=0, parts=("llm",))
    packed["vision"] = W.pack_vision(enc_state, cfg, dev)
    packed["projector"] = W.pack_projector(enc_state, cfg, dev)
    packed["audio"] = W.pack_audio(enc_state, cfg, dev)
    model = VITAMixtralForCausalLM(cfg, packed, dev, max_seq_len=1024, max_new_tokens=32)
    g = torch.Generator().manual_seed(0)
    ids = torch.randint(0, cfg.llm.vocab_size, (1, 128), generator=g)
    ids[0, 1], ids[0, 2] = IMAGE_TOKEN_INDEX, AUDIO_TOKEN_INDEX
    images = torch.randn(1, 3, 448, 448, generator=g)
    feats = torch.randn(1, 998, 80, generator=g)
    audios = {"audios": feats, "lengths": torch.tensor([998])}
    # (1) full-size encoders + splice: the CUDA path's spliced embeddings vs the oracle's (fp32, on the GPU)
    emb = model.prepare_inputs_labels_for_multimodal(ids, None, None, None, None, images, audios)[4]
    assert emb.shape == (1, 506, cfg.llm.hidden_size)
    with torch.device(dev):
        st = {k: v.to(dev) for k, v in enc_state.items()}
        st["model.embed_tokens.weight"] = packed["llm"]["embed"]
        ref_emb, lens = O.prepare_inputs_embeds(st, cfg, ids.to(dev), images.to(dev),
                                                {"audios": feats.to(dev), "lengths": audios["lengths"].to(dev)})
    assert lens == [506]
    assert_close(emb, ref_emb, rel=4e-2, what="full-size spliced inputs_embeds (InternViT 24L + Whale 24L + adapter)")
    del st
    # (2) 24 layers: prefill last-row logits + 8 free-running greedy tokens, against the routing-aligned fp32 oracle
    r = check_mixtral(model, emb[0], n_tokens=8)
    print(r)
    assert r["max_row_rel_err"] < 8e-2, r                        # every logits row (prefill + 7 decode steps)
    assert r["ids_equal_where_decided"] == r["ids_decided"], r   # every id the oracle decides beyond the row's error
    assert r["ids_equal"] >= 6, r                                # and most of the others (flat random-init logits)
    # routing: the CUDA path's expert pair differs from the oracle's own only at ties within the drift of the hidden
    # state (a few percent of the router-logit spread; extreme value over ~16k decisions below 0.5), and its mixing
    # weights are the oracle's
    assert r["routing_differ_frac"] < 0.06, r
    assert r["routing_differ_gap_over_spread_p99"] < 0.25 and r["routing_differ_gap_over_spread_max"] < 0.6, r
    assert r["routing_weight_err_p99"] < 0.05 and r["routing_weight_err_max"] < 0.15, r   # measured 0.036 / 0.07
