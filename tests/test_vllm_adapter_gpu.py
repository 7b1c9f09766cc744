"""The vLLM-facing model class (vita_b200/vllm_adapter.py) driven the way the reference's engine drives
`MixtralForConditionalGeneration` (web_demo/vllm_tools/vllm_file/mixtral.py:1130-1186): flattened tokens, engine-owned
paged KV cache in vLLM's flash layout with shuffled blocks, a prompt step that mixes a multimodal and a text-only
sequence, then steps that mix decodes of both.  Checked against `VITAMixtralForCausalLM.generate` on the same weights
(itself checked against the reference-minted goldens)."""
import pytest
import torch

from vita_b200 import weights as W
from vita_b200.config import VitaConfig, IMAGE_TOKEN_INDEX, AUDIO_TOKEN_INDEX

pytestmark = pytest.mark.gpu

IMG_ID, AUD_ID = 2000, 2001          # placeholder ids inside the tiny vocabulary (config.json: 51000 / 51001)


def _blocks_for(n_tokens, block_size, free):
    return [free.pop() for _ in range((n_tokens + block_size - 1) // block_size)]


def test_engine_call_sequence_matches_generate(golden):
    from vita_b200.model.vita_mixtral import VITAMixtralForCausalLM
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration, TokenBatch
    inp, _ = golden
    cfg = VitaConfig.tiny()
    state = W.synthetic_state(cfg, 0)
    dev = torch.device("cuda")
    # the engine hands over (name, tensor) pairs; path B skips the CMVN buffers (applied in its feature extractor)
    pairs = [("language_model." + k if k.startswith(("model.layers", "model.embed", "model.norm", "lm_head")) else k, v)
             for k, v in state.items() if "global_cmvn" not in k]
    m = MixtralForConditionalGeneration(cfg, device=dev, image_token_index=IMG_ID, audio_token_index=AUD_ID)
    used = m.load_weights(pairs)
    assert len(used) == len(pairs)
    # the path-A model with the same weights and identity CMVN is the checker
    st = dict(state)
    st[W.PREFIX_AUDIO + "encoder.global_cmvn.mean"] = torch.zeros(cfg.audio.input_dim)
    st[W.PREFIX_AUDIO + "encoder.global_cmvn.istd"] = torch.ones(cfg.audio.input_dim)
    ref = VITAMixtralForCausalLM(cfg, W.pack(st, cfg, dev), dev, max_new_tokens=16)

    images = torch.from_numpy(inp["images"])[:1]
    feats = torch.from_numpy(inp["feats"])[:1]                       # [1, 100, 80]
    n_img = cfg.vision.out_tokens
    n_aud = cfg.audio.tokens_after_adapter(cfg.audio.frames_after_subsampling(feats.shape[1]))
    g = torch.Generator().manual_seed(5)
    text_a = torch.randint(3, 1900, (7,), generator=g).tolist()
    text_b = torch.randint(3, 1900, (11,), generator=g).tolist()
    # path A prompt: one placeholder per modality; path B prompt: one placeholder id PER feature token (:1084-1128)
    ids_a_ref = torch.tensor([text_a[:2] + [IMAGE_TOKEN_INDEX] + text_a[2:5] + [AUDIO_TOKEN_INDEX] + text_a[5:]])
    ids_a = text_a[:2] + [IMG_ID] * n_img + text_a[2:5] + [AUD_ID] * n_aud + text_a[5:]
    ids_b = text_b
    N_NEW = 6
    def ref_tokens(ids, **kw):
        """tokens + how many of them were chosen with a clear top-1/top-2 margin (the engine path scores through the
        GEMM kernels, generate() through the decode GEMVs: near-ties may legitimately resolve differently)"""
        out = ref.generate(ids, max_new_tokens=N_NEW, output_scores=True, **kw)
        rows = torch.cat(list(out.scores)).float()
        top = rows.topk(2, dim=-1).values
        clear = ((top[:, 0] - top[:, 1]) > 0.03 * rows.abs().max()).tolist()
        n = 0
        while n < N_NEW and clear[n]:
            n += 1
        return out.sequences[0, ids.shape[1]:].tolist(), n

    want_a, n_a = ref_tokens(ids_a_ref, images=images, audios={"audios": feats, "lengths": torch.tensor([feats.shape[1]])})
    want_b, n_b = ref_tokens(torch.tensor([ids_b]))
    assert n_a >= 1 and n_b >= 1

    # ---- engine side: block manager with shuffled blocks, vLLM flash KV layout
    bs, n_blocks = 16, 64
    c = cfg.llm
    kv_caches = [torch.zeros(2, n_blocks, bs, c.num_key_value_heads, c.head_dim, dtype=torch.bfloat16, device=dev)
                 for _ in range(c.num_hidden_layers)]
    free = torch.randperm(n_blocks, generator=g).tolist()
    seqs = [list(ids_a), list(ids_b)]
    cap = [len(s) + N_NEW for s in seqs]
    tables = [_blocks_for(n, bs, free) for n in cap]
    max_blocks = max(len(t) for t in tables)
    bt = torch.tensor([t + [0] * (max_blocks - len(t)) for t in tables], dtype=torch.int32, device=dev)

    def slots(seq_i, positions):
        return [tables[seq_i][p // bs] * bs + p % bs for p in positions]

    # step 0: both prompts in one flattened batch (prefill tokens of A, then of B)
    pos = list(range(len(ids_a))) + list(range(len(ids_b)))
    meta = TokenBatch(torch.tensor(slots(0, range(len(ids_a))) + slots(1, range(len(ids_b))), dtype=torch.int32, device=dev),
                      bt, [0, len(ids_a), len(ids_a) + len(ids_b)], [len(ids_a), len(ids_b)])
    audio_mask = torch.ones(1, feats.shape[1], dtype=torch.bool)
    hidden = m.forward(torch.tensor(ids_a + ids_b), torch.tensor(pos), kv_caches, meta, pixel_values=images.to(dev),
                       audio_input=feats.to(dev), audio_mask=audio_mask.to(dev))
    assert hidden.shape == (len(ids_a) + len(ids_b), c.hidden_size)

    class Sel:   # SamplingMetadata stand-in: score the last token of every sequence
        selected_token_indices = torch.tensor([len(ids_a) - 1, len(ids_a) + len(ids_b) - 1])
    nxt = m.sample(m.compute_logits(hidden, Sel)).tolist()
    got = [[nxt[0]], [nxt[1]]]
    for _ in range(N_NEW - 1):      # decode steps: one token per sequence, flattened
        for i in range(2):
            seqs[i].append(got[i][-1])
        lens = [len(s) for s in seqs]
        meta = TokenBatch(torch.tensor([slots(0, [lens[0] - 1])[0], slots(1, [lens[1] - 1])[0]], dtype=torch.int32, device=dev),
                          bt, [0, 1, 2], lens)
        hidden = m.forward(torch.tensor([seqs[0][-1], seqs[1][-1]]), torch.tensor([lens[0] - 1, lens[1] - 1]), kv_caches,
                           meta)
        nxt = m.sample(m.compute_logits(hidden)).tolist()
        got[0].append(nxt[0]); got[1].append(nxt[1])
    assert got[1][:n_b] == want_b[:n_b], (got[1], want_b, n_b)
    assert got[0][:n_a] == want_a[:n_a], (got[0], want_a, n_a)


def test_placeholder_count_mismatch_raises(golden):
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration
    cfg = VitaConfig.tiny()
    dev = torch.device("cuda")
    m = MixtralForConditionalGeneration(cfg, device=dev, image_token_index=IMG_ID, audio_token_index=AUD_ID,
                                        packed=W.pack(W.synthetic_state(cfg, 0), cfg, dev))
    ids = torch.tensor([5, IMG_ID, IMG_ID, 6], device=dev)
    emb = torch.zeros(4, cfg.llm.hidden_size, dtype=torch.bfloat16, device=dev)
    with pytest.raises(ValueError, match="placeholders"):     # mixtral.py:1110-1124
        m.merge_multimodal_embeddings(ids, emb, torch.zeros(1, 3, cfg.llm.hidden_size, dtype=torch.bfloat16, device=dev),
                                      None, IMG_ID)
    with pytest.raises(ValueError, match="expected shape"):   # mixtral.py:974-979
        m._validate_pixel_values(torch.zeros(1, 3, 8, 8))


def test_adapter_equals_decoder_bitwise():
    """The adapter runs the decoder's layer loop over the engine's pages: the same kernels over the same rows.  One
    whole prompt gives the logits of `prefill(all_logits=True)`, and a decode step of two sequences (over a copy of the
    decoder's pages) the `d_logits` of `decode_step_batched`, bit for bit."""
    from vita_b200.model.mixtral import MixtralDecoder
    from vita_b200.vllm_adapter import MixtralForConditionalGeneration, TokenBatch
    cfg = VitaConfig.tiny()
    c, dev = cfg.llm, torch.device("cuda")
    packed = W.pack(W.synthetic_state(cfg, 0), cfg, dev)
    m = MixtralForConditionalGeneration(cfg, device=dev, packed=packed)
    llm = MixtralDecoder(c, packed["llm"], dev, max_batch=2, max_seq_len=128, max_new_tokens=8)
    cache, bs = llm.cache, llm.cache.page_size
    g = torch.Generator().manual_seed(6)
    prompts = [torch.randint(3, 1900, (n,), generator=g).tolist() for n in (37, 20)]
    embeds = lambda ids: packed["llm"]["embed"][torch.tensor(ids, device=dev)]

    # one whole prompt, all rows scored
    p = prompts[0]
    S = len(p)
    want = llm.prefill(embeds(p), slot=0, all_logits=True)
    kv = [torch.zeros(2, k.shape[0] // bs, bs, c.num_key_value_heads, c.head_dim, dtype=k.dtype, device=dev)
          for k in cache.k]
    meta = TokenBatch(cache.slot_map[0, :S].contiguous(), cache.block_table[:1], [0, S], [S])
    got = m.compute_logits(m.forward(torch.tensor(p), torch.arange(S), kv, meta))
    assert torch.equal(got, want), f"{int((got != want).any(-1).sum())} of {S} prompt logits rows differ"

    # one decode step of two sequences
    llm.reset()
    for b, p in enumerate(prompts):
        llm.prefill(embeds(p), slot=b)
    kv = [torch.stack([k, v]).view(2, -1, bs, c.num_key_value_heads, c.head_dim) for k, v in zip(cache.k, cache.v)]
    toks = (0xFFFFFFFF - (llm.best[:2] & 0xFFFFFFFF)).tolist()
    lens = [len(p) for p in prompts]
    meta = TokenBatch(torch.stack([cache.slot_map[b, n] for b, n in enumerate(lens)]), cache.block_table[:2], [0, 1, 2],
                      [n + 1 for n in lens])
    got = m.compute_logits(m.forward(torch.tensor(toks), torch.tensor(lens), kv, meta))
    llm.decode_step_batched(2, use_graph=False)
    assert torch.equal(got, llm.d_logits[:2]), "decode-step logits differ"
