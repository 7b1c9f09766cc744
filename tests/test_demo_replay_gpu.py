"""Replays the call sequence of the reference demo (video_audio_demo.py:163-276) against the drop-in
surface on a synthetic tiny model: CUDA `input_ids`, fp16 `audios`, `output_scores=True, return_dict_in_generate=True,
max_new_tokens=..., stopping_criteria=[KeywordsStoppingCriteria(...)]` and the `input_ids != output_ids[:, :L]` check.

The tokenizer and the stopping-criteria class are the reference's own host-side Python (out of scope for the kernel
tier); the stand-ins below restate their behaviour (vita/util/mm_utils.py:121-155) so that the
test exercises exactly what `generate()` has to support."""
import pytest
import torch

from vita_b200.config import IMAGE_TOKEN_INDEX, AUDIO_TOKEN_INDEX

pytestmark = pytest.mark.gpu


class ToyTokenizer:
    """id <-> one printable glyph; enough of the HF interface for KeywordsStoppingCriteria."""
    bos_token_id = 1

    class _Enc:
        def __init__(self, ids):
            self.input_ids = ids

    @staticmethod
    def glyph(i: int) -> str:
        return chr(0x4E00 + int(i))

    def __call__(self, text):
        return self._Enc([self.bos_token_id] + [ord(c) - 0x4E00 for c in text])

    def batch_decode(self, ids, skip_special_tokens=False):
        return ["".join(self.glyph(t) for t in row.tolist() if t >= 0) for row in ids]


class KeywordsStoppingCriteria:
    """vita/util/mm_utils.py:121-155, line for line in behaviour (counts its calls for the O(n) check)."""

    def __init__(self, keywords, tokenizer, input_ids):
        self.keywords = keywords
        self.keyword_ids = []
        self.max_keyword_len = 0
        for keyword in keywords:
            cur = tokenizer(keyword).input_ids
            if len(cur) > 1 and cur[0] == tokenizer.bos_token_id:
                cur = cur[1:]
            self.max_keyword_len = max(self.max_keyword_len, len(cur))
            self.keyword_ids.append(torch.tensor(cur))
        self.tokenizer = tokenizer
        self.start_len = input_ids.shape[1]
        self.calls = 0

    def call_for_batch(self, output_ids, scores, **kwargs):
        offset = min(output_ids.shape[1] - self.start_len, self.max_keyword_len)
        self.keyword_ids = [k.to(output_ids.device) for k in self.keyword_ids]
        for k in self.keyword_ids:
            if torch.equal(output_ids[0, -k.shape[0]:], k):
                return True
        outputs = self.tokenizer.batch_decode(output_ids[:, -offset:], skip_special_tokens=True)[0]
        return any(k in outputs for k in self.keywords)

    def __call__(self, output_ids, scores, **kwargs):
        self.calls += 1
        return all(self.call_for_batch(output_ids[i].unsqueeze(0), scores) for i in range(output_ids.shape[0]))


@pytest.fixture(scope="module")
def loaded():
    from vita_b200.model.builder import load_pretrained_model
    return load_pretrained_model("synthetic:tiny", None, "vita-tiny", "mixtral-8x7b", max_new_tokens=96)


def _demo_inputs(model, with_audio: bool):
    """video_audio_demo.py:169-247 with an in-memory image / fbank instead of files."""
    cfg = model.config
    vision_tower = model.get_vision_tower()
    if not vision_tower.is_loaded:
        vision_tower.load_model()
    audio_encoder = model.get_audio_encoder()
    audio_encoder.to(dtype=torch.float16)
    model.eval()
    g = torch.Generator().manual_seed(3)
    audio = torch.randn(300, 80, generator=g) if with_audio else torch.zeros(400, 80)       # :180-195
    audios = {"audios": audio.unsqueeze(0).half().cuda(),
              "lengths": torch.tensor(audio.shape[0]).unsqueeze(0).half().cuda()}
    px = cfg.vision.image_size
    image_tensor = torch.randn(1, 3, px, px, generator=g).to(dtype=model.dtype, device="cuda")
    ids = [1, IMAGE_TOKEN_INDEX] + torch.randint(3, cfg.llm.vocab_size, (9,), generator=g).tolist()
    if with_audio:
        ids.append(AUDIO_TOKEN_INDEX)
    ids += [5, 6]
    input_ids = torch.tensor(ids, dtype=torch.long).unsqueeze(0).cuda()                      # :235-246
    return input_ids, image_tensor, audios


@pytest.mark.parametrize("with_audio", [True, False])
def test_demo_call_sequence(loaded, with_audio):
    tokenizer, model, image_processor, context_len = loaded
    tok = ToyTokenizer()
    model.resize_token_embeddings(model.config.llm.vocab_size)                               # :167
    input_ids, image_tensor, audios = _demo_inputs(model, with_audio)
    kwargs = dict(images=image_tensor, audios=audios, do_sample=False, temperature=0.01, top_p=None, num_beams=1,
                  output_scores=True, return_dict_in_generate=True, use_cache=True)

    # free run first to learn what the model says; the stop keyword is then the glyph of its 20th new token
    with torch.inference_mode():
        free = model.generate(input_ids, max_new_tokens=64, **kwargs)
    L = input_ids.shape[1]
    assert free.sequences.device == input_ids.device and free.sequences.dtype == torch.long
    assert free.sequences.shape == (1, L + 64) and len(free.scores) == 64
    new = free.sequences[0, L:].tolist()
    free_rows = [s.clone() for s in free.scores]       # `scores` are views of a log the next call overwrites
    stop_at = [i for i in range(64) if new[i] not in new[:i]][-1]           # first occurrence ends the reply
    stop_str = tok.glyph(new[stop_at])

    stopping_criteria = KeywordsStoppingCriteria([stop_str], tok, input_ids)                # :248-250
    with torch.inference_mode():                                                             # :256-270
        output_ids = model.generate(input_ids, max_new_tokens=96, stopping_criteria=[stopping_criteria], **kwargs)
    scores = output_ids.scores
    output_ids = output_ids.sequences                                                        # :272
    input_token_len = input_ids.shape[1]
    n_diff_input_output = (input_ids != output_ids[:, :input_token_len]).sum().item()        # :274 (same device!)
    assert n_diff_input_output == 0
    outputs = tok.batch_decode(output_ids[:, input_token_len:], skip_special_tokens=False)[0].strip()
    assert outputs.endswith(stop_str)                                                        # :279-280
    assert output_ids.shape[1] == L + stop_at + 1
    assert output_ids[0, L:].tolist() == new[: stop_at + 1]
    # each new token was shown to the criteria exactly once (tokens past the stop inside a sync window are not)
    assert stopping_criteria.calls == stop_at + 1
    # scores: one [1, V] row per new token, equal to the free run's rows (same greedy trajectory), and the arg-max of
    # row i is token i (logits stay in the activation dtype, arg-max on them: vita_mixtral.py:172-173)
    assert len(scores) == stop_at + 1 and scores[0].shape == (1, model.config.llm.vocab_size)
    for i in sorted({0, min(1, stop_at), stop_at}):
        assert torch.equal(scores[i], free_rows[i])
        assert int(scores[i].float().cpu().argmax(-1)) == new[i]
    # the demo's kwargs keep the captured CUDA graph (logits variant), they do not fall back to eager launches
    assert (1, True) in model.llm._graphs


def test_scores_graph_equals_eager(loaded):
    _, model, _, _ = loaded
    input_ids, image_tensor, audios = _demo_inputs(model, True)
    kw = dict(images=image_tensor, audios=audios, output_scores=True, max_new_tokens=12)
    a = model.generate(input_ids, use_graph=True, sync_every=5, **kw)
    rows_a = torch.cat([s.clone() for s in a.scores])
    b = model.generate(input_ids, use_graph=False, **kw)
    assert a.sequences.tolist() == b.sequences.tolist()
    assert torch.equal(rows_a, torch.cat(list(b.scores)))


def test_generate_refuses_what_does_not_fit(loaded):
    _, model, _, _ = loaded
    input_ids, image_tensor, audios = _demo_inputs(model, True)
    with pytest.raises(ValueError, match="max_new_tokens"):
        model.generate(input_ids, images=image_tensor, audios=audios, max_new_tokens=97)
    long_ids = torch.randint(3, 100, (1, model.llm.cache.max_seq_len + 1)).cuda()
    with pytest.raises(ValueError, match="KV capacity"):
        model.generate(long_ids, max_new_tokens=1)


def test_prepare_inputs_for_generation_bookkeeping(loaded):
    """vita_mixtral.py:291-382: crop to the unseen suffix, positions from the mask, images / audios re-attached."""
    _, model, _, _ = loaded
    ids = torch.randint(3, 100, (1, 10)).cuda()
    first = model.prepare_inputs_for_generation(ids, past_key_values=None, attention_mask=torch.ones(1, 10).cuda(),
                                                images="IMG", audios="AUD", use_cache=True)
    assert torch.equal(first["input_ids"], ids) and first["images"] == "IMG" and first["audios"] == "AUD"
    assert first["position_ids"].tolist() == [list(range(10))] and first["use_cache"] is True
    out = model(input_ids=ids)                                       # prefill: the paged cache now holds 10 tokens
    ids11 = torch.cat([ids, torch.tensor([[7]]).cuda()], dim=1)
    nxt = model.prepare_inputs_for_generation(ids11, past_key_values=out.past_key_values,
                                              attention_mask=torch.ones(1, 11).cuda())
    assert nxt["input_ids"].tolist() == [[7]] and nxt["position_ids"].tolist() == [[10]]
    assert "images" not in nxt and nxt["past_key_values"] is out.past_key_values
    step = model(**{k: v for k, v in nxt.items() if k in ("input_ids", "past_key_values")})
    assert step.logits.shape == (1, 1, model.config.llm.vocab_size)
