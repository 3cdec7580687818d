"""CPU: oracle/blip2_ref.py against transformers' Blip2ForConditionalGeneration in float64 with the same random weights, at a reduced
configuration that keeps every quirk of blip2-opt-2.7b (vision head_dim 88, OPT head_dim 80, Q-Former layers with and without
cross-attention, 32 queries, a vocab that is not a multiple of 64), and the full configuration's state_dict naming."""
import pytest
import torch

from oracle import blip2_ref

transformers = pytest.importorskip("transformers")


def _small_cfg():
    return dict(image_size=56, patch=14, vision_width=176, vision_layers=2, vision_heads=2, vision_mlp=256,
                qformer_width=128, qformer_layers=3, qformer_heads=2, qformer_ffn=256, cross_attention_frequency=2,
                num_query_tokens=32, opt_width=160, opt_layers=2, opt_heads=2, opt_ffn=320, vocab=1000, max_positions=128,
                image_token_index=998, bos_token_id=2, eos_token_id=50)


def _hf_config(c):
    from transformers import Blip2Config, Blip2QFormerConfig, Blip2VisionConfig, OPTConfig
    v = Blip2VisionConfig(hidden_size=c["vision_width"], num_hidden_layers=c["vision_layers"], num_attention_heads=c["vision_heads"],
                          intermediate_size=c["vision_mlp"], image_size=c["image_size"], patch_size=c["patch"])
    q = Blip2QFormerConfig(hidden_size=c["qformer_width"], num_hidden_layers=c["qformer_layers"], num_attention_heads=c["qformer_heads"],
                           intermediate_size=c["qformer_ffn"], cross_attention_frequency=c["cross_attention_frequency"],
                           encoder_hidden_size=c["vision_width"])
    t = OPTConfig(hidden_size=c["opt_width"], num_hidden_layers=c["opt_layers"], num_attention_heads=c["opt_heads"], ffn_dim=c["opt_ffn"],
                  vocab_size=c["vocab"], max_position_embeddings=c["max_positions"], word_embed_proj_dim=c["opt_width"],
                  bos_token_id=c["bos_token_id"], eos_token_id=c["eos_token_id"], pad_token_id=1)
    return Blip2Config(vision_config=v.to_dict(), qformer_config=q.to_dict(), text_config=t.to_dict(),
                       num_query_tokens=c["num_query_tokens"], image_token_index=c["image_token_index"])


@pytest.fixture(scope="module")
def pair():
    from transformers import Blip2ForConditionalGeneration
    cfg = _small_cfg()
    assert cfg["vision_width"] // cfg["vision_heads"] == 88 and cfg["opt_width"] // cfg["opt_heads"] == 80 and cfg["vocab"] % 64
    p = blip2_ref.default_init(cfg, seed=1, dtype=torch.float64)
    model = Blip2ForConditionalGeneration(_hf_config(cfg)).double().eval()
    sd = dict(p)
    sd["language_model.lm_head.weight"] = p["language_model.model.decoder.embed_tokens.weight"]
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not missing and not unexpected
    px = torch.randn(1, 3, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(2), dtype=torch.float64)
    return cfg, p, model, px


def _hf_generate(model, px, eos, n=20):
    with torch.no_grad():
        out = model.generate(pixel_values=px, max_new_tokens=n, do_sample=False, num_beams=1, eos_token_id=eos,
                             output_scores=True, return_dict_in_generate=True)
    return out.sequences[0].tolist(), torch.stack([s[0] for s in out.scores])


def test_taps_logits_and_ids_match_transformers(pair):
    cfg, p, model, px = pair
    with torch.no_grad():
        img = model.vision_model(px).last_hidden_state[0]
        qo = model.qformer(query_embeds=model.query_tokens, encoder_hidden_states=img[None]).last_hidden_state[0]
        lm = model.language_projection(qo)
    ref = blip2_ref.generate(p, cfg, px, 20, eos_token_id=-1)
    for name, a, b in (("image_embeds", ref["image_embeds"], img), ("query_output", ref["query_output"], qo),
                       ("language_model_inputs", ref["language_model_inputs"], lm)):
        assert a.shape == b.shape, name
        assert float((a - b).abs().max()) < 1e-12 * max(1.0, float(b.abs().max())), name
    ids, _ = _hf_generate(model, px, eos=-1)
    assert len(ids) == 33 + 20 and ref["ids"] == ids
    # generate() hands back fp32 scores: the float64 step logits come from one forward over the decoded ids (row 32 + s predicts step s)
    with torch.no_grad():
        logits = model(pixel_values=px, input_ids=torch.tensor([ids[:-1]])).logits[0, 32:]
    assert logits.dtype == torch.float64 and logits.shape == ref["logits"].shape
    assert float((ref["logits"] - logits).abs().max()) < 1e-12 * max(1.0, float(logits.abs().max()))


def test_early_stop_at_eos(pair):
    cfg, p, model, px = pair
    full = blip2_ref.generate(p, cfg, px, 20, eos_token_id=-1)["ids"][33:]
    k = next((k for k in range(2, 20) if full[k] not in full[:k]), None)
    if k is None:
        pytest.skip("the seeded decode repeats one token throughout")
    ids, _ = _hf_generate(model, px, eos=full[k])
    ref = blip2_ref.generate(p, cfg, px, 20, eos_token_id=full[k])["ids"]
    assert ref == ids and len(ids) == 33 + k + 1 and ids[-1] == full[k]


def test_full_config_state_dict_naming():
    from transformers import Blip2ForConditionalGeneration
    cfg = blip2_ref.blip2_opt_27b_cfg()
    with torch.device("meta"):
        model = Blip2ForConditionalGeneration(_hf_config(cfg))
    sd = model.state_dict()
    assert len(sd) == 1248
    want = {k: tuple(v.shape) for k, v in sd.items() if k != "language_model.lm_head.weight"}
    got = blip2_ref.param_shapes(cfg)
    assert list(got) == list(want) and got == want
    assert sum(torch.Size(s).numel() for s in got.values()) == 3744679936
    assert tuple(sd["language_model.lm_head.weight"].shape) == got["language_model.model.decoder.embed_tokens.weight"]
