"""GPU parity of the BLIP-2 captioner (csrc/blip2_engine.cu behind nerf/blip2.py) at the full blip2-opt-2.7b configuration with seeded
weights, against the fp32 oracle (oracle/blip2_ref.py) on the same GPU; plus the weight-streaming GEMM on its own, checkpoint loading
through a save_pretrained directory, input checks and main.py:163-172 end to end (`caption`).

Tolerance, as for the other engines: the engine stores fp16 between kernels, so the oracle also runs with every stored tensor rounded to
fp16 (e16), and the engine's relative L2 error must stay within max(2.5 x that fp16-storage error, 1e-3).  Observed values are printed.
The greedy ids are compared up to the first step whose top-1 / top-2 logit margin (oracle) is under 4 x the measured logit error; the
teacher-forced logits are the strong check, since seeded-weight decodes tend to repeat one token."""
import importlib
import json

import pytest
import torch

from oracle import blip2_ref

pytestmark = pytest.mark.gpu
N_NEW = 20


def _mods():
    return importlib.import_module("make-it-3d_b200.nerf.blip2"), importlib.import_module("make-it-3d_b200._lib")


def _rel(a, b):
    a, b = a.detach().double().flatten().cpu(), b.detach().double().flatten().cpu()
    return float((a - b).norm() / b.norm())


def _pixels(seed, S=224):
    return torch.randn(1, 3, S, S, generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.fixture(scope="module")
def setup():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    b2, _ = _mods()
    cfg = blip2_ref.blip2_opt_27b_cfg()
    p = blip2_ref.default_init(cfg, seed=0, device="cuda")
    model = b2.Blip2ForConditionalGeneration(cfg=cfg, state_dict=p)
    px = _pixels(1)
    with torch.no_grad():
        ref = blip2_ref.generate(p, cfg, px, N_NEW, eos_token_id=-1)
        forced = ref["ids"][33:]
        ref16 = blip2_ref.generate(p, cfg, px, N_NEW, eos_token_id=-1, e16=True, forced_ids=forced)
    return b2, cfg, p, model, px, ref, ref16


def test_registry_is_the_transformers_naming(setup):
    model, cfg = setup[3], setup[1]
    shapes = blip2_ref.param_shapes(cfg)
    assert model.names == list(shapes) and model.shapes == [tuple(s) for s in shapes.values()]
    assert len(model.names) + 1 == 1248          # + the tied language_model.lm_head.weight
    print(f"workspace {model.workspace_bytes / 2 ** 20:.0f} MiB")


def test_taps_match_oracle(setup):
    _, cfg, _, model, px, ref, ref16 = setup
    lm = model.encode(px)
    taps = model.taps()
    torch.cuda.synchronize()
    assert torch.equal(lm, taps["language_model_inputs"])
    for name in ("image_embeds", "query_output", "language_model_inputs"):
        e, e16 = _rel(taps[name], ref[name]), _rel(ref16[name], ref[name])
        print(f"{name:22s} engine vs fp32 {e:.3e}   fp16-storage oracle vs fp32 {e16:.3e}")
        assert e <= max(2.5 * e16, 1e-3), (name, e, e16)


def test_teacher_forced_logits_match_oracle(setup):
    _, cfg, _, model, px, ref, ref16 = setup
    forced = ref["ids"][33:]
    ids, logits = model.generate(pixel_values=px, max_new_tokens=N_NEW, eos_token_id=-1, forced_ids=forced, return_logits=True)
    assert ids[0, 33:].tolist() == forced
    worst = 0.0
    for s in range(N_NEW):
        e, e16 = _rel(logits[s], ref["logits"][s]), _rel(ref16["logits"][s], ref["logits"][s])
        worst = max(worst, e / max(2.5 * e16, 1e-3))
        assert e <= max(2.5 * e16, 1e-3), (s, e, e16)
    print(f"teacher-forced logits: worst step at {worst:.2f} of its bound; max abs err {float((logits.cpu() - ref['logits'].cpu()).abs().max()):.3e}")


def test_greedy_ids_match_oracle_up_to_margin(setup):
    _, cfg, _, model, px, ref, _ = setup
    out = model.generate(pixel_values=px, max_new_tokens=N_NEW, eos_token_id=-1)
    _, logits = model.generate(pixel_values=px, max_new_tokens=N_NEW, eos_token_id=-1, forced_ids=ref["ids"][33:], return_logits=True)
    assert out.shape == (1, 33 + N_NEW) and out.dtype == torch.int64
    assert out[0, :33].tolist() == ref["ids"][:33]
    err = float((logits.cpu() - ref["logits"].cpu()).abs().max())
    top2 = ref["logits"].topk(2, dim=-1).values.cpu()
    margins = (top2[:, 0] - top2[:, 1]).tolist()
    checked = next((s for s, m in enumerate(margins) if m < 4 * err), N_NEW)
    print(f"ids checked for {checked} of {N_NEW} steps (logit max-abs error {err:.3e}, margins {[round(m, 3) for m in margins]})")
    print(f"engine ids {out[0, 33:].tolist()}\noracle ids {ref['ids'][33:]}")
    assert out[0, 33:33 + checked].tolist() == ref["ids"][33:33 + checked]
    assert checked >= 10


def test_early_stop_at_eos(setup):
    _, cfg, _, model, px, ref, _ = setup
    gen = ref["ids"][33:]
    k = next((k for k in range(2, N_NEW) if gen[k] not in gen[:k]), None)
    if k is None:
        pytest.skip("the seeded decode repeats earlier tokens throughout")
    out = model.generate(pixel_values=px, max_new_tokens=N_NEW, eos_token_id=gen[k])
    assert out.shape == (1, 33 + k + 1) and int(out[0, -1]) == gen[k]


def test_early_stop_at_eos_reduced_config():
    """the full-size seeded decode tends to repeat one token, so the early stop is also checked where the seeds can be searched cheaply:
    the first seed whose oracle decode has a fresh token at some step k >= 2"""
    b2, _ = _mods()
    cfg = _small_cfg()
    px = _pixels(6, 56)
    for seed in range(40):
        p = blip2_ref.default_init(cfg, seed=seed, device="cuda")
        with torch.no_grad():
            gen = blip2_ref.generate(p, cfg, px, N_NEW, eos_token_id=-1)["ids"][33:]
        k = next((k for k in range(2, N_NEW) if gen[k] not in gen[:k]), None)
        if k is not None:
            break
    assert k is not None, "no seed in 0..39 gives a decode with a fresh token"
    model = b2.Blip2ForConditionalGeneration(cfg=cfg, state_dict=p)
    full = model.generate(pixel_values=px, max_new_tokens=N_NEW, eos_token_id=-1)[0, 33:].tolist()
    assert full[:k + 1] == gen[:k + 1], (full, gen)
    out = model.generate(pixel_values=px, max_new_tokens=N_NEW, eos_token_id=gen[k])
    print(f"seed {seed}: eos = token {gen[k]} first generated at step {k}")
    assert out.shape == (1, 33 + k + 1) and int(out[0, -1]) == gen[k]


def test_bit_identical_across_calls_and_with_engine_graph_replay_off(setup):
    b2, _, _, model, px, ref, _ = setup
    _, L = _mods()
    runs = [model.generate(pixel_values=px, max_new_tokens=N_NEW, eos_token_id=-1, return_logits=True) for _ in range(3)]
    assert model.graph_replays() >= 1
    L.check(L.lib().mi3d_engine_set_graph_replay(model.h, 0), "set_graph_replay")
    try:
        runs.append(model.generate(pixel_values=px, max_new_tokens=N_NEW, eos_token_id=-1, return_logits=True))
    finally:
        L.check(L.lib().mi3d_engine_set_graph_replay(model.h, 1), "set_graph_replay")
    for ids, lg in runs[1:]:
        assert torch.equal(ids, runs[0][0]) and torch.equal(lg, runs[0][1])


def test_stream_gemm_matches_fp32_and_is_deterministic():
    _, L = _mods()
    import ctypes as C
    lib = L.lib()
    lib.mi3d_stream_gemm_workspace_bytes.restype = C.c_size_t
    g = torch.Generator(device="cuda").manual_seed(5)
    for M, N, K, relu in ((64, 10240, 2560, 1), (64, 2560, 10240, 0), (1, 50272, 2560, 0), (33, 7680, 2560, 0), (5, 200, 96, 1)):
        x = torch.randn(M, K, generator=g, device="cuda").half()
        w = (torch.randn(N, K, generator=g, device="cuda") * K ** -0.5).half()
        b = torch.randn(N, generator=g, device="cuda")
        res = torch.randn(M, N, generator=g, device="cuda").half()
        ws = torch.empty(lib.mi3d_stream_gemm_workspace_bytes(M, N, K), dtype=torch.uint8, device="cuda")
        ys = []
        for _ in range(2):
            y = torch.empty(M, N, dtype=torch.float16, device="cuda")
            L.check(lib.mi3d_stream_gemm_f16(L.ptr(x), L.ptr(w), L.ptr(b), L.ptr(res), relu, L.ptr(y), M, N, K, L.ptr(ws),
                                             C.c_size_t(ws.numel()), L.stream()), "stream_gemm")
            ys.append(y)
        ref = x.float() @ w.float().t() + b + res.float()
        ref = ref.relu() if relu else ref
        assert torch.equal(ys[0], ys[1])
        e = _rel(ys[0], ref)
        assert e < 2e-3, (M, N, K, e)


def _small_cfg():
    return dict(image_size=56, patch=14, vision_width=704, vision_layers=2, vision_heads=8, vision_mlp=1024,
                qformer_width=128, qformer_layers=3, qformer_heads=2, qformer_ffn=256, cross_attention_frequency=2,
                num_query_tokens=32, opt_width=320, opt_layers=2, opt_heads=4, opt_ffn=640, vocab=1000, max_positions=128,
                image_token_index=998, bos_token_id=2, eos_token_id=50)


def test_from_pretrained_directory(tmp_path):
    b2, L = _mods()
    transformers = pytest.importorskip("transformers")
    import test_blip2_oracle_cpu as cpu_test
    cfg = _small_cfg()
    p = blip2_ref.default_init(cfg, seed=4)
    hf = transformers.Blip2ForConditionalGeneration(cpu_test._hf_config(cfg))
    sd = dict(p)
    sd["language_model.lm_head.weight"] = p["language_model.model.decoder.embed_tokens.weight"]
    hf.load_state_dict(sd)
    hf.save_pretrained(str(tmp_path))
    model = b2.Blip2ForConditionalGeneration.from_pretrained(str(tmp_path), torch_dtype=torch.float16).to("cuda").eval()
    assert model.cfg == cfg
    px = _pixels(2, 56)
    pc = {k: v.cuda() for k, v in p.items()}
    with torch.no_grad():
        ref = blip2_ref.generate(pc, cfg, px, 8, eos_token_id=-1)
        ref16 = blip2_ref.encode(pc, cfg, px, e16=True)
    lm = model.encode(px)
    e, e16 = _rel(lm, ref["language_model_inputs"]), _rel(ref16[2], ref["language_model_inputs"])
    assert e <= max(2.5 * e16, 1e-3), (e, e16)
    out = model.generate(pixel_values=px, max_new_tokens=8, eos_token_id=-1)
    assert out.shape == (1, 41) and out[0, :33].tolist() == ref["ids"][:33]
    cfgjson = json.load(open(tmp_path / "config.json"))
    cfgjson["text_config"]["activation_function"] = "gelu"
    json.dump(cfgjson, open(tmp_path / "config.json", "w"))
    with pytest.raises(L.Mi3dError):
        b2.Blip2ForConditionalGeneration.from_pretrained(str(tmp_path))


def test_state_dict_mismatches_and_bad_inputs_raise():
    b2, L = _mods()
    cfg = _small_cfg()
    p = blip2_ref.default_init(cfg, seed=4)
    model = b2.Blip2ForConditionalGeneration(cfg=cfg, state_dict=p)
    tied = dict(p, **{"language_model.lm_head.weight": p["language_model.model.decoder.embed_tokens.weight"].clone()})
    model.load_state_dict(tied)
    bad = dict(tied); bad["language_model.lm_head.weight"] = bad["language_model.lm_head.weight"] + 1
    for sd in (bad, {k: v for k, v in p.items() if k != "query_tokens"}, dict(p, extra=torch.zeros(1)),
               dict(p, query_tokens=torch.zeros(1, 31, 128))):
        with pytest.raises(L.Mi3dError):
            model.load_state_dict(sd)
    px = _pixels(3, 56)
    for kw in (dict(pixel_values=px.cpu()), dict(pixel_values=px.repeat(2, 1, 1, 1)), dict(pixel_values=_pixels(3, 64)),
               dict(pixel_values=px, interpolate_pos_encoding=True), dict(pixel_values=px, do_sample=True),
               dict(pixel_values=px, num_beams=3), dict(pixel_values=px, input_ids=torch.ones(1, 4, dtype=torch.long, device="cuda")),
               dict(pixel_values=px, max_new_tokens=40), dict(pixel_values=px, temperature=0.7)):
        with pytest.raises(L.Mi3dError):
            model.generate(**kw)
    with pytest.raises(L.Mi3dError):
        b2.Blip2ForConditionalGeneration(cfg=dict(cfg, vision_heads=7), state_dict=p)
    assert model.generate(pixel_values=px, max_new_tokens=3, do_sample=False, num_beams=1).shape[1] <= 36


def test_caption_applies_main_py_replacements():
    b2, _ = _mods()
    cfg = _small_cfg()
    model = b2.Blip2ForConditionalGeneration(cfg=cfg)
    seen = {}

    class Stub:
        def __call__(self, image, return_tensors=None):
            class B(dict):
                def to(self, device, dtype):
                    return B({k: v.to(device, dtype) for k, v in self.items()})
            return B(pixel_values=torch.zeros(1, 3, 56, 56))

        def batch_decode(self, out, skip_special_tokens=False):
            seen["out"] = out
            return ["  there is a close up of a cat on a black background  "]

    assert b2.caption(model, Stub(), object()) == "a photo of a cat on a ground"
    assert seen["out"].dtype == torch.int64 and seen["out"].shape[0] == 1 and seen["out"].shape[1] >= 34
