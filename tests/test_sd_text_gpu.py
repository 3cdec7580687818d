"""GPU parity of the SD-2 text encoder (csrc/sd_text_engine.cu behind nerf/sd_text.py and StableDiffusion.get_text_embeds) against the
fp32 oracle (oracle/sd_text_ref.py), at the full SD-2 configuration and a tiny one, with seeded random weights.

Tolerance, as in test_clip_gpu.py: the engine keeps activations in fp16 between kernels, so the oracle is run a second time with every
leaf module's output rounded to fp16 (forward hooks) and the engine's relative error must stay within max(2.5 x that fp16-storage
error, 1e-3).  Observed values are printed."""
import hashlib
import importlib

import pytest
import torch

from oracle import sd_text_ref

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.detach().double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / b.norm())


class _Fp16Storage:
    """round every leaf module's output to fp16 and back while active"""

    def __init__(self, model):
        self.model = model

    def __enter__(self):
        self.hs = [m.register_forward_hook(lambda mod, inp, out: out.half().float() if torch.is_tensor(out) else out)
                   for m in self.model.modules() if len(list(m.children())) == 0]

    def __exit__(self, *a):
        for h in self.hs:
            h.remove()


def _check(name, got, ref32, ref16):
    e, e16 = _rel(got, ref32), _rel(ref16, ref32)
    print(f"{name:44s} engine vs fp32 {e:.3e}   fp16-storage oracle vs fp32 {e16:.3e}")
    assert e <= max(2.5 * e16, 1e-3), (name, e, e16)


def _mods():
    return (importlib.import_module("make-it-3d_b200.nerf.sd_text"), importlib.import_module("make-it-3d_b200.nerf.sd"),
            importlib.import_module("make-it-3d_b200._lib"))


def _oracle(cfg, seed):
    torch.manual_seed(0)
    ref = sd_text_ref.default_init(sd_text_ref.TextEncoderRef(cfg), seed=seed).eval()
    for p in ref.parameters():
        p.requires_grad_(False)
    return ref


@pytest.fixture(scope="module")
def full():
    torch.set_num_threads(min(32, torch.get_num_threads()))
    ref = _oracle(sd_text_ref.sd2_text_config(), seed=5)
    st, _, _ = _mods()
    return ref, st.TextEncoder("cuda", cfg=ref.cfg, state_dict=ref.state_dict())


@pytest.fixture(scope="module")
def tiny():
    ref = _oracle(sd_text_ref.tiny_config(), seed=6)
    st, _, _ = _mods()
    return ref, st.TextEncoder("cuda", cfg=ref.cfg, state_dict=ref.state_dict())


def _ids():
    # EOS at 1 (an empty negative prompt), 10, and 76 (a prompt truncated to 77 tokens); SD-2's tokenizer pads with id 0,
    # openai's CLIP-L tokenizer with the EOS id: both are run
    return torch.cat([sd_text_ref.make_ids((2, 11, 90), pad=0, seed=7), sd_text_ref.make_ids((2, 11, 90), pad=49407, seed=7)])


def _parity(name, ref, enc):
    ids = _ids()
    with torch.no_grad():
        f32 = ref(ids)[0]
        with _Fp16Storage(ref):
            f16 = ref(ids)[0]
    got = []
    for i in range(0, ids.shape[0], 3):                      # one B = 2 call and one B = 1 call per padding
        got += [enc(ids[i:i + 2].cuda())[0], enc(ids[i + 2:i + 3].cuda())[0]]
    got = torch.cat(got).cpu()
    assert got.shape == (6, 77, ref.cfg["width"]) and torch.isfinite(got).all()
    _check(f"{name} all 6 x 77 rows", got, f32, f16)
    for i, n in enumerate((2, 11, 77) * 2):
        _check(f"{name} prompt {i} all rows", got[i], f32[i], f16[i])
        _check(f"{name} prompt {i} rows 0..{n - 1}", got[i, :n], f32[i, :n], f16[i, :n])


def test_full_size_matches_the_fp32_oracle(full):
    ref, enc = full
    st, _, _ = _mods()
    assert enc.names == list(ref.state_dict()) and len(enc.names) == 372
    assert [tuple(s) for s in enc.shapes] == [tuple(t.shape) for t in ref.state_dict().values()]
    print(f"SD-2 text encoder workspace: {enc.workspace.numel() / 2 ** 20:.1f} MiB")
    _parity("SD-2", ref, enc)


def test_tiny_config_matches_the_oracle_with_and_without_graph_replay(tiny):
    ref, enc = tiny
    st, _, _ = _mods()
    plain = st.TextEncoder("cuda", cfg=ref.cfg, state_dict=ref.state_dict(), graph_replay=False)
    assert plain.stream is None and enc.stream is not None
    for _ in range(3):                                       # repeated calls replay the B = 1 and B = 2 lists as CUDA graphs
        _parity("tiny (graph replay)", ref, enc)
    assert enc.graph_replays() == 2
    _parity("tiny (plain launches)", ref, plain)
    assert plain.graph_replays() == 0


@pytest.mark.parametrize("which", ["tiny", "full"])
def test_results_are_bit_identical_across_calls_graph_replay_and_batching(which, request):
    ref, enc = request.getfixturevalue(which)
    st, _, _ = _mods()
    plain = st.TextEncoder("cuda", cfg=ref.cfg, state_dict=ref.state_dict(), graph_replay=False)
    ids = sd_text_ref.make_ids((2, 23), pad=0, seed=9).cuda()
    want = plain(ids)[0].clone()
    assert torch.equal(plain(ids)[0], want)                                     # run to run
    for call in range(4):
        assert torch.equal(enc(ids)[0], want), call                             # graph replay from the third call on
    assert enc.graph_replays() >= 1
    one = torch.cat([enc(ids[i:i + 1])[0] for i in range(2)])
    assert torch.equal(one, want)                                               # one B = 2 call == two B = 1 calls


class _StubTokenizer:
    """CLIPTokenizer.__call__'s contract with fixed ids per string; records its keyword arguments"""

    def __init__(self, table):
        self.table, self.calls = table, []

    def __call__(self, text, padding=None, max_length=None, truncation=False, return_tensors=None):
        self.calls.append(dict(text=list(text), padding=padding, max_length=max_length, truncation=truncation, return_tensors=return_tensors))
        return type("Enc", (), {"input_ids": torch.stack([self.table[t] for t in text])})()


def _tiny_guidance(sdm, **kw):
    from oracle import sd_ref
    torch.manual_seed(0)
    ucfg, vcfg = sd_ref.tiny_unet_config(), sd_ref.tiny_vae_config()
    unet, vae = sd_ref.UNet2DConditionModel(ucfg).eval(), sd_ref.AutoencoderKLEncoder(vcfg).eval()
    return sdm.StableDiffusion("cuda", unet_cfg=dict(ucfg, latent_hw=32), vae_cfg=dict(vcfg, image_hw=256), unet_state=unet.state_dict(),
                               vae_state=vae.state_dict(), **kw)


def test_get_text_embeds_runs_the_encoder_and_drives_a_train_step(tiny):
    ref, enc = tiny
    st, sdm, L = _mods()
    ids = sd_text_ref.make_ids((2, 14), pad=0, seed=11)
    tok = _StubTokenizer({"": ids[0], "a hamburger": ids[1]})
    guide = _tiny_guidance(sdm, tokenizer=tok)
    sd = dict(ref.state_dict(), **{"text_model.embeddings.position_ids": torch.arange(77)[None]})   # older transformers keep it
    guide.load_diffusers_state_dict(text_encoder_state=sd)
    emb = guide.get_text_embeds(["a hamburger"], [""])
    assert emb.shape == (2, 77, ref.cfg["width"]) and emb.dtype == torch.float32 and emb.is_cuda
    assert torch.equal(emb, enc(ids.cuda())[0])                                  # [uncond, cond] in one B = 2 call
    assert [c["truncation"] for c in tok.calls] == [False, True]                 # the reference truncates the prompt only
    assert all(c["padding"] == "max_length" and c["max_length"] == 77 for c in tok.calls)
    assert torch.equal(guide.get_text_embeds(ids[1:2], ids[0]), emb)             # id tensors [1,77] / [77]
    g = torch.Generator().manual_seed(12)
    rgb = torch.rand(1, 3, 64, 64, generator=g).cuda().requires_grad_()
    eps_p, eps_n = torch.randn(1, 4, 32, 32, generator=g).cuda(), torch.randn(1, 4, 32, 32, generator=g).cuda()
    loss, imgs = guide.train_step(emb, rgb, islarge=True, guidance_scale=10, t=500, eps_posterior=eps_p, noise=eps_n)
    torch.cuda.synchronize()
    assert loss == 0 and imgs is None and rgb.grad is not None
    assert torch.isfinite(rgb.grad).all() and float(rgb.grad.abs().max()) > 0


def test_get_text_embeds_without_encoder_weights_is_the_previous_stand_in():
    st, sdm, L = _mods()
    guide = _tiny_guidance(sdm)
    free = torch.cuda.memory_allocated()
    got = guide.get_text_embeds(["a hamburger"], [""])
    assert guide.text_encoder is None and torch.cuda.memory_allocated() - free <= got.numel() * 4
    want = []
    for s in ("", "a hamburger"):
        gen = torch.Generator().manual_seed(int.from_bytes(hashlib.sha256(("mi3d:" + s).encode()).digest()[:4], "little"))
        want.append(torch.randn(1, 77, guide.unet_cfg["cross_dim"], generator=gen))
    assert torch.equal(got.cpu(), torch.cat(want))


def test_bad_input_raises(tiny):
    ref, enc = tiny
    st, sdm, L = _mods()
    good = sd_text_ref.make_ids((5,), seed=13)
    for bad in (good,                                        # CPU ids
                good.cuda().int(),                           # int32
                good[:, :76].cuda(),                         # wrong length
                good[0].cuda(),                              # no batch dimension
                good.repeat(3, 1).cuda()):                   # more prompts than max_batch
        with pytest.raises(L.Mi3dError):
            enc(bad)
    for v in (-1, ref.cfg["vocab"]):                         # out of range
        x = good.clone().cuda()
        x[0, 3] = v
        with pytest.raises(L.Mi3dError):
            enc(x)
    with pytest.raises(L.Mi3dError):
        st.TextEncoder("cuda", cfg=dict(ref.cfg, heads=1))
    with pytest.raises(L.Mi3dError):                          # a state_dict with a missing tensor
        enc.load_state_dict({k: v for k, v in ref.state_dict().items() if "fc2" not in k})
    guide = _tiny_guidance(sdm)
    guide.load_diffusers_state_dict(text_encoder_state=ref.state_dict())
    with pytest.raises(L.Mi3dError, match="tokenizer"):       # strings without a tokenizer
        guide.get_text_embeds(["a hamburger"], [""])
    with pytest.raises(L.Mi3dError):                          # ids of the wrong shape
        guide.get_text_embeds(good.repeat(2, 1), good)
