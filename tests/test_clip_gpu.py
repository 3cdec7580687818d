"""GPU parity of the CLIP engine (csrc/clip_engine.cu behind nerf/clip.py) against the fp32 oracle (oracle/clip_ref.py), at a tiny
configuration and at the full ViT-B/16 configuration, with seeded random weights (LayerNorms given some spread).

Tolerance, as in test_sd_fullsize_gpu.py: the engine keeps activations in fp16 between kernels, so the oracle is run a second time with
every leaf module's output rounded to fp16 (forward hooks) and the engine's relative error must stay within
max(2.5 x that fp16-storage error, 1e-3).  Observed values are printed."""
import importlib

import pytest
import torch

from oracle import clip_ref

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
    print(f"{name:34s} engine vs fp32 {e:.3e}   fp16-storage oracle vs fp32 {e16:.3e}")
    assert e <= max(2.5 * e16, 1e-3), (name, e, e16)


def _build(cfg, seed):
    clipm = importlib.import_module("make-it-3d_b200.nerf.clip")
    torch.manual_seed(0)
    ref = clip_ref.default_init(clip_ref.CLIPRef(cfg), seed=seed).eval()
    for p in ref.parameters():
        p.requires_grad_(False)
    return clipm, ref, clipm.CLIP("cuda", cfg=cfg, state_dict=ref.state_dict())


@pytest.fixture(scope="module", params=["tiny", "vit_b16"])
def model(request):
    cfg = clip_ref.tiny_config() if request.param == "tiny" else clip_ref.vit_b16_config()
    torch.set_num_threads(min(32, torch.get_num_threads()))
    return (request.param,) + _build(cfg, seed=5)


@pytest.fixture(scope="module")
def tiny():
    return _build(clip_ref.tiny_config(), seed=6)


def _oracle_losses(ref, rgb, ref_rgb, tok, res):
    r = rgb.clone().requires_grad_()
    aug = lambda x: clip_ref.aug(x, res)
    a, b = clip_ref.img_clip_loss(ref, r, ref_rgb, aug), clip_ref.img_text_clip_loss(ref, r, tok, aug)
    (a + b).backward()
    return a.detach(), b.detach(), r.grad


def test_encode_image_without_aug_matches_oracle(model):
    name, clipm, ref, m = model
    R = ref.cfg["image_res"]
    img = torch.randn(2, 3, R, R, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        f32 = ref.encode_image(img)
        with _Fp16Storage(ref):
            f16 = ref.encode_image(img)
    got = m.encode_image(img.cuda())
    _check(f"{name} encode_image (aug 0)", got, f32, f16)


@pytest.mark.parametrize("S", [512, 128])
def test_losses_and_input_gradient_match_oracle(model, S):
    name, clipm, ref, m = model
    R = ref.cfg["image_res"]
    g = torch.Generator().manual_seed(S)
    rgb, ref_rgb = torch.rand(1, 3, S, S, generator=g), torch.rand(1, 3, S, S, generator=g)
    tok = clip_ref.make_tokens([9], seed=S)
    a32, b32, g32 = _oracle_losses(ref, rgb, ref_rgb, tok, R)
    with _Fp16Storage(ref):
        a16, b16, g16 = _oracle_losses(ref, rgb, ref_rgb, tok, R)
    r = rgb.cuda().requires_grad_()
    a, b = m.losses(r, ref_rgb.cuda(), tok.cuda())
    (a + b).backward()
    torch.cuda.synchronize()
    _check(f"{name} {S}^2 img_clip_loss", a, a32, a16)
    _check(f"{name} {S}^2 img_text_clip_loss", b, b32, b16)
    _check(f"{name} {S}^2 d rgb", r.grad, g32, g16)
    assert torch.isfinite(r.grad).all()


def test_encode_text_matches_oracle_at_several_eot_positions(model):
    name, clipm, ref, m = model
    tok = clip_ref.make_tokens([2, 20, 50, 77], seed=7)
    with torch.no_grad():
        f32 = ref.encode_text(tok)
        with _Fp16Storage(ref):
            f16 = ref.encode_text(tok)
    got = torch.cat([m.encode_text(tok[i:i + 2].cuda()) for i in (0, 2)])
    for i, n in enumerate((2, 20, 50, 77)):
        _check(f"{name} encode_text EOT at {n - 1}", got[i], f32[i], f16[i])


def test_losses_gradient_equals_the_two_call_formulation(tiny):
    """The reference encodes rgb twice (nerf/utils.py:436-453).  At a res x res input the reference's aug written as (x - mean) * (1/std)
    is bit-identical to the engine's, so the two formulations see the same patches:
    (1) encode rgb ONCE through encode_image, use the features in both losses: equal to losses() to 1e-5 (one backward of the same
        summed feature gradient; batching [rgb, ref_rgb] changes nothing for rgb's rows);
    (2) the literal two-call form: two engine backwards whose results autograd adds.  The input-gradient pass stores gradients in fp16,
        so backward(a) + backward(b) equals backward(a + b) only to fp16 rounding.
    ref_rgb is marked as requiring a gradient so that its features come from the same (taped, materialised-attention) forward as inside
    losses(); a forward without a tape uses the fused attention kernel, whose fp16 rounding differs in the last bits."""
    clipm, ref, m = tiny
    R = ref.cfg["image_res"]
    g = torch.Generator().manual_seed(11)
    rgb, ref_rgb = torch.rand(1, 3, R, R, generator=g).cuda(), torch.rand(1, 3, R, R, generator=g).cuda()
    tok = clip_ref.make_tokens([12], seed=11).cuda()
    mean = torch.tensor(clip_ref.CLIP_MEAN, device="cuda").view(1, 3, 1, 1)
    inv_std = 1 / torch.tensor(clip_ref.CLIP_STD, device="cuda").view(1, 3, 1, 1)
    aug = lambda x: (x - mean) * inv_std
    norm = lambda z: z / z.norm(dim=-1, keepdim=True)
    r0 = rgb.clone().requires_grad_()
    a, b = m.losses(r0, ref_rgb, tok)
    (a + b).backward()
    ref_g = ref_rgb.clone().requires_grad_()
    r1 = rgb.clone().requires_grad_()
    z1 = norm(m.encode_image(aug(r1)))
    z2 = norm(m.encode_image(aug(ref_g)))
    zt = norm(m.encode_text(tok))
    (-(z1 * z2).sum(-1).mean() - (z1 * zt).sum(-1).mean()).backward()
    r2 = rgb.clone().requires_grad_()
    l2 = clip_ref.img_clip_loss(m, r2, ref_g, aug) + clip_ref.img_text_clip_loss(m, r2, tok, aug)
    l2.backward()
    torch.cuda.synchronize()
    e1, e2 = _rel(r1.grad, r0.grad), _rel(r2.grad, r0.grad)
    print(f"d rgb: one encode + summed feature gradient {e1:.2e}, literal two-call form {e2:.2e}")
    assert e1 <= 1e-5, e1
    assert e2 <= 3e-3, e2
    assert abs(float(l2.detach()) - float((a + b).detach())) <= 1e-5 * abs(float((a + b).detach())) + 1e-6


def test_graph_replay_and_repeated_runs_are_bit_identical(tiny):
    clipm, ref, m = tiny
    plain = clipm.CLIP("cuda", cfg=ref.cfg, state_dict=ref.state_dict(), graph_replay=False)
    assert plain.engine.stream is None and m.engine.stream is not None
    g = torch.Generator().manual_seed(13)
    rgb, ref_rgb = torch.rand(1, 3, 96, 96, generator=g).cuda(), torch.rand(1, 3, 96, 96, generator=g).cuda()
    tok = clip_ref.make_tokens([30], seed=13).cuda()

    def one(mm):
        r = rgb.clone().requires_grad_()
        a, b = mm.losses(r, ref_rgb, tok)
        (a + b).backward()
        feats = mm.encode_image(clip_ref.aug(rgb, ref.cfg["image_res"]))
        torch.cuda.synchronize()
        return a.detach().clone(), b.detach().clone(), r.grad.clone(), feats.clone()
    want = one(plain)
    assert all(torch.equal(x, y) for x, y in zip(one(plain), want))                  # run to run
    for call in range(4):
        got = one(m)
        assert all(torch.equal(x, y) for x, y in zip(got, want)), call                # graph replay from the third call on
    assert m.engine.graph_replays() >= 4 and plain.engine.graph_replays() == 0


def test_denoise_branch_with_native_clip_returns_the_oracle_losses(tiny):
    from oracle import sd_ref
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    clipm, ref, m = tiny
    torch.manual_seed(0)
    ucfg, vcfg = sd_ref.tiny_unet_config(), sd_ref.tiny_vae_config()
    unet, vae = sd_ref.UNet2DConditionModel(ucfg).eval(), sd_ref.AutoencoderKLEncoder(vcfg).eval()
    guide = sdm.StableDiffusion("cuda", unet_cfg=dict(ucfg, latent_hw=32), vae_cfg=dict(vcfg, image_hw=256), unet_state=unet.state_dict(),
                                vae_state=vae.state_dict())
    g = torch.Generator().manual_seed(17)
    rgb = torch.rand(1, 3, 64, 64, generator=g).cuda().requires_grad_()
    ctx = torch.randn(2, 77, ucfg["cross_dim"], generator=g).cuda()
    ref_rgb = torch.rand(1, 3, 256, 256, generator=g)
    tok = clip_ref.make_tokens([15], seed=17)
    loss, imgs = guide.train_step(ctx, rgb, islarge=False, t=350, ref_rgb=ref_rgb.cuda(), ref_text=tok.cuda(), clip_model=m)
    assert rgb.grad is None and imgs.shape == (1, 3, 256, 256) and torch.is_tensor(loss)
    R = ref.cfg["image_res"]
    aug = lambda x: clip_ref.aug(x, R)

    def oracle():
        with torch.no_grad():
            return 10 * clip_ref.img_clip_loss(ref, imgs.cpu(), ref_rgb, aug) + 10 * clip_ref.img_text_clip_loss(ref, imgs.cpu(), tok, aug)
    l32 = oracle()
    with _Fp16Storage(ref):
        l16 = oracle()
    _check("denoise branch 10 (img + text) loss", loss.detach(), l32, l16)


def test_cpu_tensors_and_bad_arguments_raise(tiny):
    clipm, ref, m = tiny
    L = importlib.import_module("make-it-3d_b200._lib")
    R = ref.cfg["image_res"]
    with pytest.raises(L.Mi3dError):
        m.encode_image(torch.rand(1, 3, R, R))
    with pytest.raises(L.Mi3dError):
        m.encode_text(clip_ref.make_tokens([5]))
    with pytest.raises(L.Mi3dError):                          # more images than max_batch
        m.encode_image(torch.rand(3, 3, R, R, device="cuda"))
    with pytest.raises(L.Mi3dError):                          # aug 0 needs res x res
        m.encode_image(torch.rand(1, 3, R + 16, R, device="cuda"))
    with pytest.raises(L.Mi3dError):
        m.encode_text(torch.zeros(1, 76, dtype=torch.long, device="cuda"))
    fresh = clipm.ClipEngine(ref.cfg, "cuda")
    with pytest.raises(L.Mi3dError):                          # backward without a tape
        fresh.encode_image_backward(torch.zeros(1, ref.cfg["embed_dim"], device="cuda"), 1, R, R)
    fresh.encode_image(torch.rand(1, 3, R, R, device="cuda"), 0, True)
    with pytest.raises(L.Mi3dError):                          # n_grad larger than the taped batch
        fresh.encode_image_backward(torch.zeros(2, ref.cfg["embed_dim"], device="cuda"), 2, R, R)
    fresh.encode_image(torch.rand(1, 3, R, R, device="cuda"), 0, False)
    with pytest.raises(L.Mi3dError):                          # a forward without grad drops the tape
        fresh.encode_image_backward(torch.zeros(1, ref.cfg["embed_dim"], device="cuda"), 1, R, R)
