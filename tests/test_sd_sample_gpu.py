"""GPU checks of the sampler (produce_latents / prompt_to_img on mi3d_sd_sample) against the fp32 restatement of the reference's loop
(tests/sd_sample_ref.py on oracle/sd_ref's U-Net), on the tiny configuration of test_sd_gpu.py and on seeded full-size SD-2.0.

Tolerance.  The engine stores activations in fp16, so every U-Net pass carries the fp16 storage error that test_sd_fullsize_gpu.py
measures, CFG multiplies the (text - uncond) part of it by the guidance scale, and each DDIM step feeds the previous step's error
back in.  The bounds below are that floor compounded over the steps, set from observed values with about 3x headroom.  Observed on
an H100 80GB HBM3 at 700 W: 5.5e-5 after one step; 6.5e-3 after two (v-prediction, trailing spacing, tiny U-Net at 64^2 latents);
2.8e-3 after two at 768 (full-size SD-2.0); 2.3e-3 / 2.9e-3 after three (full-size SD-2.0 at 512 / tiny at 384); 2.6e-3 / 3.9e-3
after four (epsilon / v); 1.9e-3 / 2.3e-3 after ten.
Graph replay against plain launches, and prompt_to_img against its three calls, are bitwise equal on the tiny configuration.  The
VAE decoder at 512 runs split-K GEMMs whose fp32 RED order varies from run to run, so two engines' decodes are held at 1e-3.
"""
import importlib
import json
import os

import pytest
import torch

import sd_sample_ref as ref
from oracle import sd_ref, sd_text_ref

pytestmark = pytest.mark.gpu

# relative L2 of the sampled latents against the fp32 oracle, per number of steps (tiny configuration, guidance 7.5)
TINY_BOUND = {1: 2e-4, 2: 2e-2, 3: 1e-2, 4: 1e-2, 10: 1e-2}


def _rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / b.norm()), float(torch.dot(a, b) / (a.norm() * b.norm()))


def _equal(a, b):
    print(f"max |diff| = {float((a - b).abs().max()):.3e}")
    return torch.equal(a, b)


@pytest.fixture
def fp32_oracle_on_gpu():
    m, c = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = m, c


def _spread(*models):
    with torch.no_grad():
        for mod in models:
            for m in mod.modules():
                if isinstance(m, (torch.nn.GroupNorm, torch.nn.LayerNorm)):
                    m.weight.uniform_(0.5, 1.5); m.bias.uniform_(-0.3, 0.3)


@pytest.fixture(scope="module")
def tiny():
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    torch.manual_seed(0)
    ucfg, vcfg = sd_ref.tiny_unet_config(), sd_ref.tiny_vae_config()
    unet, enc, dec = sd_ref.UNet2DConditionModel(ucfg).eval(), sd_ref.AutoencoderKLEncoder(vcfg).eval(), sd_ref.AutoencoderKLDecoder(vcfg).eval()
    _spread(unet, enc, dec)
    vae_state = {**enc.state_dict(), **dec.state_dict()}
    g = sdm.StableDiffusion("cuda", unet_cfg=dict(ucfg, latent_hw=32), vae_cfg=dict(vcfg, image_hw=256), unet_state=unet.state_dict(),
                            vae_state=vae_state)
    return sdm, g, unet, dec, vae_state


def _inputs(seed, hw=32, D=128):
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(1, 4, hw, hw, generator=gen), torch.randn(2, 77, D, generator=gen)


@pytest.mark.parametrize("pred", ["epsilon", "v_prediction"])
@pytest.mark.parametrize("n", [1, 4, 10])
def test_produce_latents_matches_the_oracle(tiny, n, pred):
    sdm, g, unet, dec, _ = tiny
    lat, ctx = _inputs(10 + n)
    want = ref.produce_latents_ref(unet, ctx, lat, n, 7.5, pred)
    g.prediction_type = pred
    try:
        got = g.produce_latents(ctx.cuda(), 256, 256, num_inference_steps=n, latents=lat.cuda())
    finally:
        g.prediction_type = "epsilon"
    e, c = _rel(got, want)
    print(f"n={n} {pred}: latents rel_l2={e:.3e} cos={c:.6f}")
    assert got.shape == (1, 4, 32, 32) and e < TINY_BOUND[n] and c > 1 - TINY_BOUND[n] ** 2 / 2
    if n == 4 and pred == "epsilon":
        e, c = _rel(g.decode_latents(got), sd_ref.decode_latents_ref(dec, want))
        print(f"decoded image rel_l2={e:.3e} cos={c:.6f}")
        assert e < 2e-2 and c > 0.9998


def test_graph_replay_matches_plain_launches(tiny):
    sdm, g, unet, _, vae_state = tiny
    plain = sdm.StableDiffusion("cuda", unet_cfg=g.unet_cfg, vae_cfg=g.vae_cfg, unet_state=unet.state_dict(), vae_state=vae_state,
                                graph_replay=False)
    lat, ctx = _inputs(3)
    lat, ctx = lat.cuda(), ctx.cuda()
    rep = sdm.StableDiffusion("cuda", unet_cfg=g.unet_cfg, vae_cfg=g.vae_cfg, unet_state=unet.state_dict(), vae_state=vae_state)
    want = plain.produce_latents(ctx, 256, 256, num_inference_steps=4, latents=lat)
    assert rep.engine.graph_replays() == 0
    assert _equal(rep.produce_latents(ctx, 256, 256, num_inference_steps=4, latents=lat), want)
    assert rep.engine.graph_replays() == 1                     # the sampling step list: captured at step 2, replayed after it
    assert _equal(rep.produce_latents(ctx, 256, 256, num_inference_steps=4, latents=lat), want)
    assert rep.engine.graph_replays() == 1 and plain.engine.graph_replays() == 0
    assert torch.equal(lat, _inputs(3)[0].cuda())          # x_T is not written


def test_no_host_synchronisation_once_the_schedule_is_cached(tiny):
    sdm, g, *_ = tiny
    lat, ctx = _inputs(4)
    lat, ctx = lat.cuda(), ctx.cuda()
    g.produce_latents(ctx, 256, 256, num_inference_steps=5, latents=lat)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = g.produce_latents(ctx, 256, 256, num_inference_steps=5, latents=lat)
        out2 = g.produce_latents(torch.cat([ctx[:1], ctx[:1], ctx[1:], ctx[1:]]), 256, 256, num_inference_steps=5)   # B = 2, drawn x_T
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert out2.shape == (2, 4, 32, 32) and torch.isfinite(out).all() and torch.isfinite(out2).all()


def test_prompt_to_img_composes_the_three_calls(tiny):
    sdm, g, *_ = tiny
    te = sd_text_ref.default_init(sd_text_ref.TextEncoderRef(sd_text_ref.tiny_config()), seed=3)
    g.load_diffusers_state_dict(text_encoder_state=te.state_dict())
    try:
        ids, neg = sd_text_ref.make_ids([9], seed=1), sd_text_ref.make_ids([2], seed=2)
        lat = _inputs(5)[0].cuda()
        imgs = g.prompt_to_img(ids, neg, 256, 256, num_inference_steps=3, latents=lat)
        want = g.decode_latents(g.produce_latents(g.get_text_embeds(ids, neg), 256, 256, num_inference_steps=3, latents=lat))
        assert imgs.shape == (1, 3, 256, 256) and _equal(imgs, want)
    finally:
        g.text_encoder = None


def test_second_size_plans_a_cached_engine(tiny):
    """384: latent widths 48 / 24 / 12 and VAE widths 192 / 96 / 48 neither divide 128 nor are multiples of it, so their convs run on
    the spatial-block tiles; the 12 x 12 level at batch 2 is 288 rows, off the 128-row grid"""
    sdm, g, unet, dec, _ = tiny
    lat, ctx = _inputs(6, hw=48)
    want = ref.produce_latents_ref(unet, ctx, lat, 3, 7.5)
    got = g.produce_latents(ctx.cuda(), 384, 384, num_inference_steps=3, latents=lat.cuda())
    assert list(g._size_engines) == [384]
    eng = g._size_engines[384]
    e, c = _rel(got, want)
    print(f"384: latents rel_l2={e:.3e} cos={c:.6f}")
    assert e < TINY_BOUND[3]
    e, c = _rel(g.decode_latents(got), sd_ref.decode_latents_ref(dec, want))
    print(f"384: decoded image rel_l2={e:.3e} cos={c:.6f}")
    assert e < 2e-2
    g.produce_latents(ctx.cuda(), 384, 384, num_inference_steps=3, latents=lat.cuda())
    assert list(g._size_engines) == [384] and g._size_engines[384] is eng
    for bad in (dict(height=384, width=256), dict(height=200, width=200)):
        with pytest.raises(sdm.L.Mi3dError):
            g.produce_latents(ctx.cuda(), num_inference_steps=3, **bad)
    with pytest.raises(sdm.L.Mi3dError):
        g.produce_latents(ctx.cuda(), 256, 256, num_inference_steps=0)
    with pytest.raises(sdm.L.Mi3dError):
        g.produce_latents(ctx.cuda(), 256, 256, latents=lat.cuda())             # 48^2 latents at 256
    with pytest.raises(sdm.L.Mi3dError):
        g.produce_latents(ctx[:1].cuda(), 256, 256)


def test_from_pretrained_reads_a_diffusers_directory(tiny, tmp_path):
    st = pytest.importorskip("safetensors.torch")
    sdm, g, unet, _, vae_state = tiny
    ucfg, vcfg = sd_ref.tiny_unet_config(), sd_ref.tiny_vae_config()
    te = sd_text_ref.default_init(sd_text_ref.TextEncoderRef(sd_text_ref.tiny_config()), seed=4)
    files = {
        "unet/config.json": dict(block_out_channels=list(ucfg["block_out"]), layers_per_block=1, attention_head_dim=list(ucfg["heads"]),
                                 cross_attention_dim=128, norm_num_groups=32, in_channels=4, out_channels=4, sample_size=32,
                                 use_linear_projection=True),
        "vae/config.json": dict(block_out_channels=list(vcfg["block_out"]), layers_per_block=1, norm_num_groups=32, in_channels=3,
                                latent_channels=4, out_channels=3, sample_size=256, scaling_factor=0.18215),
        "text_encoder/config.json": dict(hidden_act="gelu", hidden_size=128),
        "scheduler/scheduler_config.json": dict(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                                                num_train_timesteps=1000, prediction_type="v_prediction", set_alpha_to_one=False,
                                                steps_offset=1, timestep_spacing="trailing"),
    }
    for name, cfg in files.items():
        os.makedirs(tmp_path / os.path.dirname(name), exist_ok=True)
        (tmp_path / name).write_text(json.dumps(cfg))
    st.save_file({k: v.contiguous() for k, v in unet.state_dict().items()}, str(tmp_path / "unet" / "diffusion_pytorch_model.safetensors"))
    st.save_file({k: v.half().contiguous() for k, v in vae_state.items()}, str(tmp_path / "vae" / "diffusion_pytorch_model.fp16.safetensors"))
    st.save_file({k: v.contiguous() for k, v in te.state_dict().items()}, str(tmp_path / "text_encoder" / "model.safetensors"))
    p = sdm.StableDiffusion.from_pretrained(str(tmp_path), "cuda")
    assert (p.prediction_type, p.timestep_spacing, p.steps_offset, p.set_alpha_to_one) == ("v_prediction", "trailing", 1, False)
    assert p.unet_cfg == dict(ucfg, latent_hw=64) and p.vae_cfg["image_hw"] == 512 and p.text_encoder is not None
    q = sdm.StableDiffusion("cuda", unet_cfg=p.unet_cfg, vae_cfg=p.vae_cfg, unet_state=unet.state_dict(),
                            vae_state={k: v.half().float() for k, v in vae_state.items()})
    q.prediction_type, q.timestep_spacing = "v_prediction", "trailing"
    lat, ctx = _inputs(8, hw=64)
    a = p.produce_latents(ctx.cuda(), num_inference_steps=2, latents=lat.cuda())
    b = q.produce_latents(ctx.cuda(), num_inference_steps=2, latents=lat.cuda())
    assert _equal(a, b)
    e, _ = _rel(a, ref.produce_latents_ref(unet, ctx, lat, 2, 7.5, "v_prediction", "trailing"))
    print(f"from_pretrained v / trailing: latents rel_l2={e:.3e}")
    assert e < TINY_BOUND[2]
    assert _rel(p.decode_latents(a), q.decode_latents(a))[0] < 1e-3
    # a checkpoint missing a tensor, carrying one the configuration has no place for, or with a shape the configuration disagrees with
    # is refused, not filled with seeded weights, dropped, or read out of bounds
    good = {k: v.contiguous() for k, v in unet.state_dict().items()}
    first = next(iter(good))
    for bad in ({k: v for k, v in good.items() if k != first}, dict(good, **{"class_embedding.linear_1.weight": torch.zeros(8, 8)}),
                dict(good, **{first: torch.zeros(good[first].numel() + 64)})):
        st.save_file(bad, str(tmp_path / "unet" / "diffusion_pytorch_model.safetensors"))
        with pytest.raises(sdm.L.Mi3dError):
            sdm.StableDiffusion.from_pretrained(str(tmp_path), "cuda")


@pytest.fixture(scope="module")
def full():
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    g = sdm.StableDiffusion("cuda")                       # seeded SD-2.0 (the benchmark's weights)
    unet = ref.UNet(sd_ref.sd20_unet_config()).eval()
    unet.load_state_dict({k.replace("/", "."): v.detach().cpu() for k, v in g.unet.items()})
    for p in unet.parameters():
        p.requires_grad_(False)
    return sdm, g, unet.cuda()


def _oracle_cuda(unet, ctx, lat, n):
    return ref.produce_latents_ref(unet, ctx.cuda(), lat.cuda(), n, 7.5).cpu()


def test_full_size_512(full, fp32_oracle_on_gpu):
    sdm, g, unet = full
    lat, ctx = _inputs(9, hw=64, D=1024)
    got = g.produce_latents(ctx.cuda(), num_inference_steps=3, latents=lat.cuda())
    e, c = _rel(got, _oracle_cuda(unet, ctx, lat, 3))
    print(f"SD-2.0 512, 3 steps: latents rel_l2={e:.3e} cos={c:.6f}")
    assert e < TINY_BOUND[3]
    torch.manual_seed(0)
    lat50 = g.produce_latents(ctx.cuda())                 # the reference's defaults: 512, 50 steps, guidance 7.5, drawn x_T
    imgs = g.decode_latents(lat50)
    assert torch.isfinite(lat50).all() and imgs.shape == (1, 3, 512, 512) and float(imgs.min()) >= 0 and float(imgs.max()) <= 1


def test_full_size_768(full, fp32_oracle_on_gpu):
    """a 96 x 96 latent plan: 9 216-token self-attention at the first level; widths 96 / 48 / 24 / 12 on the spatial-block conv tiles,
    a 288-row deepest level, and a second U-Net + VAE engine planned and cached for the size"""
    sdm, g, unet = full
    lat, ctx = _inputs(11, hw=96, D=1024)
    got = g.produce_latents(ctx.cuda(), 768, 768, num_inference_steps=2, latents=lat.cuda())
    e, c = _rel(got, _oracle_cuda(unet, ctx, lat, 2))
    print(f"SD-2.0 768, 2 steps: latents rel_l2={e:.3e} cos={c:.6f}")
    assert torch.isfinite(got).all() and e < TINY_BOUND[2]
    imgs = g.decode_latents(got)
    assert imgs.shape == (1, 3, 768, 768) and torch.isfinite(imgs).all() and list(g._size_engines) == [768]
    g._size_engines.clear()
    torch.cuda.empty_cache()
