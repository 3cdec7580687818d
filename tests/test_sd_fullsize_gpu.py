"""GPU parity of the SD guidance engine AT BENCHMARK SIZE (BASELINE config 2: SD-2.0-base U-Net shapes, 64x64 latents, batch 2;
SD VAE encoder at 512x512) against the fp32 oracle (oracle/sd_ref.py) run once on the box's host cores.

This is the only place the engine's full-size PLAN is checked, not just run: the BN = 160 / 256 tiles, the split-K planner for
the 8x8 / 16x16 levels (K up to 23 040), T = 4096 self-attention and the 512x512 implicit-GEMM convolutions.

Tolerance.  north_star asks "within a stated fp16 tolerance ... 1e-3 rel of reference".  The engine keeps activations in fp16
between kernels (fp32 accumulate).  What that storage format alone costs is MEASURED here, not assumed: the same oracle is run a
second time with every module output rounded to fp16 (forward hooks: fp16 storage, fp32 arithmetic -- the most favourable fp16
execution there is) and its deviation from the fp32 oracle is printed next to the engine's.  The assertions are
    engine error  <=  max(2.5 x fp16-storage error of the oracle itself, 1e-3)
per tensor, i.e. the engine may not be meaningfully worse than the best possible fp16 execution of the reference arithmetic.
Random-init weights make this a harsh test: without trained weights nothing damps rounding noise through 25 residual blocks, and
classifier-free guidance multiplies the (text - uncond) difference by 10.
Measured on an H100 80GB HBM3 (sm_90a, 400 W power limit), engine (fp16-storage oracle) relative L2 error vs fp32: U-Net taps
2.9e-4 .. 1.9e-3 (2.1e-4 .. 1.3e-3), CFG noise_pred 1.08e-2 (9.0e-3), SDS grad 4.7e-3 (3.9e-3), latents 3.8e-4 (3.3e-4), d pred_rgb
3.3e-3 (2.7e-3): the engine sits within 1.5x of the fp16-storage floor everywhere; the 1e-3 figure of north_star is not reachable by ANY fp16-activation execution of this network."""
import importlib
import json
import os
import time

import pytest
import torch

from oracle import sd_ref

pytestmark = pytest.mark.gpu
REGISTRY = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sd20_registry.json")


def _rel(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / b.norm())


def _fp16_storage_hooks(model):
    """round every leaf module's output to fp16 and back: fp16 activations between kernels, fp32 math inside them"""
    hs = []
    for m in model.modules():
        if len(list(m.children())) == 0:
            hs.append(m.register_forward_hook(lambda mod, inp, out: out.half().float() if torch.is_tensor(out) else out))
    return hs


@pytest.fixture(scope="module")
def full():
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    torch.set_num_threads(min(32, torch.get_num_threads()))
    torch.manual_seed(0)
    t0 = time.time()
    unet = sd_ref.UNet2DConditionModel(sd_ref.sd20_unet_config()).eval()
    vae = sd_ref.AutoencoderKLEncoder(sd_ref.sd_vae_config()).eval()
    with torch.no_grad():
        for m in list(unet.modules()) + list(vae.modules()):
            if isinstance(m, (torch.nn.GroupNorm, torch.nn.LayerNorm)):
                m.weight.uniform_(0.8, 1.2); m.bias.uniform_(-0.1, 0.1)
    for p in list(unet.parameters()) + list(vae.parameters()):
        p.requires_grad_(False)
    g = sdm.StableDiffusion("cuda", unet_state=unet.state_dict(), vae_state=vae.state_dict())
    print(f"[full-size fixtures built in {time.time() - t0:.1f} s]")
    return sdm, g, unet, vae


def test_full_size_unet_cfg_sds(full):
    sdm, g, unet, vae = full
    gen = torch.Generator().manual_seed(11)
    lat = torch.randn(1, 4, 64, 64, generator=gen) * 0.8
    noise = torch.randn(1, 4, 64, 64, generator=gen)
    ctx = torch.randn(2, 77, 1024, generator=gen)
    t = 437
    a = sd_ref.alphas_cumprod()[t]
    x = torch.cat([a.sqrt() * lat + (1 - a).sqrt() * noise] * 2)

    def oracle():
        with torch.no_grad():
            out = unet(x, torch.tensor([t]), ctx)
        taps = {k: v.clone() for k, v in unet.taps.items()}
        un, tx = out.chunk(2)
        npred = tx + 10.0 * (tx - un)
        return taps, out, npred, torch.nan_to_num((1 - a) * (npred - noise))
    t0 = time.time()
    taps32, raw32, np32, grad32 = oracle()
    hooks = _fp16_storage_hooks(unet)
    taps16, raw16, np16, grad16 = oracle()
    for h in hooks:
        h.remove()
    print(f"[oracle fp32 + fp16-storage passes: {time.time() - t0:.1f} s on {torch.get_num_threads()} host threads]")
    tt = torch.tensor([t], dtype=torch.long, device="cuda")
    npred, grad = g.unet_sds(lat.cuda(), noise.cuda(), tt, ctx.cuda(), 10.0)
    torch.cuda.synchronize()
    print(f"{'tensor':16s} {'engine vs fp32':>15s} {'fp16-storage oracle vs fp32':>28s}")
    worst = 0.0
    for name, ref in taps32.items():
        got = g.engine.debug_tensor(name).float().view(ref.shape[0], ref.shape[2], ref.shape[3], ref.shape[1]).permute(0, 3, 1, 2)
        e, e16 = _rel(got, ref), _rel(taps16[name], ref)
        print(f"{name:16s} {e:15.3e} {e16:28.3e}")
        assert e <= max(2.5 * e16, 1e-3), (name, e, e16)
        worst = max(worst, e)
    e, e16 = _rel(npred, np32), _rel(np16, np32)
    print(f"{'noise_pred (CFG)':16s} {e:15.3e} {e16:28.3e}")
    assert e <= max(2.5 * e16, 1e-3)
    e, e16 = _rel(grad, grad32), _rel(grad16, grad32)
    print(f"{'SDS grad':16s} {e:15.3e} {e16:28.3e}")
    assert e <= max(2.5 * e16, 1e-3)
    assert torch.isfinite(npred).all() and torch.isfinite(grad).all()


def test_full_size_vae_encode_and_input_gradient(full):
    sdm, g, unet, vae = full
    gen = torch.Generator().manual_seed(12)
    rgb = torch.rand(1, 3, 128, 128, generator=gen)
    eps = torch.randn(1, 4, 64, 64, generator=gen)
    glat = torch.randn(1, 4, 64, 64, generator=gen)

    def oracle():
        r = rgb.clone().requires_grad_()
        img = torch.nn.functional.interpolate(r, (512, 512), mode="bilinear", align_corners=False)       # nerf/sd.py:124
        mean, logvar = vae(2 * img - 1)
        lat = (mean + torch.exp(0.5 * logvar) * eps) * 0.18215                                             # nerf/sd.py:217-218
        lat.backward(glat)
        return lat.detach(), r.grad.clone()
    t0 = time.time()
    lat32, g32 = oracle()
    hooks = _fp16_storage_hooks(vae)
    lat16, g16 = oracle()                 # fp16-rounded forward activations; the backward of the hooks passes gradients through unrounded
    for h in hooks:
        h.remove()
    print(f"[oracle VAE fwd+bwd x2: {time.time() - t0:.1f} s]")
    r_cu = rgb.cuda().requires_grad_()
    lat = g.encode_imgs(r_cu, eps.cuda())
    lat.backward(glat.cuda())
    torch.cuda.synchronize()
    e, e16 = _rel(lat.detach(), lat32), _rel(lat16, lat32)
    print(f"{'latents':16s} engine vs fp32 {e:.3e}   fp16-storage oracle vs fp32 {e16:.3e}")
    assert e <= max(2.5 * e16, 1e-3)
    e, e16 = _rel(r_cu.grad, g32), _rel(g16, g32)
    print(f"{'d pred_rgb':16s} engine vs fp32 {e:.3e}   fp16-storage(fwd) oracle vs fp32 {e16:.3e}")
    # the engine also stores the BACKWARD activations in fp16, which the hooked oracle does not emulate: allow 4x
    assert e <= max(4 * e16, 1e-3)
    assert torch.isfinite(r_cu.grad).all()


def test_registry_order_is_pinned(full):
    """StableDiffusion.__init__ draws the seeded stand-in weights in registry order, so the SD-2.0 registry keeps its names and
    shapes in the recorded order (tests/golden/make_golden_sd_registry.py); it does not depend on which state dicts were loaded"""
    sdm, g, unet, vae = full
    with open(REGISTRY) as f:
        ref = json.load(f)
    assert len(g.engine.names) == len(ref) == 936
    assert g.engine.names == [n for n, _ in ref]
    assert g.engine.shapes == [tuple(s) for _, s in ref]
