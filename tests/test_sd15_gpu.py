"""GPU: Stable Diffusion 1.5 guidance (`StableDiffusion(sd_version='1.5')`).

* The fused attention at SD-1.5's head dims (40, 80, 160; 64 as the control) through `mi3d_op_attention_core`, i.e. through
  Builder::attention_core as the SD engine records it, against float64 computed from exactly the fp16 values the kernel reads.  The
  element-wise bound is the one of test_op_layer_gpu.py's fused-attention case with the head dim generalised (a d-term fp32 dot
  product, scale 1 / sqrt(d)); the worst err / bound ratio of every case is printed.
* The full-size SD-1.5 U-Net (64x64 latents, batch 2, 1x1-conv projections loaded from `[C, C, 1, 1]` tensors) + CFG + SDS gradient
  against the fp32 oracle (tests/sd15_ref.py: oracle/sd_ref.py's U-Net with conv projections), and the SD-1.5 text encoder
  (quick-GELU) against sd15_ref's form of oracle/sd_text_ref.py, both under the rule of test_sd_fullsize_gpu.py: engine error <= max(2.5 x the fp16-storage oracle's error, 1e-3).
* `train_step` on both branches, its repeatability (run to run, graph replay, plain launches), and the parameter registry against
  diffusers' names and shapes.
"""
import ctypes as C
import importlib
import math
import time

import pytest
import torch

import sd15_ref
from oracle import sd_ref, sd_text_ref

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
U16 = 2.0 ** -11
SUB16 = 2.0 ** -25
ERR_ARG = 1000001


@pytest.fixture(scope="module")
def L():
    return importlib.import_module("make-it-3d_b200._lib")


def _rel(a, b):
    a, b = a.detach().double().flatten().cpu(), b.double().flatten().cpu()
    return float((a - b).norm() / b.norm())


class _Fp16Storage:
    """round every leaf module's output to fp16 and back while active: fp16 activations between kernels, fp32 math inside them"""

    def __init__(self, model):
        self.model = model

    def __enter__(self):
        self.hs = [m.register_forward_hook(lambda mod, inp, out: out.half().float() if torch.is_tensor(out) else out)
                   for m in self.model.modules() if len(list(m.children())) == 0]

    def __exit__(self, *a):
        for h in self.hs:
            h.remove()


def _check16(name, got, ref32, ref16):
    e, e16 = _rel(got, ref32), _rel(ref16, ref32)
    print(f"{name:44s} engine vs fp32 {e:.3e}   fp16-storage oracle vs fp32 {e16:.3e}")
    assert e <= max(2.5 * e16, 1e-3), (name, e, e16)


# ------------------------------------------------------------------------------------------------------------------------------
# fused attention at every head dim
# ------------------------------------------------------------------------------------------------------------------------------
def _col(x, c):
    """device pointer of column c of the fp16 matrix x (q, k and v of a packed projection)"""
    return C.c_void_p(x.data_ptr() + 2 * c)


def _attention(L, q, ldq, k, ldk, v, ldv, o, B, T, Tk, valid, heads, d):
    """q, k, v: device pointers"""
    return L.lib().mi3d_op_attention_core(q, C.c_longlong(ldq), k, C.c_longlong(ldk), v, C.c_longlong(ldv), L.ptr(o),
                                          C.c_longlong(o.shape[1]), C.c_int(B), C.c_int(T), C.c_int(Tk), C.c_int(valid), C.c_int(heads),
                                          C.c_int(d), L.stream())


def _heads_view(x, B, tokens, heads, d):
    """[B][heads][tokens][d] float64 of the token matrix x [B*tokens, >= heads*d] (head h at columns h*d .. h*d + d - 1)"""
    return x[:, :heads * d].double().reshape(B, tokens, heads, d).permute(0, 2, 1, 3)


def _check_attention(what, o, Q, K, V, valid):
    """o [B*T, heads*d] fp16 vs fp64 softmax(Q K^T / sqrt d) V over the first `valid` keys, element-wise; one (batch, head) at a time.
    Bound per key term (test_op_layer_gpu.py): a logit error sigma (fp32 dot of d products, exp / ex2 ulps and the rounding of its
    argument) moves p_j by p_j (sigma_j + sum_i p_i sigma_i); P is rounded to fp16 before the PV product (2^-11 p_j + 2^-25 per
    term), the PV product accumulates the keys in fp32, and O is rounded to fp16 once."""
    B, heads, T, d = Q.shape
    Tk = K.shape[2]
    worst = 0.0
    for b in range(B):
        for h in range(heads):
            q, kk, vv = Q[b, h], K[b, h, :valid], V[b, h, :valid]
            z = (q @ kk.T) / math.sqrt(d)
            P = torch.softmax(z, dim=-1)
            ref = P @ vv
            zmax = z.amax(-1, keepdim=True)
            dot = 2 * d * U32 * (q.abs() @ kk.abs().T) / math.sqrt(d)
            ulp = 2.0 ** -20 + 2 * U32 * (z.abs() + zmax.abs())
            sigma = dot + ulp
            ebar = (P * sigma).sum(-1, keepdim=True)
            rho = 1.01 * (sigma + ebar + ulp.amax(-1, keepdim=True) + (Tk / 4 + 16) * U32)
            p_bound = P * rho + U16 * P + SUB16
            e = p_bound @ vv.abs() + 2 * Tk * U32 * (P @ vv.abs())
            bound = e + U16 * (ref.abs() + e) + SUB16
            got = o.view(B, T, heads, d)[b, :, h].double()
            worst = max(worst, ((got - ref).abs() / bound).max().item())
    print(f"{what}: worst err/bound {worst:.3g}")
    assert worst <= 1.0, f"{what}: err/bound {worst:.3g}"           # NaN fails here too


# (head_dim, tokens): the self-attention levels of SD-1.5 at 64x64 latents (8 heads everywhere; 64 tokens = the mid block), and the
# SD-2 head dim as the control
LEVELS = [(40, 4096), (80, 1024), (160, 256), (160, 64), (64, 256)]


@pytest.mark.parametrize("d,T", LEVELS)
def test_self_attention_on_packed_qkv_matches_fp64(L, d, T):
    """the U-Net's self-attention layout: q | k | v side by side in one [B*T, 3C] matrix (ld = 3C), every key valid"""
    B, heads = 2, 8
    Cm = heads * d
    g = torch.Generator(device="cuda").manual_seed(d * 7 + T)
    qkv = torch.randn(B * T, 3 * Cm, device="cuda", generator=g).half()
    o = torch.empty(B * T, Cm, dtype=torch.float16, device="cuda")
    L.check(_attention(L, _col(qkv, 0), 3 * Cm, _col(qkv, Cm), 3 * Cm, _col(qkv, 2 * Cm), 3 * Cm, o, B, T, T, T, heads, d), "op_attention_core")
    torch.cuda.synchronize()
    Q, K, V = (_heads_view(qkv[:, i * Cm:], B, T, heads, d) for i in range(3))
    _check_attention(f"self attention d{d} T{T}", o, Q, K, V, T)
    o1 = torch.empty_like(o)                                          # no atomics: launch to launch bit-identical
    L.check(_attention(L, _col(qkv, 0), 3 * Cm, _col(qkv, Cm), 3 * Cm, _col(qkv, 2 * Cm), 3 * Cm, o1, B, T, T, T, heads, d), "op_attention_core")
    torch.cuda.synchronize()
    assert torch.equal(o.view(torch.int16), o1.view(torch.int16))


@pytest.mark.parametrize("d,T", LEVELS)
def test_cross_attention_on_padded_context_matches_fp64(L, d, T):
    """the U-Net's cross-attention layout: q [B*T, C], k | v side by side in one [B*128, 2C] matrix (ld = 2C) of the text context
    padded to 128 rows, of which the first 77 take part; the padded rows hold +-60000 and must not reach the output"""
    B, heads, Tk, valid = 2, 8, 128, 77
    Cm = heads * d
    g = torch.Generator(device="cuda").manual_seed(d * 11 + T)
    q = torch.randn(B * T, Cm, device="cuda", generator=g).half()
    kv = torch.randn(B * Tk, 2 * Cm, device="cuda", generator=g)
    kv.view(B, Tk, 2 * Cm)[:, valid:] = (torch.randint(0, 2, (B, Tk - valid, 2 * Cm), device="cuda", generator=g) * 2 - 1) * 60000.0
    kv = kv.half()
    o = torch.empty(B * T, Cm, dtype=torch.float16, device="cuda")
    L.check(_attention(L, _col(q, 0), Cm, _col(kv, 0), 2 * Cm, _col(kv, Cm), 2 * Cm, o, B, T, Tk, valid, heads, d), "op_attention_core")
    torch.cuda.synchronize()
    _check_attention(f"cross attention d{d} T{T} keys {valid}/{Tk}", o, _heads_view(q, B, T, heads, d),
                     _heads_view(kv, B, Tk, heads, d), _heads_view(kv[:, Cm:], B, Tk, heads, d), valid)


@pytest.mark.parametrize("d", [40, 80, 160])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_attention_online_rescale(L, d, sign):
    """Logits that keep growing along the key axis force the online rescale (O rows in registers multiplied by alpha) in every key
    block; logits that shrink never trigger it.  The ramp is carried by the first and the last column of each head, so it also
    passes through the zero-filled tail of the last 64-column chunk."""
    B, T, Tk, heads = 1, 256, 1024, 2
    Cm = heads * d
    g = torch.Generator(device="cuda").manual_seed(d + (sign > 0))
    q = torch.zeros(B * T, Cm, device="cuda")
    k = torch.randn(B * Tk, Cm, device="cuda", generator=g) * 0.05
    ramp = sign * torch.linspace(0.0, 60.0, Tk, device="cuda")
    for h in range(heads):
        for col in (h * d, h * d + d - 1):
            q[:, col] = math.sqrt(d) / 2                     # every query: logit = ramp(key)
            k[:, col] = ramp
    v = torch.randn(B * Tk, Cm, device="cuda", generator=g)
    q, k, v = q.half(), k.half(), v.half()
    o = torch.empty(B * T, Cm, dtype=torch.float16, device="cuda")
    L.check(_attention(L, _col(q, 0), Cm, _col(k, 0), Cm, _col(v, 0), Cm, o, B, T, Tk, Tk, heads, d), "op_attention_core")
    torch.cuda.synchronize()
    assert torch.isfinite(o).all()
    _check_attention(f"rescale d{d} sign {sign:+.0f}", o, _heads_view(q, B, T, heads, d), _heads_view(k, B, Tk, heads, d),
                     _heads_view(v, B, Tk, heads, d), Tk)


def test_attention_rejects_other_head_dims(L):
    B, T, heads, d = 1, 128, 2, 48
    x = torch.zeros(B * T, 3 * heads * d, dtype=torch.float16, device="cuda")
    o = torch.zeros(B * T, heads * d, dtype=torch.float16, device="cuda")
    assert _attention(L, _col(x, 0), 3 * heads * d, _col(x, 0), 3 * heads * d, _col(x, 0), 3 * heads * d, o, B, T, T, T, heads, d) == ERR_ARG
    assert (o == 0).all()


# ------------------------------------------------------------------------------------------------------------------------------
# full-size SD-1.5
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    torch.set_num_threads(min(32, torch.get_num_threads()))
    torch.manual_seed(0)
    t0 = time.time()
    unet = sd15_ref.sd15_unet().eval()
    vae = sd_ref.AutoencoderKLEncoder(sd_ref.sd_vae_config()).eval()
    with torch.no_grad():
        for m in list(unet.modules()) + list(vae.modules()):
            if isinstance(m, (torch.nn.GroupNorm, torch.nn.LayerNorm)):
                m.weight.uniform_(0.8, 1.2); m.bias.uniform_(-0.1, 0.1)
    for p in list(unet.parameters()) + list(vae.parameters()):
        p.requires_grad_(False)
    g = sdm.StableDiffusion("cuda", sd_version="1.5", unet_state=unet.state_dict(), vae_state=vae.state_dict())
    print(f"[SD-1.5 fixtures built in {time.time() - t0:.1f} s]")
    return sdm, g, unet, vae


def test_registry_matches_the_diffusers_sd15_state_dict(full):
    sdm, g, unet, vae = full
    assert g.unet_cfg == sdm.sd15_unet_cfg()
    ref = unet.state_dict()
    names, shapes = [], []
    for n, s in zip(g.engine.names, g.engine.shapes):
        if "#" not in n and n.split(".")[0] not in ("encoder", "quant_conv", "decoder", "post_quant_conv"):
            names.append(n); shapes.append(tuple(s))
    assert sorted(names) == sorted(ref) and len(names) == 686
    assert dict(zip(names, shapes)) == {k: tuple(v.shape) for k, v in ref.items()}
    assert shapes[names.index("down_blocks.0.attentions.0.proj_in.weight")] == (320, 320, 1, 1)
    assert shapes[names.index("mid_block.attentions.0.proj_out.weight")] == (1280, 1280, 1, 1)
    assert sum(math.prod(s) for s in shapes) == 859_520_964


def test_full_size_sd15_unet_cfg_sds(full):
    sdm, g, unet, vae = full
    gen = torch.Generator().manual_seed(11)
    lat = torch.randn(1, 4, 64, 64, generator=gen) * 0.8
    noise = torch.randn(1, 4, 64, 64, generator=gen)
    ctx = torch.randn(2, 77, 768, generator=gen)
    t = 437
    a = sd_ref.alphas_cumprod()[t]
    x = torch.cat([a.sqrt() * lat + (1 - a).sqrt() * noise] * 2)

    def oracle():
        with torch.no_grad():
            out = unet(x, torch.tensor([t]), ctx)
        taps = {k: v.clone() for k, v in unet.taps.items()}
        un, tx = out.chunk(2)
        npred = tx + 10.0 * (tx - un)
        return taps, npred, torch.nan_to_num((1 - a) * (npred - noise))
    t0 = time.time()
    taps32, np32, grad32 = oracle()
    with _Fp16Storage(unet):
        taps16, np16, grad16 = oracle()
    print(f"[oracle fp32 + fp16-storage passes: {time.time() - t0:.1f} s on {torch.get_num_threads()} host threads]")
    tt = torch.tensor([t], dtype=torch.long, device="cuda")
    npred, grad = g.unet_sds(lat.cuda(), noise.cuda(), tt, ctx.cuda(), 10.0)
    torch.cuda.synchronize()
    for name, ref in taps32.items():
        got = g.engine.debug_tensor(name).float().view(ref.shape[0], ref.shape[2], ref.shape[3], ref.shape[1]).permute(0, 3, 1, 2)
        _check16(f"SD-1.5 {name}", got, ref, taps16[name])
    _check16("SD-1.5 noise_pred (CFG)", npred, np32, np16)
    _check16("SD-1.5 SDS grad", grad, grad32, grad16)
    assert torch.isfinite(npred).all() and torch.isfinite(grad).all()


def _text_oracle():
    ref = sd_text_ref.default_init(sd15_ref.sd15_text_encoder(), seed=5).eval()
    for p in ref.parameters():
        p.requires_grad_(False)
    return ref


def test_sd15_text_encoder_matches_the_fp32_oracle(full):
    sdm, g, unet, vae = full
    ref = _text_oracle()
    g.load_diffusers_state_dict(text_encoder_state=ref.state_dict())
    enc = g.text_encoder
    assert enc.cfg["hidden_act"] == "quick_gelu" and enc.act == 1 and enc.cfg["width"] == 768 and enc.cfg["layers"] == 12
    assert enc.names == list(ref.state_dict()) and len(enc.names) == 196
    ids = torch.cat([sd_text_ref.make_ids((2, 11, 90), pad=49407, seed=7), sd_text_ref.make_ids((5,), pad=49407, seed=8)])
    with torch.no_grad():
        f32 = ref(ids)[0]
        with _Fp16Storage(ref):
            f16 = ref(ids)[0]
    got = torch.cat([enc(ids[:2].cuda())[0], enc(ids[2:].cuda())[0]]).cpu()
    assert got.shape == (4, 77, 768) and torch.isfinite(got).all()
    _check16("SD-1.5 text encoder, 4 prompts", got, f32, f16)
    for i in range(4):
        _check16(f"SD-1.5 text encoder, prompt {i}", got[i], f32[i], f16[i])
    # StableDiffusion.get_text_embeds with token ids (no tokenizer): [negative, positive] in one call
    emb = g.get_text_embeds(ids[1:2], ids[0:1])
    assert emb.shape == (2, 77, 768)
    _check16("SD-1.5 get_text_embeds", emb.cpu(), f32[[0, 1]], f16[[0, 1]])


def _step(g, islarge, t, seed):
    gen = torch.Generator().manual_seed(seed)
    rgb = torch.rand(1, 3, 128, 128, generator=gen).cuda().requires_grad_()
    emb = torch.randn(2, 77, g.unet_cfg["cross_dim"], generator=gen).cuda()
    eps, noise = torch.randn(1, 4, 64, 64, generator=gen).cuda(), torch.randn(1, 4, 64, 64, generator=gen).cuda()
    loss, imgs = g.train_step(emb, rgb, islarge=islarge, guidance_scale=10, t=t, eps_posterior=eps, noise=noise)
    torch.cuda.synchronize()
    return rgb.grad, loss, imgs


def _spread(grads):
    return max(_rel(a, grads[0]) for a in grads[1:])


def test_sd15_train_step_branches_repeatability_and_graph_replay(full):
    """Both branches of train_step on the SD-1.5 engine.  Repeated calls, graph replay (calls 3 and 4) and plain launches on a second
    engine must agree: not bit for bit, because the full-size plan splits the K dimension of the deep levels' GEMMs and their fp32
    partial sums meet by RED in whatever order the SMs finish (fp16 rounding flips then travel through 25 residual blocks and CFG's
    x10), exactly as in the SD-2.0 plan, whose spread is measured alongside.  The bound is the fp16-storage floor of the SDS
    gradient measured in test_full_size_sd15_unet_cfg_sds (3.8e-3 .. 3.9e-3 relative L2), times 2.5.  The fused attention itself has no
    atomics: test_self_attention_on_packed_qkv_matches_fp64 checks it is bit-identical launch to launch."""
    sdm, g, unet, vae = full
    grads = [_step(g, True, 600, 21)[0] for _ in range(4)]
    assert grads[0] is not None and torch.isfinite(grads[0]).all() and grads[0].abs().sum() > 0
    assert g.engine.graph_replays() > 0
    plain = sdm.StableDiffusion("cuda", sd_version="1.5", unet_state=unet.state_dict(), vae_state=vae.state_dict(), graph_replay=False)
    grads.append(_step(plain, True, 600, 21)[0])
    del plain
    sd20 = sdm.StableDiffusion("cuda", sd_version="2.0")
    s20 = _spread([_step(sd20, True, 600, 21)[0] for _ in range(4)])
    del sd20
    torch.cuda.empty_cache()
    s15 = _spread(grads)
    print(f"d pred_rgb spread over 4 calls + plain launches: SD-1.5 {s15:.3e} (SD-2.0 over 4 calls: {s20:.3e})")
    assert s15 <= 2.5 * 3.8e-3
    _, loss, imgs = _step(g, False, 300, 22)                            # t <= 0.4 T on a small view: the denoise branch
    assert loss == 0 and imgs is not None and imgs.shape == (1, 3, 512, 512) and torch.isfinite(imgs).all()
    assert float(imgs.min()) >= 0.0 and float(imgs.max()) <= 1.0


def test_sd15_without_a_checkpoint_is_refused():
    sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
    with pytest.raises(ValueError, match="state dicts"):
        sdm.StableDiffusion("cuda", sd_version="1.5")
