"""fp32 torch restatement of DPT-Hybrid (`DPTDepthModel(backbone="vitb_rn50_384", non_negative=True)`, the reference's depth prior,
main.py:111-127, 196-214), keyed by the reference's `state_dict()` names.  Test infrastructure only (CPU or GPU, fp32).

Architecture (DPT/dpt/{vit,blocks,models}.py over timm's `vit_base_resnet50_384`):
* ResNetV2 trunk, not pre-activated: weight-standardised convs ((w - mean) / sqrt(var + 1e-8), biased variance, per output channel),
  TF-"same" padding, GroupNorm(32, eps 1e-5).  Stem 7x7/2 conv 3->64 (pad 2 before, 3 after) + GN + ReLU, 3x3/2 max-pool (pad 0 / 1).
  Stages of 3 / 4 / 9 bottlenecks (64->256, 128->512, 256->1024), stride on conv2 of block 0 of stages 1 and 2,
  out = relu(norm3(conv3(.)) + shortcut), shortcut = norm(conv1x1/s(x)) on block 0.
* Tokens: 1x1 conv 1024->768 on 24x24, cls token, pos_embed (at 384^2 its resize is the identity); 12 pre-LN ViT-B blocks (12 heads of
  64, exact GELU, LayerNorm eps 1e-6).  The final norm and the classifier head are never read.
* Reassemble: layer_1 / layer_2 are the stage-0 / stage-1 outputs; layer_3 / layer_4 take blocks 8 / 11: GELU(Linear([tokens | cls]))
  -> 1x1 conv (layer_4: then a 3x3/2 pad-1 conv).
* Decoder: layer{k}_rn 3x3 convs to 256 (no bias); four fusion blocks out = x0 (+ RCU1(x1)), RCU2, bilinear x2 (align_corners=True),
  1x1 out_conv; RCU(x) = x + conv2(relu(conv1(relu(x)))).  Head: 3x3 256->128, bilinear x2, 3x3 128->32 + ReLU, 1x1 32->1 + ReLU.

The 1x1 out_conv runs before the upsample: the align-corners bilinear weights sum to 1, so the two commute exactly in real arithmetic
(and this is the order csrc/dpt_engine.cu computes in).  `e16=True` rounds every tensor to fp16 where the engine stores one (weights of
its GEMMs, activations between kernels), which measures what fp16 storage alone costs.
"""
from collections import OrderedDict

import torch
import torch.nn.functional as F

WIDTHS = ((64, 256), (128, 512), (256, 1024))
DEPTHS = (3, 4, 9)
HOOKS = (8, 11)
IGNORED_PREFIXES = ("pretrained.model.norm.", "pretrained.model.head.", "scratch.refinenet4.resConfUnit1.")


def _trunk_names():
    b = "pretrained.model.patch_embed.backbone."
    out = [(b + "stem.conv.weight", (64, 3, 7, 7)), (b + "stem.norm.weight", (64,)), (b + "stem.norm.bias", (64,))]
    cin = 64
    for s, ((mid, cout), depth) in enumerate(zip(WIDTHS, DEPTHS)):
        for i in range(depth):
            p = f"{b}stages.{s}.blocks.{i}."
            if i == 0:
                out += [(p + "downsample.conv.weight", (cout, cin, 1, 1)), (p + "downsample.norm.weight", (cout,)),
                        (p + "downsample.norm.bias", (cout,))]
            c_in = cin if i == 0 else cout
            for j, (ci, co, k) in enumerate(((c_in, mid, 1), (mid, mid, 3), (mid, cout, 1)), 1):
                out += [(p + f"conv{j}.weight", (co, ci, k, k)), (p + f"norm{j}.weight", (co,)), (p + f"norm{j}.bias", (co,))]
        cin = cout
    return out


def param_shapes():
    """every tensor the forward reads, in the engine's registry order"""
    m, C = "pretrained.model.", 768
    out = [(m + "cls_token", (1, 1, C)), (m + "pos_embed", (1, 577, C))] + _trunk_names()
    out += [(m + "patch_embed.proj.weight", (C, 1024, 1, 1)), (m + "patch_embed.proj.bias", (C,))]
    for i in range(12):
        p = f"{m}blocks.{i}."
        out += [(p + "norm1.weight", (C,)), (p + "norm1.bias", (C,)), (p + "attn.qkv.weight", (3 * C, C)), (p + "attn.qkv.bias", (3 * C,)),
                (p + "attn.proj.weight", (C, C)), (p + "attn.proj.bias", (C,)), (p + "norm2.weight", (C,)), (p + "norm2.bias", (C,)),
                (p + "mlp.fc1.weight", (4 * C, C)), (p + "mlp.fc1.bias", (4 * C,)), (p + "mlp.fc2.weight", (C, 4 * C)), (p + "mlp.fc2.bias", (C,))]
    for k in (3, 4):
        p = f"pretrained.act_postprocess{k}."
        out += [(p + "0.project.0.weight", (C, 2 * C)), (p + "0.project.0.bias", (C,)), (p + "3.weight", (C, C, 1, 1)), (p + "3.bias", (C,))]
        if k == 4:
            out += [(p + "4.weight", (C, C, 3, 3)), (p + "4.bias", (C,))]
    for k, cin in enumerate((256, 512, 768, 768), 1):
        out.append((f"scratch.layer{k}_rn.weight", (256, cin, 3, 3)))
    for k in (4, 3, 2, 1):
        p = f"scratch.refinenet{k}."
        for u in ((1, 2) if k < 4 else (2,)):
            for j in (1, 2):
                out += [(p + f"resConfUnit{u}.conv{j}.weight", (256, 256, 3, 3)), (p + f"resConfUnit{u}.conv{j}.bias", (256,))]
        out += [(p + "out_conv.weight", (256, 256, 1, 1)), (p + "out_conv.bias", (256,))]
    out += [("scratch.output_conv.0.weight", (128, 256, 3, 3)), ("scratch.output_conv.0.bias", (128,)),
            ("scratch.output_conv.2.weight", (32, 128, 3, 3)), ("scratch.output_conv.2.bias", (32,)),
            ("scratch.output_conv.4.weight", (1, 32, 1, 1)), ("scratch.output_conv.4.bias", (1,))]
    return OrderedDict(out)


def ignored_shapes():
    """the reference tensors the forward never reads (timm's final norm and ImageNet head, the deepest fusion block's unused RCU)"""
    out = [("pretrained.model.norm.weight", (768,)), ("pretrained.model.norm.bias", (768,)), ("pretrained.model.head.weight", (1000, 768)),
           ("pretrained.model.head.bias", (1000,))]
    for j in (1, 2):
        out += [(f"scratch.refinenet4.resConfUnit1.conv{j}.weight", (256, 256, 3, 3)), (f"scratch.refinenet4.resConfUnit1.conv{j}.bias", (256,))]
    return OrderedDict(out)


def hf_name_map():
    """reference name -> transformers' `DPTForDepthEstimation` name (hybrid config), for every reference tensor but timm's head"""
    b, h = "pretrained.model.patch_embed.backbone.", "dpt.embeddings.backbone.bit."
    m = {b + "stem.conv.weight": h + "embedder.convolution.weight", b + "stem.norm.weight": h + "embedder.norm.weight",
         b + "stem.norm.bias": h + "embedder.norm.bias"}
    for name, _ in _trunk_names()[3:]:
        m[name] = h + "encoder." + name[len(b):].replace(".blocks.", ".layers.")
    M = "pretrained.model."
    m.update({M + "cls_token": "dpt.embeddings.cls_token", M + "pos_embed": "dpt.embeddings.position_embeddings",
              M + "patch_embed.proj.weight": "dpt.embeddings.projection.weight", M + "patch_embed.proj.bias": "dpt.embeddings.projection.bias",
              M + "norm.weight": "dpt.layernorm.weight", M + "norm.bias": "dpt.layernorm.bias"})
    for i in range(12):
        p, q = f"{M}blocks.{i}.", f"dpt.encoder.layer.{i}."
        for a, c in (("norm1", "layernorm_before"), ("norm2", "layernorm_after"), ("attn.proj", "attention.output.dense"),
                     ("mlp.fc1", "intermediate.dense"), ("mlp.fc2", "output.dense")):
            for t in ("weight", "bias"):
                m[f"{p}{a}.{t}"] = f"{q}{c}.{t}"
        for t in ("weight", "bias"):    # packed q | k | v: see to_hf_state_dict / from_hf_state_dict
            m[f"{p}attn.qkv.{t}"] = tuple(f"{q}attention.attention.{s}.{t}" for s in ("query", "key", "value"))
    for k, i in ((3, 2), (4, 3)):
        p, q = f"pretrained.act_postprocess{k}.", f"neck.reassemble_stage."
        for t in ("weight", "bias"):
            m[f"{p}0.project.0.{t}"] = f"{q}readout_projects.{i}.0.{t}"
            m[f"{p}3.{t}"] = f"{q}layers.{i}.projection.{t}"
            if k == 4:
                m[f"{p}4.{t}"] = f"{q}layers.{i}.resize.{t}"
    for k in range(1, 5):
        m[f"scratch.layer{k}_rn.weight"] = f"neck.convs.{k - 1}.weight"
        p, q = f"scratch.refinenet{k}.", f"neck.fusion_stage.layers.{4 - k}."
        for t in ("weight", "bias"):
            m[f"{p}out_conv.{t}"] = f"{q}projection.{t}"
            for u in (1, 2):
                for j in (1, 2):
                    m[f"{p}resConfUnit{u}.conv{j}.{t}"] = f"{q}residual_layer{u}.convolution{j}.{t}"
    for i in (0, 2, 4):
        for t in ("weight", "bias"):
            m[f"scratch.output_conv.{i}.{t}"] = f"head.head.{i}.{t}"
    return m


def from_hf_state_dict(hf):
    """transformers' DPTForDepthEstimation state_dict -> the reference's names (without timm's ImageNet head, which it lacks)"""
    out = {}
    for ref, hfn in hf_name_map().items():
        out[ref] = torch.cat([hf[n] for n in hfn]) if isinstance(hfn, tuple) else hf[hfn]
    return out


def default_init(seed=0):
    """seeded weights in the spirit of transformers' DPT init (normal(0, 0.02) linears / convs, zero biases, unit norms)"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in list(param_shapes().items()) + list(ignored_shapes().items()):
        if ".norm" in name:
            out[name] = torch.ones(shape) if name.endswith("weight") else torch.zeros(shape)
        elif name.endswith("bias"):
            out[name] = torch.zeros(shape)
        else:
            out[name] = torch.randn(shape, generator=g) * 0.02
    return out


def _ws(w):
    flat = w.reshape(w.shape[0], -1)
    mean, var = flat.mean(1, keepdim=True), flat.var(1, unbiased=False, keepdim=True)
    return ((flat - mean) / torch.sqrt(var + 1e-8)).reshape(w.shape)


def forward(p, x, e16=False, taps=False):
    """p: reference-named fp32 tensors; x fp32 [1, 3, 384, 384] (normalised) -> inverse depth [1, 384, 384] (and the reassembled
    layer_1 .. layer_4 as NCHW fp32 when taps)"""
    r = (lambda t: t.half().float()) if e16 else (lambda t: t)
    W = lambda n: r(p[n])                                       # a weight the engine stores in fp16
    gn = lambda t, n: F.group_norm(t, 32, p[n + ".weight"], p[n + ".bias"], 1e-5)
    b = "pretrained.model.patch_embed.backbone."
    # trunk
    y = r(F.conv2d(F.pad(x, (2, 3, 2, 3)), r(_ws(p[b + "stem.conv.weight"])), stride=2))
    y = r(F.relu(gn(y, b + "stem.norm")))
    y = F.max_pool2d(F.pad(y, (0, 1, 0, 1), value=float("-inf")), 3, 2)
    feats = []
    for s, depth in enumerate(DEPTHS):
        for i in range(depth):
            q = f"{b}stages.{s}.blocks.{i}."
            stride = 2 if (s > 0 and i == 0) else 1
            if i == 0:
                sc = r(F.conv2d(y, r(_ws(p[q + "downsample.conv.weight"])), stride=stride))
                sc = r(gn(sc, q + "downsample.norm"))
            else:
                sc = y
            a = r(F.relu(gn(r(F.conv2d(y, r(_ws(p[q + "conv1.weight"])))), q + "norm1")))
            a = F.pad(a, (0, 1, 0, 1)) if stride == 2 else F.pad(a, (1, 1, 1, 1))
            a = r(F.relu(gn(r(F.conv2d(a, r(_ws(p[q + "conv2.weight"])), stride=stride)), q + "norm2")))
            y = r(F.relu(gn(r(F.conv2d(a, r(_ws(p[q + "conv3.weight"])))), q + "norm3") + sc))
        feats.append(y)
    # tokens and ViT
    M, C = "pretrained.model.", 768
    pos = p[M + "pos_embed"][0]
    t = r(F.conv2d(y, W(M + "patch_embed.proj.weight"), p[M + "patch_embed.proj.bias"]).flatten(2).transpose(1, 2)[0] + pos[1:])
    t = torch.cat([r(p[M + "cls_token"][0, 0] + pos[0])[None], t])                  # [577, C]
    ln = lambda v, n: r(F.layer_norm(v, (C,), p[n + ".weight"], p[n + ".bias"], 1e-6))
    lin = lambda v, n: v @ W(n + ".weight").t() + p[n + ".bias"]
    outs = {}
    for i in range(12):
        q = f"{M}blocks.{i}."
        qkv = r(lin(ln(t, q + "norm1"), q + "attn.qkv")).view(577, 3, 12, 64).permute(1, 2, 0, 3)
        a = F.softmax(qkv[0] @ qkv[1].transpose(1, 2) * 0.125, -1) @ qkv[2]
        a = r(a.transpose(0, 1).reshape(577, C))
        t = r(lin(a, q + "attn.proj") + t)
        t = r(lin(r(F.gelu(lin(ln(t, q + "norm2"), q + "mlp.fc1"))), q + "mlp.fc2") + t)
        if i in HOOKS:
            outs[i] = t
    def reassemble(tok, k):
        q = f"pretrained.act_postprocess{k}."
        w = W(q + "0.project.0.weight")
        v = r(F.gelu(tok[1:] @ w[:, :C].t() + (w[:, C:] @ tok[0] + p[q + "0.project.0.bias"])))
        v = v.t().reshape(1, C, 24, 24)
        v = r(F.conv2d(v, W(q + "3.weight"), p[q + "3.bias"]))
        if k == 4:
            v = r(F.conv2d(v, W(q + "4.weight"), p[q + "4.bias"], stride=2, padding=1))
        return v
    layers = [feats[0], feats[1], reassemble(outs[8], 3), reassemble(outs[11], 4)]
    # decoder
    conv3 = lambda v, n, bias=True: F.conv2d(v, W(n + ".weight"), p[n + ".bias"] if bias else None, padding=1)
    up = lambda v: r(F.interpolate(v, scale_factor=2, mode="bilinear", align_corners=True))
    rn = [r(conv3(v, f"scratch.layer{k}_rn", False)) for k, v in enumerate(layers, 1)]
    def rcu(v, n, add):                                         # add + conv2(relu(conv1(relu(v)))), add = v (+ x0)
        return r(conv3(r(F.relu(conv3(F.relu(v), n + ".conv1"))), n + ".conv2") + add)
    path = None
    for k in (4, 3, 2, 1):
        q = f"scratch.refinenet{k}."
        v = rn[k - 1] if path is None else rcu(rn[k - 1], q + "resConfUnit1", r(path + rn[k - 1]))
        v = rcu(v, q + "resConfUnit2", v)
        path = up(r(F.conv2d(v, W(q + "out_conv.weight"), p[q + "out_conv.bias"])))
    h = up(r(conv3(path, "scratch.output_conv.0")))
    h = r(F.relu(conv3(h, "scratch.output_conv.2")))
    out = F.relu(F.conv2d(h, p["scratch.output_conv.4.weight"], p["scratch.output_conv.4.bias"]))[:, 0]
    return (out, layers) if taps else out
