"""Functional restatement of transformers' `Blip2ForConditionalGeneration.generate(pixel_values)` (blip2-opt, greedy, no text prompt):
weights dict (state_dict names) + pixel_values -> image_embeds, query_output, language_model_inputs, the last-row logits of every step
and the greedy ids.  Runs in the dtype of the weights it is given (float64 for the CPU parity test, float32 on the GPU).  e16=True
rounds every tensor the engine stores (activations between kernels, weights, the query tokens) to fp16: the precision floor of
csrc/blip2_engine.cu.  Each step recomputes the whole causal pass (no KV cache), as the engine does."""
import math

import torch
import torch.nn.functional as F


def blip2_opt_27b_cfg():
    """Salesforce/blip2-opt-2.7b's config.json"""
    return dict(image_size=224, patch=14, vision_width=1408, vision_layers=39, vision_heads=16, vision_mlp=6144,
                qformer_width=768, qformer_layers=12, qformer_heads=12, qformer_ffn=3072, cross_attention_frequency=2,
                num_query_tokens=32, opt_width=2560, opt_layers=32, opt_heads=32, opt_ffn=10240, vocab=50272, max_positions=2048,
                image_token_index=50265, bos_token_id=2, eos_token_id=50118)


def param_shapes(cfg):
    """{state_dict name: shape} of Blip2ForConditionalGeneration at cfg, in its order, without the tied language_model.lm_head.weight"""
    c = cfg
    Cv, Cq, Co, nq, P = c["vision_width"], c["qformer_width"], c["opt_width"], c["num_query_tokens"], c["patch"]
    Tv = (c["image_size"] // P) ** 2 + 1
    s = {"query_tokens": (1, nq, Cq), "vision_model.embeddings.class_embedding": (1, 1, Cv),
         "vision_model.embeddings.position_embedding": (1, Tv, Cv), "vision_model.embeddings.patch_embedding.weight": (Cv, 3, P, P),
         "vision_model.embeddings.patch_embedding.bias": (Cv,)}
    for i in range(c["vision_layers"]):
        p = f"vision_model.encoder.layers.{i}."
        s.update({p + "self_attn.qkv.weight": (3 * Cv, Cv), p + "self_attn.qkv.bias": (3 * Cv,), p + "self_attn.projection.weight": (Cv, Cv),
                  p + "self_attn.projection.bias": (Cv,), p + "layer_norm1.weight": (Cv,), p + "layer_norm1.bias": (Cv,),
                  p + "mlp.fc1.weight": (c["vision_mlp"], Cv), p + "mlp.fc1.bias": (c["vision_mlp"],), p + "mlp.fc2.weight": (Cv, c["vision_mlp"]),
                  p + "mlp.fc2.bias": (Cv,), p + "layer_norm2.weight": (Cv,), p + "layer_norm2.bias": (Cv,)})
    s.update({"vision_model.post_layernorm.weight": (Cv,), "vision_model.post_layernorm.bias": (Cv,),
              "qformer.layernorm.weight": (Cq,), "qformer.layernorm.bias": (Cq,)})
    for i in range(c["qformer_layers"]):
        p = f"qformer.encoder.layer.{i}."
        for n in ("query", "key", "value"):
            s.update({p + f"attention.attention.{n}.weight": (Cq, Cq), p + f"attention.attention.{n}.bias": (Cq,)})
        s.update({p + "attention.output.dense.weight": (Cq, Cq), p + "attention.output.dense.bias": (Cq,),
                  p + "attention.output.LayerNorm.weight": (Cq,), p + "attention.output.LayerNorm.bias": (Cq,)})
        if i % c["cross_attention_frequency"] == 0:
            for n, k in (("query", Cq), ("key", Cv), ("value", Cv)):
                s.update({p + f"crossattention.attention.{n}.weight": (Cq, k), p + f"crossattention.attention.{n}.bias": (Cq,)})
            s.update({p + "crossattention.output.dense.weight": (Cq, Cq), p + "crossattention.output.dense.bias": (Cq,),
                      p + "crossattention.output.LayerNorm.weight": (Cq,), p + "crossattention.output.LayerNorm.bias": (Cq,)})
        s.update({p + "intermediate_query.dense.weight": (c["qformer_ffn"], Cq), p + "intermediate_query.dense.bias": (c["qformer_ffn"],),
                  p + "output_query.dense.weight": (Cq, c["qformer_ffn"]), p + "output_query.dense.bias": (Cq,),
                  p + "output_query.LayerNorm.weight": (Cq,), p + "output_query.LayerNorm.bias": (Cq,)})
    d = "language_model.model.decoder."
    s.update({"language_projection.weight": (Co, Cq), "language_projection.bias": (Co,), d + "embed_tokens.weight": (c["vocab"], Co),
              d + "embed_positions.weight": (c["max_positions"] + 2, Co), d + "final_layer_norm.weight": (Co,),
              d + "final_layer_norm.bias": (Co,)})
    for i in range(c["opt_layers"]):
        p = f"{d}layers.{i}."
        for n in ("k", "v", "q", "out"):
            s.update({p + f"self_attn.{n}_proj.weight": (Co, Co), p + f"self_attn.{n}_proj.bias": (Co,)})
        s.update({p + "self_attn_layer_norm.weight": (Co,), p + "self_attn_layer_norm.bias": (Co,), p + "fc1.weight": (c["opt_ffn"], Co),
                  p + "fc1.bias": (c["opt_ffn"],), p + "fc2.weight": (Co, c["opt_ffn"]), p + "fc2.bias": (Co,),
                  p + "final_layer_norm.weight": (Co,), p + "final_layer_norm.bias": (Co,)})
    return s


def default_init(cfg, seed=0, device="cpu", dtype=torch.float32):
    """seeded stand-in weights: LayerNorms at identity, small biases, linears ~ N(0, 1/fan_in), embeddings ~ N(0, 0.02^2)...
    drawn tensor by tensor on `device`"""
    g = torch.Generator(device=device).manual_seed(seed)
    out = {}
    for name, shape in param_shapes(cfg).items():
        if "LayerNorm" in name or "layer_norm" in name or "layernorm" in name:
            t = torch.ones(shape, device=device) if name.endswith("weight") else torch.zeros(shape, device=device)
            if name.endswith("weight"):
                t = t + 0.1 * torch.randn(shape, generator=g, device=device)
            else:
                t = t + 0.02 * torch.randn(shape, generator=g, device=device)
        elif name.endswith("bias"):
            t = 0.02 * torch.randn(shape, generator=g, device=device)
        elif "embed_tokens" in name:
            t = 0.05 * torch.randn(shape, generator=g, device=device)
        elif "embed" in name or "query_tokens" in name:
            t = 0.02 * torch.randn(shape, generator=g, device=device)
        else:
            fan_in = math.prod(shape[1:])
            t = torch.randn(shape, generator=g, device=device) * fan_in ** -0.5
        out[name] = t.to(dtype)
    return out


def _r(x, e16):
    return x.half().to(x.dtype) if e16 else x


def _ln(x, p, name, eps, e16):
    return _r(F.layer_norm(x, x.shape[-1:], p[name + ".weight"], p[name + ".bias"], eps), e16)


def _attn(q, k, v, heads, causal=False):
    T, C = q.shape
    d = C // heads
    q, k, v = (t.reshape(t.shape[0], heads, d).transpose(0, 1) for t in (q, k, v))
    s = q @ k.transpose(1, 2) * d ** -0.5
    if causal:
        s = s.masked_fill(torch.ones(T, k.shape[1], dtype=torch.bool, device=s.device).triu(1), float("-inf"))
    return (s.softmax(-1) @ v).transpose(0, 1).reshape(T, C)


def encode(p, cfg, pixel_values, e16=False):
    """pixel_values [1,3,S,S] -> (image_embeds [T,Cv], query_output [nq,Cq], language_model_inputs [nq,Co])"""
    c = cfg
    r = lambda x: _r(x, e16)
    W = {k: r(v) for k, v in p.items()} if e16 else p
    lin = lambda x, n, act=None: r((act or (lambda y: y))(F.linear(x, W[n + ".weight"], W[n + ".bias"])))
    gelu = lambda y: F.gelu(y)
    x = F.conv2d(r(pixel_values.to(W["vision_model.embeddings.patch_embedding.weight"].dtype)),
                 W["vision_model.embeddings.patch_embedding.weight"], W["vision_model.embeddings.patch_embedding.bias"], stride=c["patch"])
    x = r(x.flatten(2).transpose(1, 2)[0])
    x = torch.cat([p["vision_model.embeddings.class_embedding"][0], x], 0)
    x = r(x + p["vision_model.embeddings.position_embedding"][0])
    for i in range(c["vision_layers"]):
        pre = f"vision_model.encoder.layers.{i}."
        h = _ln(x, p, pre + "layer_norm1", 1e-6, e16)
        qkv = lin(h, pre + "self_attn.qkv")
        C = x.shape[1]
        a = r(_attn(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], c["vision_heads"]))
        x = r(F.linear(a, W[pre + "self_attn.projection.weight"], W[pre + "self_attn.projection.bias"]) + x)
        h = _ln(x, p, pre + "layer_norm2", 1e-6, e16)
        h = lin(h, pre + "mlp.fc1", gelu)
        x = r(F.linear(h, W[pre + "mlp.fc2.weight"], W[pre + "mlp.fc2.bias"]) + x)
    img = _ln(x, p, "vision_model.post_layernorm", 1e-6, e16)
    q = _ln(W["query_tokens"][0], p, "qformer.layernorm", 1e-12, e16)
    for i in range(c["qformer_layers"]):
        pre = f"qformer.encoder.layer.{i}."
        at = pre + "attention.attention."
        a = r(_attn(lin(q, at + "query"), lin(q, at + "key"), lin(q, at + "value"), c["qformer_heads"]))
        q = _ln(r(F.linear(a, W[pre + "attention.output.dense.weight"], W[pre + "attention.output.dense.bias"]) + q), p,
                pre + "attention.output.LayerNorm", 1e-12, e16)
        if i % c["cross_attention_frequency"] == 0:
            ca = pre + "crossattention.attention."
            a = r(_attn(lin(q, ca + "query"), lin(img, ca + "key"), lin(img, ca + "value"), c["qformer_heads"]))
            q = _ln(r(F.linear(a, W[pre + "crossattention.output.dense.weight"], W[pre + "crossattention.output.dense.bias"]) + q), p,
                    pre + "crossattention.output.LayerNorm", 1e-12, e16)
        h = lin(q, pre + "intermediate_query.dense", gelu)
        q = _ln(r(F.linear(h, W[pre + "output_query.dense.weight"], W[pre + "output_query.dense.bias"]) + q), p,
                pre + "output_query.LayerNorm", 1e-12, e16)
    return img, q, lin(q, "language_projection")


def decoder_logits(p, cfg, lm_inputs, ids, e16=False):
    """OPT over the prompt rows: lm_inputs [nq,Co] for rows < nq, embed_tokens[ids[t]] after; positions t + 2.  -> last-row logits [V]"""
    c = cfg
    r = lambda x: _r(x, e16)
    W = {k: r(v) for k, v in p.items()} if e16 else p
    d = "language_model.model.decoder."
    nq, T = c["num_query_tokens"], len(ids)
    tok = W[d + "embed_tokens.weight"]
    x = torch.cat([lm_inputs, tok[torch.as_tensor(ids[nq:], device=tok.device)]], 0)
    x = r(x + W[d + "embed_positions.weight"][2:T + 2])
    C = x.shape[1]
    for i in range(c["opt_layers"]):
        pre = f"{d}layers.{i}."
        h = _ln(x, p, pre + "self_attn_layer_norm", 1e-5, e16)
        qkv = [r(F.linear(h, W[pre + f"self_attn.{n}_proj.weight"], W[pre + f"self_attn.{n}_proj.bias"])) for n in "qkv"]
        a = r(_attn(*qkv, c["opt_heads"], causal=True))
        x = r(F.linear(a, W[pre + "self_attn.out_proj.weight"], W[pre + "self_attn.out_proj.bias"]) + x)
        h = _ln(x, p, pre + "final_layer_norm", 1e-5, e16)
        h = r(F.relu(F.linear(h, W[pre + "fc1.weight"], W[pre + "fc1.bias"])))
        x = r(F.linear(h, W[pre + "fc2.weight"], W[pre + "fc2.bias"]) + x)
    h = _ln(x[-1:], p, d + "final_layer_norm", 1e-5, e16)
    return (h @ tok.t())[0]


def generate(p, cfg, pixel_values, max_new_tokens=20, eos_token_id=None, e16=False, forced_ids=None):
    """-> dict(image_embeds, query_output, language_model_inputs, logits [n, V] (last row of every step), ids [33 + n] list).
    eos_token_id=None: the config's eos; -1: none.  forced_ids: teacher forcing (step s appends forced_ids[s])."""
    eos = cfg["eos_token_id"] if eos_token_id is None else eos_token_id
    img, q, lm = encode(p, cfg, pixel_values, e16)
    ids = [cfg["image_token_index"]] * cfg["num_query_tokens"] + [cfg["bos_token_id"]]
    logits = []
    for s in range(max_new_tokens):
        lg = decoder_logits(p, cfg, lm, ids, e16)
        logits.append(lg)
        tok = int(forced_ids[s]) if forced_ids is not None else int(lg.argmax())
        ids.append(tok)
        if eos >= 0 and tok == eos and forced_ids is None:
            break
    return dict(image_embeds=img, query_output=q, language_model_inputs=lm, logits=torch.stack(logits), ids=ids)
