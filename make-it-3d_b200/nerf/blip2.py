"""B9 seam: the BLIP-2 captioner (`Blip2ForConditionalGeneration.from_pretrained("Salesforce/blip2-opt-2.7b", torch_dtype=float16)`,
main.py:158-172) on libmi3d.so.

`Blip2ForConditionalGeneration.from_pretrained(local_dir)` or `Blip2ForConditionalGeneration(cfg=None, state_dict=None)` runs EVA
ViT-g/14, the Q-Former and a greedy OPT-2.7B decode in the engine of csrc/blip2_engine.cu (tile GEMM for the encoders, the
weight-streaming GEMM for the decoder, the greedy step on the device); there is no CPU or eager-PyTorch fallback.

* Weights carry transformers' state_dict names.  Every name the forward reads is required and no other is accepted, except
  `language_model.lm_head.weight`, which must equal `embed_tokens` (the checkpoint ties them).  Without weights the model runs on seeded
  stand-ins.
* `generate(pixel_values=..., max_new_tokens=20, eos_token_id=None)` -> int64 ids `[1, 33 + n]` with the prompt ids included, as
  transformers returns them, so `processor.batch_decode(out, skip_special_tokens=True)` works unchanged.
* The image processor and the BPE detokenizer stay the caller's (they need the checkpoint's files).
"""
import contextlib
import ctypes as C
import glob
import json
import os

import torch

from .. import _lib as L

ROWS = 64


class Blip2Cfg(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("image_size", "patch", "vision_width", "vision_layers", "vision_heads", "vision_mlp", "qformer_width",
                                       "qformer_layers", "qformer_heads", "qformer_ffn", "cross_attention_frequency", "num_query_tokens",
                                       "opt_width", "opt_layers", "opt_heads", "opt_ffn", "vocab", "max_positions", "image_token_index",
                                       "bos_token_id", "eos_token_id")]


def blip2_opt_27b_cfg():
    """Salesforce/blip2-opt-2.7b's config.json"""
    return dict(image_size=224, patch=14, vision_width=1408, vision_layers=39, vision_heads=16, vision_mlp=6144,
                qformer_width=768, qformer_layers=12, qformer_heads=12, qformer_ffn=3072, cross_attention_frequency=2,
                num_query_tokens=32, opt_width=2560, opt_layers=32, opt_heads=32, opt_ffn=10240, vocab=50272, max_positions=2048,
                image_token_index=50265, bos_token_id=2, eos_token_id=50118)


def cfg_from_config_json(conf):
    """the engine's cfg from a Blip2Config dict (config.json); only blip2-opt (OPT decoder, pre-LN, ReLU) is accepted"""
    if conf.get("model_type") != "blip-2":
        raise L.Mi3dError(f"not a BLIP-2 config (model_type {conf.get('model_type')!r})")
    v, q, t = conf.get("vision_config", {}), conf.get("qformer_config", {}), conf.get("text_config", {})
    if t.get("model_type", "opt") != "opt" or not t.get("do_layer_norm_before", True) or t.get("activation_function", "relu") != "relu" \
            or t.get("word_embed_proj_dim", t.get("hidden_size")) != t.get("hidden_size") or q.get("use_qformer_text_input", False):
        raise L.Mi3dError("only BLIP-2 with an OPT decoder (pre-LN, ReLU, no word-embedding projection) is supported")
    if v.get("hidden_act", "gelu") != "gelu" or q.get("hidden_act", "gelu") != "gelu" or not v.get("qkv_bias", True):
        raise L.Mi3dError("unsupported BLIP-2 vision / Q-Former activation or bias settings")
    d = blip2_opt_27b_cfg()
    get = lambda src, k, default: int(src.get(k, default))
    return dict(image_size=get(v, "image_size", 224), patch=get(v, "patch_size", 14), vision_width=get(v, "hidden_size", 1408),
                vision_layers=get(v, "num_hidden_layers", 39), vision_heads=get(v, "num_attention_heads", 16),
                vision_mlp=get(v, "intermediate_size", 6144), qformer_width=get(q, "hidden_size", 768),
                qformer_layers=get(q, "num_hidden_layers", 12), qformer_heads=get(q, "num_attention_heads", 12),
                qformer_ffn=get(q, "intermediate_size", 3072), cross_attention_frequency=get(q, "cross_attention_frequency", 2),
                num_query_tokens=get(conf, "num_query_tokens", 32), opt_width=get(t, "hidden_size", d["opt_width"]),
                opt_layers=get(t, "num_hidden_layers", d["opt_layers"]), opt_heads=get(t, "num_attention_heads", d["opt_heads"]),
                opt_ffn=get(t, "ffn_dim", d["opt_ffn"]), vocab=get(t, "vocab_size", d["vocab"]),
                max_positions=get(t, "max_position_embeddings", 2048),
                image_token_index=int(conf.get("image_token_index", conf.get("image_token_id", d["image_token_index"]))),
                bos_token_id=get(t, "bos_token_id", 2), eos_token_id=get(t, "eos_token_id", d["eos_token_id"]))


class Blip2ForConditionalGeneration:
    def __init__(self, cfg=None, state_dict=None, device="cuda", graph_replay=True):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise L.Mi3dError("the BLIP-2 captioner runs on sm_90a only; there is no CPU fallback")
        self.cfg = dict(cfg or blip2_opt_27b_cfg())
        lib = L.lib()
        lib.mi3d_blip2_workspace_bytes.restype = C.c_size_t
        lib.mi3d_blip2_create.restype = C.c_void_p
        lib.mi3d_blip2_param_name.restype = C.c_char_p
        self.struct = Blip2Cfg(*(int(self.cfg[k]) for k, _ in Blip2Cfg._fields_))
        nbytes = lib.mi3d_blip2_workspace_bytes(C.byref(self.struct))
        if nbytes == 0:
            raise L.Mi3dError(f"unsupported BLIP-2 configuration {self.cfg}")
        self.workspace_bytes = nbytes
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        h = lib.mi3d_blip2_create(C.byref(self.struct), L.ptr(self.workspace), C.c_size_t(nbytes))
        if not h:
            raise L.Mi3dError("mi3d_blip2_create failed (TMA descriptor encoding error)")
        self.h = C.c_void_p(h)
        self.names, self.shapes = [], []
        shp = (C.c_int * 4)()
        for i in range(lib.mi3d_blip2_num_params(self.h)):
            self.names.append(lib.mi3d_blip2_param_name(self.h, C.c_int(i)).decode())
            r = lib.mi3d_blip2_param_shape(self.h, C.c_int(i), shp)
            self.shapes.append(tuple(shp[k] for k in range(r)))
        # as in the other engines: an engine-owned stream so the launch lists can replay as CUDA graphs
        self.stream = torch.cuda.Stream(self.device) if graph_replay else None
        L.check(lib.mi3d_blip2_set_graph_replay(self.h, C.c_int(1 if graph_replay else 0)), "blip2_set_graph_replay")
        self.load_state_dict(state_dict if state_dict is not None else _default_state(self.names, self.shapes, self.device))

    # ------------------------------------------------------------------ loading
    @classmethod
    def from_pretrained(cls, local_dir, torch_dtype=None, **kwargs):
        """a local checkpoint directory (config.json + model.safetensors or sharded *.safetensors with their index); never the network"""
        if not os.path.isdir(local_dir):
            raise L.Mi3dError(f"{local_dir} is not a local checkpoint directory (this loader never downloads)")
        with open(os.path.join(local_dir, "config.json")) as f:
            cfg = cfg_from_config_json(json.load(f))
        from safetensors.torch import load_file
        idx = os.path.join(local_dir, "model.safetensors.index.json")
        if os.path.exists(idx):
            with open(idx) as f:
                files = sorted(set(json.load(f)["weight_map"].values()))
        else:
            files = sorted(os.path.basename(p) for p in glob.glob(os.path.join(local_dir, "*.safetensors")))
        if not files:
            raise L.Mi3dError(f"no *.safetensors weights in {local_dir}")
        state = {}
        for fn in files:
            state.update(load_file(os.path.join(local_dir, fn)))
        return cls(cfg=cfg, state_dict=state, **kwargs)

    def load_state_dict(self, state_dict):
        tied = "language_model.lm_head.weight"
        emb = "language_model.model.decoder.embed_tokens.weight"
        missing = [n for n in self.names if n not in state_dict]
        unexpected = [k for k in state_dict if k not in self.names and k != tied]
        if missing or unexpected:
            raise L.Mi3dError(f"BLIP-2 state_dict mismatch: missing {missing[:4]}, unexpected {unexpected[:4]}")
        if tied in state_dict:
            a, b = state_dict[tied], state_dict[emb]
            if a.shape != b.shape or not torch.equal(a.detach().to(b.device, b.dtype), b.detach()):
                raise L.Mi3dError(f"{tied} must equal {emb} (lm_head is tied to the token embedding)")
        lib = L.lib()
        for i, (name, shape) in enumerate(zip(self.names, self.shapes)):
            t = state_dict[name].detach()
            if tuple(t.shape) != shape:
                raise L.Mi3dError(f"{name}: shape {tuple(t.shape)}, expected {shape}")
            src = t.to(self.device, torch.float32).contiguous()
            L.check(lib.mi3d_blip2_load_param(self.h, C.c_int(i), L.ptr(src), L.stream()), f"blip2_load_param({name})")
        torch.cuda.synchronize(self.device)
        return self

    def to(self, *args, **kwargs):
        return self

    def eval(self):
        return self

    def graph_replays(self):
        return int(L.lib().mi3d_blip2_graph_replays(self.h))

    @contextlib.contextmanager
    def on_stream(self):
        if self.stream is None:
            yield
            return
        cur = torch.cuda.current_stream()
        self.stream.wait_stream(cur)
        with torch.cuda.stream(self.stream):
            yield
        cur.wait_stream(self.stream)

    # ------------------------------------------------------------------ running
    def _pixels(self, pixel_values):
        S = self.cfg["image_size"]
        if not torch.is_tensor(pixel_values) or not pixel_values.is_floating_point():
            raise L.Mi3dError("pixel_values must be a float tensor")
        L.require_cuda(pixel_values)
        if pixel_values.dim() != 4 or pixel_values.shape[0] != 1:
            raise L.Mi3dError(f"batch size 1 only; got pixel_values {tuple(pixel_values.shape)}")
        if tuple(pixel_values.shape[1:]) != (3, S, S):
            raise L.Mi3dError(f"pixel_values must be [1,3,{S},{S}]; got {tuple(pixel_values.shape)}")
        return pixel_values.to(torch.float32).contiguous()

    def encode(self, pixel_values):
        """pixel_values [1,3,S,S] -> language_model_inputs fp32 [num_query_tokens, opt_width]"""
        px = self._pixels(pixel_values)
        out = torch.empty(self.cfg["num_query_tokens"], self.cfg["opt_width"], dtype=torch.float32, device=self.device)
        with self.on_stream():
            L.check(L.lib().mi3d_blip2_encode(self.h, L.ptr(px), L.ptr(out), L.stream()), "blip2_encode")
        return out

    def taps(self):
        """the last call's image_embeds, query_output and language_model_inputs (fp32)"""
        c = self.cfg
        Tv = (c["image_size"] // c["patch"]) ** 2 + 1
        shapes = {"image_embeds": (Tv, c["vision_width"]), "query_output": (c["num_query_tokens"], c["qformer_width"]),
                  "language_model_inputs": (c["num_query_tokens"], c["opt_width"])}
        out = {}
        with self.on_stream():
            for name, shape in shapes.items():
                t = torch.empty(shape, dtype=torch.float32, device=self.device)
                L.check(L.lib().mi3d_blip2_tap(self.h, name.encode(), L.ptr(t), L.stream()), f"blip2_tap({name})")
                out[name] = t
        return out

    def max_new_tokens_limit(self):
        return ROWS - self.cfg["num_query_tokens"] - 1

    def generate(self, pixel_values=None, input_ids=None, attention_mask=None, inputs_embeds=None, interpolate_pos_encoding=False,
                 max_new_tokens=20, eos_token_id=None, forced_ids=None, return_logits=False, **kwargs):
        """greedy caption of one image -> int64 ids [1, num_query_tokens + 1 + n] (prompt included).  forced_ids (teacher forcing) and
        return_logits=True (-> (ids, last-row logits [n, vocab])) serve the parity tests."""
        if input_ids is not None or attention_mask is not None or inputs_embeds is not None:
            raise L.Mi3dError("text-conditioned captioning (input_ids / attention_mask / inputs_embeds) is not supported")
        if interpolate_pos_encoding:
            raise L.Mi3dError("interpolate_pos_encoding is not supported (one image size)")
        # greedy only: do_sample=False / num_beams=1 / num_return_sequences=1 are accepted, any other generation argument raises
        greedy = {"do_sample": False, "num_beams": 1, "num_return_sequences": 1}
        if any(k not in greedy or v != greedy[k] for k, v in kwargs.items()):
            raise L.Mi3dError(f"only greedy decoding is supported; got {sorted(kwargs)}")
        n = int(max_new_tokens)
        if not 1 <= n <= self.max_new_tokens_limit():
            raise L.Mi3dError(f"max_new_tokens must lie in 1..{self.max_new_tokens_limit()}")
        eos = self.cfg["eos_token_id"] if eos_token_id is None else int(eos_token_id)
        px = self._pixels(pixel_values)
        fo = None
        if forced_ids is not None:
            fo = torch.as_tensor(forced_ids, dtype=torch.long, device=self.device).reshape(-1)[:n].contiguous()
            if fo.numel() != n:
                raise L.Mi3dError(f"forced_ids needs {n} ids")
        ids = torch.empty(ROWS, dtype=torch.long, device=self.device)
        count = torch.empty(1, dtype=torch.int32, device=self.device)
        logits = torch.empty(n, self.cfg["vocab"], dtype=torch.float32, device=self.device) if return_logits else None
        with self.on_stream():
            L.check(L.lib().mi3d_blip2_generate(self.h, L.ptr(px), C.c_int(n), C.c_longlong(eos), L.ptr(fo), L.ptr(ids), L.ptr(count),
                                                L.ptr(logits), L.stream()), "blip2_generate")
        out = ids[: int(count.item())][None].clone()
        return (out, logits) if return_logits else out

    def __del__(self):
        try:
            if getattr(self, "h", None):
                L.lib().mi3d_blip2_destroy(self.h)
        except Exception:
            pass


def _default_state(names, shapes, device, seed=0):
    """seeded stand-in weights (no BLIP-2 checkpoint exists offline), drawn tensor by tensor on the device: LayerNorms near identity,
    small biases, linears ~ N(0, 1 / fan_in), embeddings ~ N(0, 0.02^2)"""
    g = torch.Generator(device=device).manual_seed(seed)
    out = {}
    for name, shape in zip(names, shapes):
        r = torch.randn(shape, generator=g, device=device)
        if "LayerNorm" in name or "layer_norm" in name or "layernorm" in name:
            out[name] = 1 + 0.1 * r if name.endswith("weight") else 0.02 * r
        elif name.endswith("bias"):
            out[name] = 0.02 * r
        elif "embed_tokens" in name:
            out[name] = 0.05 * r
        elif "embed" in name or "query_tokens" in name:
            out[name] = 0.02 * r
        else:
            out[name] = r * (r[0].numel() ** -0.5)
    return out


def caption(model, processor, image_pil):
    """main.py:163-172 end to end: processor -> generate -> decode -> the reference's string replacements"""
    inputs = processor(image_pil, return_tensors="pt").to(model.device, torch.float16)
    out = model.generate(**inputs)
    text = processor.batch_decode(out, skip_special_tokens=True)[0].strip()
    text = text.replace("there is ", "")
    text = text.replace("close up", "photo")
    for d in ["black background", "white background"]:
        if d in text:
            text = text.replace(d, "ground")
    return text
