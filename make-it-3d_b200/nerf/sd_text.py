"""B3' seam: the Stable Diffusion text encoder (`CLIPTextModel.from_pretrained(model_key, subfolder="text_encoder")`, nerf/sd.py:42)
on libmi3d.so.

`TextEncoder(device, cfg=None, state_dict=None, graph_replay=True, max_batch=2)` runs OpenCLIP ViT-H/14's text tower as SD-2.x ships it
(23 layers, width 1024, exact GELU; `sd2_text_cfg()`) or OpenAI CLIP ViT-L/14's text tower as SD-1.x ships it (12 layers, width 768,
quick-GELU; `sd15_text_cfg()`) in the engine of csrc/sd_text_engine.cu (tile GEMM with the activation in its epilogue, materialised
causal attention, fused memory-bound kernels); there is no CPU or eager-PyTorch fallback.  `cfg["hidden_act"]` takes transformers'
names, "gelu" (the default) or "quick_gelu"; a state dict does not record it, so `cfg_from_state_dict` takes it as an argument.

* Weights are named like transformers' `CLIPTextModel.state_dict()`, so `load_state_dict(text_encoder.state_dict())` of a diffusers SD-2
  checkpoint loads directly (`text_model.embeddings.position_ids` is ignored when present).  Each tensor passes through the device on
  its way into the engine's fp16 copy; no fp32 copy of the 1.36 GB of weights is kept.  Without a state_dict the weights are seeded
  random tensors.
* `encoder(input_ids)` -> `(last_hidden_state,)`: int64 CUDA ids `[B, 77]` -> fp32 `[B, 77, 1024]`, no gradient (the encoder is frozen),
  so the reference's `self.text_encoder(ids)[0]` works unchanged.
"""
import ctypes as C

import torch

from .. import _lib as L


class SdTextCfg(C.Structure):
    _fields_ = [("width", C.c_int), ("layers", C.c_int), ("heads", C.c_int), ("context_len", C.c_int), ("vocab", C.c_int),
                ("max_batch", C.c_int)]


ACTS = {"gelu": 0, "quick_gelu": 1}     # transformers' hidden_act -> the act argument of mi3d_sd_text_act_create


def sd2_text_cfg():
    """SD-2.0-base / 2.1-base / 2.1 text_encoder/config.json"""
    return dict(width=1024, layers=23, heads=16, context_len=77, vocab=49408, hidden_act="gelu")


def sd15_text_cfg():
    """SD-1.5 (and every SD-1.x) text_encoder/config.json: OpenAI CLIP ViT-L/14's text tower"""
    return dict(width=768, layers=12, heads=12, context_len=77, vocab=49408, hidden_act="quick_gelu")


def cfg_from_state_dict(state_dict, hidden_act="gelu"):
    """the encoder's shape read off a CLIPTextModel state_dict (head_dim 64, as in every SD-1.x / SD-2.x checkpoint); the activation
    is not in the state dict: "gelu" for SD-2.x, "quick_gelu" for SD-1.x"""
    if hidden_act not in ACTS:
        raise L.Mi3dError(f"hidden_act must be one of {sorted(ACTS)}; got {hidden_act!r}")
    tok = state_dict["text_model.embeddings.token_embedding.weight"]
    layers = {k.split(".")[3] for k in state_dict if k.startswith("text_model.encoder.layers.")}
    return dict(width=tok.shape[1], layers=len(layers), heads=tok.shape[1] // 64,
                context_len=state_dict["text_model.embeddings.position_embedding.weight"].shape[0], vocab=tok.shape[0],
                hidden_act=hidden_act)


class TextEncoder(L.Engine):
    def __init__(self, device, cfg=None, state_dict=None, graph_replay=True, max_batch=2):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise L.Mi3dError("the SD text encoder runs on sm_90a only; there is no CPU fallback")
        self.cfg = dict(cfg or sd2_text_cfg())
        act = self.cfg.setdefault("hidden_act", "gelu")
        if act not in ACTS:
            raise L.Mi3dError(f"hidden_act must be one of {sorted(ACTS)}; got {act!r}")
        self.struct = SdTextCfg(*(int(self.cfg[k]) for k, _ in SdTextCfg._fields_[:-1]), int(max_batch))
        self.act = ACTS[act]
        super().__init__("sd_text_act", (C.byref(self.struct), C.c_int(self.act)), self.device, graph_replay,
                         f"SD text encoder configuration {self.cfg} with max_batch={max_batch}")
        self.load_state_dict(state_dict if state_dict is not None else _default_state(self.names, self.shapes))

    @property
    def max_batch(self):
        return self.struct.max_batch

    def load_state_dict(self, state_dict):
        """tensors named like transformers' CLIPTextModel.state_dict() (any float dtype, any device); every entry is required, and no
        other entry but `text_model.embeddings.position_ids` is accepted"""
        return self.load_strict(state_dict, lambda k: k.endswith("position_ids"))

    def __call__(self, input_ids):
        """input_ids int64 CUDA [B, context_len] -> (last_hidden_state fp32 [B, context_len, width],)"""
        T, V = self.cfg["context_len"], self.cfg["vocab"]
        if not torch.is_tensor(input_ids) or input_ids.dtype != torch.long:
            raise L.Mi3dError(f"the SD text encoder takes int64 token ids [B,{T}]")
        L.require_cuda(input_ids)
        if input_ids.dim() != 2 or input_ids.shape[1] != T or not 1 <= input_ids.shape[0] <= self.max_batch:
            raise L.Mi3dError(f"the SD text encoder takes ids [B,{T}] with 1 <= B <= {self.max_batch}; got {tuple(input_ids.shape)}")
        if bool(((input_ids < 0) | (input_ids >= V)).any()):
            raise L.Mi3dError(f"token ids must lie in [0, {V})")
        ids = input_ids.contiguous()
        B = ids.shape[0]
        out = torch.empty(B, T, self.cfg["width"], dtype=torch.float32, device=ids.device)
        with self.on_stream():
            L.check(L.lib().mi3d_sd_text_encode(self.h, L.ptr(ids), C.c_int(B), L.ptr(out), L.stream()), "sd_text_encode")
        return (out,)


def _default_state(names, shapes, seed=0):
    """seeded stand-in weights (no SD-2 weights exist offline), CLIP's initialisers in spirit"""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in zip(names, shapes):
        if "layer_norm" in name:
            out[name] = torch.ones(shape) if name.endswith("weight") else torch.zeros(shape)
        elif name.endswith("bias"):
            out[name] = torch.zeros(shape)
        elif "embedding" in name:
            out[name] = torch.randn(shape, generator=g) * (0.02 if "token" in name else 0.01)
        else:
            out[name] = torch.randn(shape, generator=g) * shape[1] ** -0.5
    return out
