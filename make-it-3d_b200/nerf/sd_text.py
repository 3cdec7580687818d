"""B3' seam: the Stable Diffusion 2 text encoder (`CLIPTextModel.from_pretrained(model_key, subfolder="text_encoder")`, nerf/sd.py:42)
on libmi3d.so.

`TextEncoder(device, cfg=None, state_dict=None, graph_replay=True, max_batch=2)` runs OpenCLIP ViT-H/14's text tower as SD-2.x ships it
(23 layers, width 1024) in the engine of csrc/sd_text_engine.cu (tile GEMM with an exact-GELU epilogue, materialised causal attention,
fused memory-bound kernels); there is no CPU or eager-PyTorch fallback.

* Weights are named like transformers' `CLIPTextModel.state_dict()`, so `load_state_dict(text_encoder.state_dict())` of a diffusers SD-2
  checkpoint loads directly (`text_model.embeddings.position_ids` is ignored when present).  Each tensor passes through the device on
  its way into the engine's fp16 copy; no fp32 copy of the 1.36 GB of weights is kept.  Without a state_dict the weights are seeded
  random tensors.
* `encoder(input_ids)` -> `(last_hidden_state,)`: int64 CUDA ids `[B, 77]` -> fp32 `[B, 77, 1024]`, no gradient (the encoder is frozen),
  so the reference's `self.text_encoder(ids)[0]` works unchanged.
"""
import contextlib
import ctypes as C

import torch

from .. import _lib as L


class SdTextCfg(C.Structure):
    _fields_ = [("width", C.c_int), ("layers", C.c_int), ("heads", C.c_int), ("context_len", C.c_int), ("vocab", C.c_int),
                ("max_batch", C.c_int)]


def sd2_text_cfg():
    """SD-2.0-base / 2.1-base / 2.1 text_encoder/config.json"""
    return dict(width=1024, layers=23, heads=16, context_len=77, vocab=49408)


def cfg_from_state_dict(state_dict):
    """the encoder's shape read off a CLIPTextModel state_dict (head_dim 64, as in every SD-2.x checkpoint)"""
    tok = state_dict["text_model.embeddings.token_embedding.weight"]
    layers = {k.split(".")[3] for k in state_dict if k.startswith("text_model.encoder.layers.")}
    return dict(width=tok.shape[1], layers=len(layers), heads=tok.shape[1] // 64,
                context_len=state_dict["text_model.embeddings.position_embedding.weight"].shape[0], vocab=tok.shape[0])


class TextEncoder:
    def __init__(self, device, cfg=None, state_dict=None, graph_replay=True, max_batch=2):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise L.Mi3dError("the SD-2 text encoder runs on sm_90a only; there is no CPU fallback")
        self.cfg = dict(cfg or sd2_text_cfg())
        lib = L.lib()
        lib.mi3d_sd_text_workspace_bytes.restype = C.c_size_t
        lib.mi3d_sd_text_create.restype = C.c_void_p
        lib.mi3d_sd_text_param_name.restype = C.c_char_p
        self.struct = SdTextCfg(*(int(self.cfg[k]) for k, _ in SdTextCfg._fields_[:-1]), int(max_batch))
        nbytes = lib.mi3d_sd_text_workspace_bytes(C.byref(self.struct))
        if nbytes == 0:
            raise L.Mi3dError(f"unsupported SD text encoder configuration {self.cfg} with max_batch={max_batch}")
        self.workspace = torch.zeros(nbytes, dtype=torch.uint8, device=self.device)
        h = lib.mi3d_sd_text_create(C.byref(self.struct), L.ptr(self.workspace), C.c_size_t(nbytes))
        if not h:
            raise L.Mi3dError("mi3d_sd_text_create failed (TMA descriptor encoding error)")
        self.h = C.c_void_p(h)
        self.names, self.shapes = [], []
        shp = (C.c_int * 4)()
        for i in range(lib.mi3d_sd_text_num_params(self.h)):
            self.names.append(lib.mi3d_sd_text_param_name(self.h, C.c_int(i)).decode())
            r = lib.mi3d_sd_text_param_shape(self.h, C.c_int(i), shp)
            self.shapes.append(tuple(shp[k] for k in range(r)))
        # as in the other engines: the launch list runs on an engine-owned stream so that it can replay as a CUDA graph (torch's legacy
        # default stream cannot be captured); graph_replay=False keeps plain launches on the caller's stream
        self.stream = torch.cuda.Stream(self.device) if graph_replay else None
        L.check(lib.mi3d_sd_text_set_graph_replay(self.h, C.c_int(1 if graph_replay else 0)), "sd_text_set_graph_replay")
        self.load_state_dict(state_dict if state_dict is not None else _default_state(self.names, self.shapes))

    @property
    def max_batch(self):
        return self.struct.max_batch

    def graph_replays(self):
        return int(L.lib().mi3d_sd_text_graph_replays(self.h))

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

    def load_state_dict(self, state_dict):
        """tensors named like transformers' CLIPTextModel.state_dict() (any float dtype, any device); every entry is required, and no
        other entry but `text_model.embeddings.position_ids` is accepted"""
        missing = [n for n in self.names if n not in state_dict]
        unexpected = [k for k in state_dict if k not in self.names and not k.endswith("position_ids")]
        if missing or unexpected:
            raise L.Mi3dError(f"SD text encoder state_dict mismatch: missing {missing[:4]}, unexpected {unexpected[:4]}")
        lib = L.lib()
        for i, (name, shape) in enumerate(zip(self.names, self.shapes)):
            t = state_dict[name].detach()
            if tuple(t.shape) != shape:
                raise L.Mi3dError(f"{name}: shape {tuple(t.shape)}, expected {shape}")
            src = t.to(self.device, torch.float32).contiguous()
            # the caching allocator reuses src's memory only after the load kernel queued behind it on this stream
            L.check(lib.mi3d_sd_text_load_param(self.h, C.c_int(i), L.ptr(src), L.stream()), f"sd_text_load_param({name})")
        torch.cuda.synchronize(self.device)
        return self

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

    def __del__(self):
        try:
            if getattr(self, "h", None):
                L.lib().mi3d_sd_text_destroy(self.h)
        except Exception:
            pass


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
