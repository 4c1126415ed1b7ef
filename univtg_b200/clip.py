"""CLIP feature extraction on the GPU: the run-on-your-own-video front end of UniVTG.

The reference extracts a video's features with OpenAI CLIP ViT-B/32 one frame per encode_image call
(run_on_video/video_extractor.py:31-63) and the query's with encode_text (txt2clip, :79-87), then normalises them and adds the
TEF columns in main_gradio.load_data (main_gradio.py:58-80).  This module does the same work through the CUDA library
(include/univtg_b200.h, univtg_clip_*):

    enc = ClipEncoder.from_state_dict(torch.load("ViT-B-32.pt").state_dict(), operand_format="fp16").cuda()
    vid = enc.encode_image(frames)                       # uint8 [T, 224, 224, 3] (ffmpeg rgb24) -> [T, 512]
    txt, mask = enc.text_features(tokens)                # clip.tokenize ids [1, 77] -> [1, Lq, 512] valid rows
    inputs, targets = grounding_inputs(vid, txt[0][mask[0] > 0])
    out = model(**inputs); windows = postproc.decode_mr(out, targets, None)

Only ViT CLIP state dicts are supported (ResNet CLIP raises NotImplementedError).  Inference only; there is no CPU or eager
fallback.  Tokenisation stays with clip.tokenize.
"""
import ctypes

import torch
from torch import nn

from . import _lib

_INT_ENTRIES = ("input_resolution", "context_length", "vocab_size")  # dropped as the reference's build_model drops them
_FORMATS = {"fp16": 0, "bf16": 1}
CONFIG_FIELDS = ("embed_dim", "vision_width", "vision_layers", "patch_size", "image_resolution", "text_width", "text_layers",
                 "context_length", "vocab_size")


def config_from_state_dict(sd):
    """The architecture the reference's build_model(state_dict) infers (run_on_video/clip/model.py:395-418), ViT only."""
    if "visual.proj" not in sd:
        if any(k.startswith("visual.layer1.") for k in sd):
            raise NotImplementedError("ClipEncoder: this is a ResNet CLIP state dict (visual.layer1.*, ModifiedResNet); only ViT CLIP "
                                      "(visual.conv1 + visual.proj) is supported")
        raise ValueError("ClipEncoder: not a CLIP state dict (no visual.proj)")
    conv = sd["visual.conv1.weight"]
    grid = round((sd["visual.positional_embedding"].shape[0] - 1) ** 0.5)
    return dict(embed_dim=sd["text_projection"].shape[1], vision_width=conv.shape[0],
                vision_layers=len([k for k in sd if k.startswith("visual.") and k.endswith(".attn.in_proj_weight")]),
                patch_size=conv.shape[-1], image_resolution=conv.shape[-1] * grid, text_width=sd["ln_final.weight"].shape[0],
                text_layers=len(set(k.split(".")[2] for k in sd if k.startswith("transformer.resblocks"))),
                context_length=sd["positional_embedding"].shape[0], vocab_size=sd["token_embedding.weight"].shape[0])


class _Params(nn.Module):
    def __init__(self, **shapes):
        super().__init__()
        for name, shape in shapes.items():
            self.register_parameter(name, nn.Parameter(torch.zeros(shape)))


class _Attn(nn.Module):  # keys of nn.MultiheadAttention
    def __init__(self, W):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.zeros(3 * W, W))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * W))
        self.out_proj = _Params(weight=(W, W), bias=(W,))


class _Block(nn.Module):  # ResidualAttentionBlock (model.py:167-188)
    def __init__(self, W):
        super().__init__()
        self.attn = _Attn(W)
        self.ln_1 = _Params(weight=(W,), bias=(W,))
        self.mlp = nn.Module()
        self.mlp.c_fc = _Params(weight=(4 * W, W), bias=(4 * W,))
        self.mlp.c_proj = _Params(weight=(W, 4 * W), bias=(W,))
        self.ln_2 = _Params(weight=(W,), bias=(W,))

    def abi_params(self):
        a, m = self.attn, self.mlp
        return [a.in_proj_weight, a.in_proj_bias, a.out_proj.weight, a.out_proj.bias, self.ln_1.weight, self.ln_1.bias, m.c_fc.weight,
                m.c_fc.bias, m.c_proj.weight, m.c_proj.bias, self.ln_2.weight, self.ln_2.bias]


class _Transformer(nn.Module):
    def __init__(self, W, n):
        super().__init__()
        self.resblocks = nn.ModuleList([_Block(W) for _ in range(n)])


class _Visual(nn.Module):  # VisualTransformer (model.py:202-217)
    def __init__(self, c):
        super().__init__()
        W, P, g = c["vision_width"], c["patch_size"], c["image_resolution"] // c["patch_size"]
        self.conv1 = _Params(weight=(W, 3, P, P))
        self.class_embedding = nn.Parameter(torch.zeros(W))
        self.positional_embedding = nn.Parameter(torch.zeros(g * g + 1, W))
        self.ln_pre = _Params(weight=(W,), bias=(W,))
        self.transformer = _Transformer(W, c["vision_layers"])
        self.ln_post = _Params(weight=(W,), bias=(W,))
        self.proj = nn.Parameter(torch.zeros(W, c["embed_dim"]))


class ClipEncoder(nn.Module):
    """Inference-only ViT CLIP with the reference's parameter names (load_state_dict(sd, strict=True) takes an OpenAI CLIP state
    dict; its integer entries are dropped).  Every matrix product, LayerNorm and attention runs in the CUDA library."""

    def __init__(self, config, operand_format="fp16"):
        super().__init__()
        if operand_format not in _FORMATS:
            raise ValueError(f"ClipEncoder: operand_format={operand_format!r} is not supported; use 'fp16' or 'bf16' "
                             "(the split-fp16 mode 'fp16x3' exists for the grounding model only)")
        self.config = {k: int(config[k]) for k in CONFIG_FIELDS}
        self.operand_format = operand_format
        c = self.config
        self.visual = _Visual(c)
        self.transformer = _Transformer(c["text_width"], c["text_layers"])
        self.token_embedding = _Params(weight=(c["vocab_size"], c["text_width"]))
        self.positional_embedding = nn.Parameter(torch.zeros(c["context_length"], c["text_width"]))
        self.ln_final = _Params(weight=(c["text_width"],), bias=(c["text_width"],))
        self.text_projection = nn.Parameter(torch.zeros(c["text_width"], c["embed_dim"]))
        self.logit_scale = nn.Parameter(torch.zeros(()))  # kept for strict loading; feature extraction does not use it
        self._packed = None
        self._packed_key = None
        self._ws = None

    @classmethod
    def from_state_dict(cls, sd, operand_format="fp16"):
        """Build from a CLIP state dict (architecture inferred as build_model does), in the state dict's dtype, in eval mode."""
        m = cls(config_from_state_dict(sd), operand_format)
        dtype = sd["visual.conv1.weight"].dtype
        if dtype in (torch.float16, torch.float32):
            m.to(dtype)
        m.load_state_dict(sd, strict=True)
        return m.eval()

    def load_state_dict(self, state_dict, strict=True, **kw):
        return super().load_state_dict({k: v for k, v in state_dict.items() if k not in _INT_ENTRIES}, strict=strict, **kw)

    # ---- C ABI plumbing ----
    def _cfg(self):
        return _lib.ClipConfig(*[self.config[k] for k in CONFIG_FIELDS], _FORMATS[self.operand_format])

    def _abi_params(self):
        v = self.visual
        out = [v.conv1.weight, v.class_embedding, v.positional_embedding, v.ln_pre.weight, v.ln_pre.bias]
        for b in v.transformer.resblocks:
            out += b.abi_params()
        out += [v.ln_post.weight, v.ln_post.bias, v.proj, self.token_embedding.weight, self.positional_embedding]
        for b in self.transformer.resblocks:
            out += b.abi_params()
        return out + [self.ln_final.weight, self.ln_final.bias, self.text_projection]

    def _device(self):
        dev = self.text_projection.device
        if dev.type != "cuda":
            raise RuntimeError("ClipEncoder: the parameters are on the CPU; the CLIP encoder runs on a CUDA device only (call .cuda())")
        return dev

    def _check_mode(self):
        if self.training:
            raise RuntimeError("ClipEncoder is inference-only (training mode is not supported); call .eval()")

    def _ensure_packed(self):
        dev = self._device()
        params = self._abi_params()
        dtype = params[0].dtype
        if dtype not in (torch.float32, torch.float16) or any(p.dtype != dtype for p in params):
            raise TypeError(f"ClipEncoder: parameters must all be float32 or all float16, got {sorted({str(p.dtype) for p in params})}")
        key = (dev.index, self.operand_format) + tuple((p.data_ptr(), p._version) for p in params)
        if self._packed is not None and self._packed_key == key:
            return self._packed
        lib = _lib.load_library()
        cfg = self._cfg()
        nbytes = lib.univtg_clip_packed_bytes(ctypes.byref(cfg))
        if nbytes == 0:
            raise RuntimeError(f"univtg_b200: univtg_clip_packed_bytes failed: {_lib.last_error()}")
        packed = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        ptrs = [p.detach().contiguous() for p in params]
        arr = (ctypes.c_void_p * len(ptrs))(*[p.data_ptr() for p in ptrs])
        with torch.cuda.device(dev):
            _lib.check(lib.univtg_clip_pack_weights(ctypes.byref(cfg), arr, len(ptrs), 0 if dtype == torch.float32 else 1, _lib.ptr(packed),
                                                    _lib.stream_ptr()), "univtg_clip_pack_weights")
        self._packed, self._packed_key = packed, key
        return packed

    def _workspace(self, dev, n_images, n_texts, text_len):
        lib = _lib.load_library()
        cfg = self._cfg()
        nbytes = lib.univtg_clip_workspace_bytes(ctypes.byref(cfg), n_images, n_texts, text_len)
        if nbytes == 0:
            raise RuntimeError(f"univtg_b200: univtg_clip_workspace_bytes failed: {_lib.last_error()}")
        if self._ws is None or self._ws.numel() < nbytes or self._ws.device != dev:
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        return self._ws

    def _input(self, t, name, dev):
        if not torch.is_tensor(t) or t.device != dev:
            raise RuntimeError(f"ClipEncoder: {name} must be a tensor on {dev} (CPU tensors are not accepted)")
        return t.contiguous()

    @staticmethod
    def _check_count(n, name):
        if not 1 <= n <= 65535:
            raise ValueError(f"ClipEncoder: {name} must hold between 1 and 65535 rows per call, got {n}")

    # ---- public entry points ----
    def encode_image(self, frames):
        """frames: uint8 [T, R, R, 3] RGB as ffmpeg's rgb24 decodes them (normalised in-kernel like run_on_video Preprocessing),
        or float32 [T, 3, R, R] already normalised (encode_image's input).  Returns float32 [T, embed_dim]."""
        self._check_mode()
        dev = self._device()
        frames = self._input(frames, "frames", dev)
        R = self.config["image_resolution"]
        if frames.dtype == torch.uint8 and frames.dim() == 4 and tuple(frames.shape[1:]) == (R, R, 3):
            kind = 0
        elif frames.dtype == torch.float32 and frames.dim() == 4 and tuple(frames.shape[1:]) == (3, R, R):
            kind = 1
        else:
            raise TypeError(f"ClipEncoder.encode_image: frames must be uint8 [T, {R}, {R}, 3] or float32 [T, 3, {R}, {R}], "
                            f"got {frames.dtype} {tuple(frames.shape)}")
        T = frames.shape[0]
        self._check_count(T, "frames")
        packed = self._ensure_packed()
        ws = self._workspace(dev, T, 0, 0)
        out = torch.empty(T, self.config["embed_dim"], dtype=torch.float32, device=dev)
        lib = _lib.load_library()
        with torch.cuda.device(dev):
            _lib.check(lib.univtg_clip_encode_image(ctypes.byref(self._cfg()), _lib.ptr(packed), _lib.ptr(frames), kind, T, _lib.ptr(ws),
                                                    ws.numel(), _lib.ptr(out), _lib.stream_ptr()), "univtg_clip_encode_image")
        return out

    def _encode_text(self, tokens, ctx_used, want_last, want_pooled):
        self._check_mode()
        dev = self._device()
        tokens = self._input(tokens, "tokens", dev)
        C = self.config["context_length"]
        if tokens.dtype != torch.int64 or tokens.dim() != 2 or tokens.shape[1] != C:
            raise TypeError(f"ClipEncoder: tokens must be int64 [N, {C}] (clip.tokenize ids), got {tokens.dtype} {tuple(tokens.shape)}")
        N = tokens.shape[0]
        self._check_count(N, "tokens")
        packed = self._ensure_packed()
        ws = self._workspace(dev, 0, N, ctx_used)
        last = torch.empty(N, ctx_used, self.config["text_width"], dtype=torch.float32, device=dev) if want_last else None
        pooled = torch.empty(N, self.config["embed_dim"], dtype=torch.float32, device=dev) if want_pooled else None
        lib = _lib.load_library()
        with torch.cuda.device(dev):
            _lib.check(lib.univtg_clip_encode_text(ctypes.byref(self._cfg()), _lib.ptr(packed), _lib.ptr(tokens), N, ctx_used, _lib.ptr(ws),
                                                   ws.numel(), _lib.ptr(last), _lib.ptr(pooled), _lib.stream_ptr()),
                       "univtg_clip_encode_text")
        return last, pooled

    def encode_text(self, tokens):
        """tokens: int64 [N, context_length] -> {"last_hidden_state": [N, context_length, text_width], "pooler_output":
        [N, embed_dim]} (float32), as the reference's encode_text returns them."""
        last, pooled = self._encode_text(tokens, self.config["context_length"], True, True)
        return {"last_hidden_state": last, "pooler_output": pooled}

    def text_features(self, tokens):
        """The query features txt2clip keeps: the first (tokens != 0).sum(1) rows of last_hidden_state.  The text tower runs only
        up to the batch's longest valid length (the causal mask makes those rows independent of what follows).  Returns
        (features float32 [N, Lq, text_width] with zero rows past each query's length, mask float32 [N, Lq])."""
        if not torch.is_tensor(tokens) or tokens.dim() != 2:
            raise TypeError("ClipEncoder.text_features: tokens must be an int64 [N, context_length] tensor")
        self._check_count(tokens.shape[0], "tokens")
        lengths = (tokens != 0).sum(1)
        lq = max(int(lengths.max()), 1)  # host sync: the length decides the launch shapes
        feats, _ = self._encode_text(tokens, lq, True, False)
        mask = (torch.arange(lq, device=feats.device)[None] < lengths[:, None]).to(torch.float32)
        return feats * mask[..., None], mask

    def num_launches(self, tower, text_outputs=3):
        """Kernels one encode_image (tower 0) / text call (tower 1; bit 0 last_hidden_state, bit 1 pooler_output) launches."""
        n = _lib.load_library().univtg_clip_num_launches(ctypes.byref(self._cfg()), tower, text_outputs)
        if n < 0:
            raise RuntimeError(f"univtg_b200: univtg_clip_num_launches failed: {_lib.last_error()}")
        return n


def grounding_inputs(vid_feats, txt_feats, clip_len=2):
    """main_gradio.load_data (main_gradio.py:58-80) on the device: L2-normalised features (norm + 1e-5,
    utils/basic_utils.py:97-99), TEF columns, all-ones masks and the clip timestamps.

    vid_feats [T, D] (encode_image), txt_feats [Lq, Dt] (one query's text_features rows).  Returns (inputs for Model.forward,
    targets for postproc.decode_mr), batch 1."""
    if not (torch.is_tensor(vid_feats) and torch.is_tensor(txt_feats)) or vid_feats.dim() != 2 or txt_feats.dim() != 2:
        raise TypeError("grounding_inputs: vid_feats [T, D] and txt_feats [Lq, Dt] tensors expected")
    if vid_feats.device.type != "cuda" or txt_feats.device != vid_feats.device:
        raise RuntimeError("grounding_inputs: vid_feats and txt_feats must be on the same CUDA device")
    vid = vid_feats.float()
    txt = txt_feats.float()
    vid = vid / (vid.norm(dim=-1, keepdim=True) + 1e-5)
    txt = txt / (txt.norm(dim=-1, keepdim=True) + 1e-5)
    T, dev = vid.shape[0], vid.device
    ar = torch.arange(T, dtype=torch.float32, device=dev)
    tef = torch.stack([ar / T, ar / T + 1.0 / T], dim=1)
    ts = ((ar + clip_len / 2) / T).unsqueeze(1).repeat(1, 2)
    inputs = {"src_vid": torch.cat([vid, tef], dim=1)[None], "src_vid_mask": torch.ones(1, T, device=dev), "src_txt": txt[None],
              "src_txt_mask": torch.ones(1, txt.shape[0], device=dev)}
    return inputs, {"timestamp": ts[None], "timestamp_mask": torch.ones(1, T, device=dev)}
