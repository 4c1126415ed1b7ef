"""CPU oracle of the CLIP feature extractor -- TEST INFRASTRUCTURE ONLY.

A from-scratch restatement (explicit tensor algebra, fp64 by default) of OpenAI CLIP's ViT image tower and text tower as the
UniVTG reference vendors them, plus the glue that turns their features into UniVTG inputs.  It is the checker for
univtg_b200/clip.py and csrc/clip.cu; tests/test_clip_cpu.py pins it to outputs of the unmodified reference
(tests/golden/reference_clip.npz).  The product package never imports it.

`opq` is the operand-rounding hook of oracle/univtg_oracle.py: every value the CUDA path stores as a 16-bit GEMM or attention
operand goes through it (round_fp16 / round_bf16 emulate the kernels; None = exact).  `dtype` selects the arithmetic type; with
torch.float16 on a GPU the functions are the reference's own fp16 execution (convert_weights, model.py:371-392): matrices in fp16,
LayerNorm in fp32 (model.py:153-159), attention softmax in fp32.

Reference lines each function follows (paths relative to the UniVTG repository root):
  preprocess          run_on_video/preprocessing.py:4-25 (/255, then (x - mean) / (std + 1e-8))
  encode_image        run_on_video/clip/model.py:219-236 (VisualTransformer.forward)
  encode_text         run_on_video/clip/model.py:339-352 with the causal mask of 324-330
  _block              run_on_video/clip/model.py:167-188 (ResidualAttentionBlock, pre-norm, QuickGELU 162-164),
                      attention as torch nn.MultiheadAttention (in_proj packed q | k | v, q scaled by dh**-0.5)
  grounding_inputs    main_gradio.py:58-80 (load_data) with utils/basic_utils.py:97-99 (l2_normalize_np_array)
"""
import math

import torch

from oracle.univtg_oracle import round_bf16, round_fp16  # noqa: F401  (the same operand quantisers)

MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)


def _ident(t):
    return t


def _acc(dtype):
    return torch.promote_types(dtype, torch.float32)


def layer_norm(x, w, b, eps=1e-5):
    """LayerNorm in at least fp32, result in x's dtype (model.py:153-159)."""
    a = x.to(_acc(x.dtype))
    xc = a - a.mean(dim=-1, keepdim=True)
    var = (xc * xc).mean(dim=-1, keepdim=True)
    return (xc * torch.rsqrt(var + eps) * w.to(a.dtype) + b.to(a.dtype)).to(x.dtype)


def mm(a, w, opq, bias=None):
    """a [.., K] @ w[N, K]^T (+ bias), both operands through the operand quantiser."""
    y = opq(a) @ opq(w).transpose(-1, -2)
    return y + bias if bias is not None else y


def quick_gelu(x):
    return x * torch.sigmoid(1.702 * x)


def _attention(x, sd, pre, causal, opq):
    """nn.MultiheadAttention(x, x, x, attn_mask=triu(-inf) when causal); x [S, L, W], heads of 64."""
    S, L, W = x.shape
    H = W // 64
    qkv = opq(mm(x, sd[pre + "in_proj_weight"], opq, sd[pre + "in_proj_bias"]))
    q, k, v = (qkv[..., i * W:(i + 1) * W].reshape(S, L, H, 64).transpose(1, 2) for i in range(3))
    acc = _acc(x.dtype)
    s = (q.to(acc) @ k.to(acc).transpose(-1, -2)) * (1.0 / math.sqrt(64))
    if causal:
        s = s.masked_fill(torch.ones(L, L, dtype=torch.bool, device=x.device).triu(1), float("-inf"))
    s = s - s.amax(dim=-1, keepdim=True)
    p = torch.exp(s)
    o = (opq(p) @ v.to(acc)) / p.sum(dim=-1, keepdim=True)  # the CUDA path rounds un-normalised probabilities
    o = opq(o.to(x.dtype)).transpose(1, 2).reshape(S, L, W)
    return mm(o, sd[pre + "out_proj.weight"], opq, sd[pre + "out_proj.bias"])


def _block(x, sd, pre, causal, opq):
    x = x + _attention(opq(layer_norm(x, sd[pre + "ln_1.weight"], sd[pre + "ln_1.bias"])), sd, pre + "attn.", causal, opq)
    h = mm(opq(layer_norm(x, sd[pre + "ln_2.weight"], sd[pre + "ln_2.bias"])), sd[pre + "mlp.c_fc.weight"], opq, sd[pre + "mlp.c_fc.bias"])
    return x + mm(opq(quick_gelu(h)), sd[pre + "mlp.c_proj.weight"], opq, sd[pre + "mlp.c_proj.bias"])


def _cast(sd, dtype, device):
    return {k: v.to(device=device, dtype=dtype) for k, v in sd.items() if torch.is_tensor(v) and v.is_floating_point()}


def preprocess(frames):
    """uint8 [T, R, R, 3] RGB -> normalised f32 [T, 3, R, R], in fp32 as the reference computes it."""
    x = frames.permute(0, 3, 1, 2).to(torch.float32) / 255.0
    mean = torch.tensor(MEAN, dtype=torch.float32, device=frames.device).view(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=torch.float32, device=frames.device).view(1, 3, 1, 1)
    return (x - mean) / (std + 1e-8)


def encode_image(sd, cfg, images, opq=None, dtype=torch.float64):
    """images: normalised [T, 3, R, R] -> [T, embed_dim] (in `dtype`)."""
    opq = opq or _ident
    dev = images.device
    sd = _cast(sd, dtype, dev)
    P, W = cfg["patch_size"], cfg["vision_width"]
    T, _, R, _ = images.shape
    g = R // P
    # conv1 (stride = kernel = P, no bias) as a product over (c, ky, kx) patches
    patches = images.to(dtype).reshape(T, 3, g, P, g, P).permute(0, 2, 4, 1, 3, 5).reshape(T, g * g, 3 * P * P)
    x = mm(patches, sd["visual.conv1.weight"].reshape(W, -1), opq)
    x = torch.cat([sd["visual.class_embedding"].expand(T, 1, W), x], dim=1) + sd["visual.positional_embedding"]
    x = layer_norm(x, sd["visual.ln_pre.weight"], sd["visual.ln_pre.bias"])
    for l in range(cfg["vision_layers"]):
        x = _block(x, sd, f"visual.transformer.resblocks.{l}.", False, opq)
    c = opq(layer_norm(x[:, 0], sd["visual.ln_post.weight"], sd["visual.ln_post.bias"]))
    return c @ opq(sd["visual.proj"])


def encode_text(sd, cfg, tokens, opq=None, dtype=torch.float64):
    """tokens: int64 [N, context_length] -> {"last_hidden_state" [N, C, Wt], "pooler_output" [N, embed_dim]}."""
    opq = opq or _ident
    sd = _cast(sd, dtype, tokens.device)
    x = sd["token_embedding.weight"][tokens] + sd["positional_embedding"]
    for l in range(cfg["text_layers"]):
        x = _block(x, sd, f"transformer.resblocks.{l}.", True, opq)
    x = layer_norm(x, sd["ln_final.weight"], sd["ln_final.bias"])
    eot = x[torch.arange(x.shape[0], device=x.device), tokens.argmax(dim=-1)]
    return {"last_hidden_state": x, "pooler_output": opq(eot) @ opq(sd["text_projection"])}


def grounding_inputs(vid_feats, txt_feats, clip_len=2):
    """vid_feats [T, D], txt_feats [Lq, Dt] -> (Model.forward inputs with batch 1, decode targets) as load_data builds them."""
    vid = vid_feats / (vid_feats.norm(dim=-1, keepdim=True) + 1e-5)
    txt = txt_feats / (txt_feats.norm(dim=-1, keepdim=True) + 1e-5)
    T = vid.shape[0]
    ar = torch.arange(T, dtype=vid.dtype, device=vid.device)
    tef = torch.stack([ar / T, ar / T + 1.0 / T], dim=1)
    ts = ((ar + clip_len / 2) / T).unsqueeze(1).repeat(1, 2)
    inputs = {"src_vid": torch.cat([vid, tef], dim=1)[None], "src_vid_mask": torch.ones(1, T, dtype=vid.dtype, device=vid.device),
              "src_txt": txt[None], "src_txt_mask": torch.ones(1, txt.shape[0], dtype=vid.dtype, device=vid.device)}
    return inputs, {"timestamp": ts[None], "timestamp_mask": torch.ones(1, T, dtype=vid.dtype, device=vid.device)}
