"""The CPU oracle's Model.forward (oracle/univtg_oracle.py) with train-mode attention dropout: `attn_masks` holds one
[B, H, L, L] multiplier tensor per encoder layer (0 or 1/(1-p); row = query, column = key, L = Lv + Lt), applied to the
normalised probabilities before `@ v` as torch's F.multi_head_attention_forward does with dropout_p > 0 in training
(the reference's nn.MultiheadAttention(dropout=args.dropout), model/transformer_encoder_droppath.py:93).

Everything else is the oracle's own building blocks.  Under an operand quantiser `opq` the product p * m of the un-normalised
probabilities is rounded where the CUDA kernels round it, then divided by the fp32 (un-dropped) row sum.  With
attn_masks=None the result is bit-identical to oracle.univtg_oracle.forward (tests/test_attention_dropout_cpu.py checks it)."""
import math

import torch

from oracle import univtg_oracle as O


def multi_head_attention(xq, xv, key_valid, w_in, b_in, w_out, b_out, nheads, opq, mask=None):
    B, L, d = xq.shape
    dh = d // nheads
    q = O.mm(xq, w_in[:d], opq, b_in[:d])
    k = O.mm(xq, w_in[d:2 * d], opq, b_in[d:2 * d])
    v = O.mm(xv, w_in[2 * d:], opq, b_in[2 * d:])
    q = opq(q).reshape(B, L, nheads, dh).permute(0, 2, 1, 3).contiguous()
    k = opq(k).reshape(B, L, nheads, dh).permute(0, 2, 3, 1).contiguous()
    v = opq(v).reshape(B, L, nheads, dh).permute(0, 2, 1, 3).contiguous()
    s = (q @ k) * (1.0 / math.sqrt(dh))
    s = s.masked_fill(~key_valid[:, None, None, :], float("-inf"))
    s = s - s.amax(dim=-1, keepdim=True)
    p = torch.exp(s)
    denom = p.sum(dim=-1, keepdim=True)  # the normaliser is the un-dropped row sum
    if mask is not None:
        p = p * mask.to(p.dtype)
    o = (opq(p) @ v) / denom
    o = o.permute(0, 2, 1, 3).reshape(B, L, d)
    return O.mm(o, w_out, opq, b_out)


def encoder_layer(x, pos, key_valid, sd, pre, nheads, s1, s2, opq, mask=None):
    a = multi_head_attention(x + pos, x, key_valid, sd[pre + "self_attn.in_proj_weight"], sd[pre + "self_attn.in_proj_bias"],
                             sd[pre + "self_attn.out_proj.weight"], sd[pre + "self_attn.out_proj.bias"], nheads, opq, mask)
    x = O.layer_norm(x + opq(s1[:, None, None] * a), sd[pre + "norm1.weight"], sd[pre + "norm1.bias"])
    h = O.gelu_erf(O.mm(x, sd[pre + "linear1.weight"], opq, sd[pre + "linear1.bias"]))
    f = O.mm(h, sd[pre + "linear2.weight"], opq, sd[pre + "linear2.bias"])
    return O.layer_norm(x + opq(s2[:, None, None] * f), sd[pre + "norm2.weight"], sd[pre + "norm2.bias"])


def forward(sd, cfg, src_txt, src_txt_mask, src_vid, src_vid_mask, dp_scale=None, dtype=torch.float64, opq=None,
            drop_masks=None, attn_masks=None):
    """oracle.univtg_oracle.forward plus attn_masks (one [B, H, L, L] multiplier per encoder layer, or None)."""
    opq = opq or O._ident
    sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
    d, H, N, n_proj = cfg["hidden_dim"], cfg["nheads"], cfg["enc_layers"], cfg["n_input_proj"]
    src_txt, src_vid = src_txt.to(dtype), src_vid.to(dtype)
    tmask, vmask = src_txt_mask.to(dtype), src_vid_mask.to(dtype)
    B, Lv = src_vid.shape[:2]
    Lt = src_txt.shape[1]
    mv = drop_masks[:n_proj] if drop_masks is not None else None
    mt = drop_masks[n_proj:2 * n_proj] if drop_masks is not None else None
    x_v = O.input_proj(src_vid, sd, "input_vid_proj.", n_proj, opq, mv) + sd["token_type_embeddings.weight"][1]
    x_t = O.input_proj(src_txt, sd, "input_txt_proj.", n_proj, opq, mt) + sd["token_type_embeddings.weight"][0]
    x = torch.cat([x_v, x_t], dim=1)
    key_valid = torch.cat([vmask, tmask], dim=1) != 0
    pos = torch.cat([O.sine_position(vmask, d, dtype), torch.zeros(B, Lt, d, dtype=dtype, device=src_vid.device)], dim=1)
    ones = torch.ones(B, dtype=dtype, device=src_vid.device)
    for l in range(N):
        s1 = dp_scale[2 * l].to(dtype) if dp_scale is not None else ones
        s2 = dp_scale[2 * l + 1].to(dtype) if dp_scale is not None else ones
        m = attn_masks[l] if attn_masks is not None else None
        x = encoder_layer(x, pos, key_valid, sd, f"transformer.encoder.layers.{l}.", H, s1, s2, opq, m)
    vid_mem = x[:, :Lv]
    pred_logits = torch.sigmoid(O.conv_head(vid_mem, sd, "class_embed.", opq))
    spans = torch.sigmoid(O.conv_head(vid_mem, sd, "span_embed.", opq))
    pred_spans = spans * torch.tensor([-1.0, 1.0], dtype=dtype, device=src_vid.device)
    pooled, _ = O.weighted_pool(x_t, tmask, sd["weightedpool.weight"])
    tiny = torch.tensor(2.0 ** -149, dtype=dtype, device=src_vid.device)
    sal = O.cosine(x_v, pooled[:, None, :]) + torch.log(vmask + tiny)
    return {"pred_logits": pred_logits, "pred_spans": pred_spans, "src_vid_mask": src_vid_mask, "vid_mem_proj": x_v,
            "txt_mem_proj": pooled[:, None, :], "saliency_scores": sal}
