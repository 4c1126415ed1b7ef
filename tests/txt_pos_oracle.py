"""The CPU oracle's Model.forward with learned text positions (args.use_txt_pos; reference model/univtg.py:123,
model/position_encoding.py:19-41):

    pos_t = Dropout(LayerNorm_txtpos(x_t + P[:Lt]))      x_t = projected text tokens + token-type row 0

takes the place of the zero text half of `pos`, so it is added to the text rows of q = k = x + pos in every encoder layer
(v stays x).  `txt_pos_mul` is the train-mode dropout multiplier [B, Lt, d] (0 or 1/(1-p)) or None.  Everything else is the
attention-dropout oracle (tests/attn_dropout_oracle.py) and the oracle's own building blocks; with use_txt_pos=False the result
is bit-identical to oracle.univtg_oracle.forward (tests/test_txt_pos_cpu.py checks it)."""
import torch

from oracle import univtg_oracle as O
from tests import attn_dropout_oracle as AO


def text_positions(sd, x_t, txt_pos_mul=None):
    Lt = x_t.shape[1]
    u = x_t + sd["txt_position_embed.position_embeddings.weight"][:Lt][None]
    pos_t = O.layer_norm(u, sd["txt_position_embed.LayerNorm.weight"], sd["txt_position_embed.LayerNorm.bias"])
    if txt_pos_mul is not None:
        pos_t = pos_t * txt_pos_mul.to(pos_t.dtype)
    return pos_t


def forward(sd, cfg, src_txt, src_txt_mask, src_vid, src_vid_mask, dp_scale=None, dtype=torch.float64, opq=None,
            drop_masks=None, attn_masks=None, use_txt_pos=False, txt_pos_mul=None):
    """tests.attn_dropout_oracle.forward plus use_txt_pos / txt_pos_mul."""
    opq = opq or O._ident
    sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}
    d, H, N, n_proj = cfg["hidden_dim"], cfg["nheads"], cfg["enc_layers"], cfg["n_input_proj"]
    src_txt, src_vid = src_txt.to(dtype), src_vid.to(dtype)
    tmask, vmask = src_txt_mask.to(dtype), src_vid_mask.to(dtype)
    B, Lv = src_vid.shape[:2]
    Lt = src_txt.shape[1]
    if use_txt_pos and Lt > sd["txt_position_embed.position_embeddings.weight"].shape[0]:
        raise ValueError(f"{Lt} text tokens exceed the position table")
    mv = drop_masks[:n_proj] if drop_masks is not None else None
    mt = drop_masks[n_proj:2 * n_proj] if drop_masks is not None else None
    x_v = O.input_proj(src_vid, sd, "input_vid_proj.", n_proj, opq, mv) + sd["token_type_embeddings.weight"][1]
    x_t = O.input_proj(src_txt, sd, "input_txt_proj.", n_proj, opq, mt) + sd["token_type_embeddings.weight"][0]
    x = torch.cat([x_v, x_t], dim=1)
    key_valid = torch.cat([vmask, tmask], dim=1) != 0
    pos_t = text_positions(sd, x_t, txt_pos_mul) if use_txt_pos else torch.zeros(B, Lt, d, dtype=dtype, device=src_vid.device)
    pos = torch.cat([O.sine_position(vmask, d, dtype), pos_t], dim=1)
    ones = torch.ones(B, dtype=dtype, device=src_vid.device)
    for l in range(N):
        s1 = dp_scale[2 * l].to(dtype) if dp_scale is not None else ones
        s2 = dp_scale[2 * l + 1].to(dtype) if dp_scale is not None else ones
        m = attn_masks[l] if attn_masks is not None else None
        x = AO.encoder_layer(x, pos, key_valid, sd, f"transformer.encoder.layers.{l}.", H, s1, s2, opq, m)
    vid_mem = x[:, :Lv]
    pred_logits = torch.sigmoid(O.conv_head(vid_mem, sd, "class_embed.", opq))
    spans = torch.sigmoid(O.conv_head(vid_mem, sd, "span_embed.", opq))
    pred_spans = spans * torch.tensor([-1.0, 1.0], dtype=dtype, device=src_vid.device)
    pooled, _ = O.weighted_pool(x_t, tmask, sd["weightedpool.weight"])
    tiny = torch.tensor(2.0 ** -149, dtype=dtype, device=src_vid.device)
    sal = O.cosine(x_v, pooled[:, None, :]) + torch.log(vmask + tiny)
    return {"pred_logits": pred_logits, "pred_spans": pred_spans, "src_vid_mask": src_vid_mask, "vid_mem_proj": x_v,
            "txt_mem_proj": pooled[:, None, :], "saliency_scores": sal}
