"""CPU oracle of the UniVTG hot path -- TEST INFRASTRUCTURE ONLY.
(Device-agnostic tensor algebra: bench.py's `gpu_eager_baseline` leg also runs it on the GPU through torch eager / cuBLAS as the
"reference on the same GPU" baseline of SURVEY.md section 8(d) - a baseline beside the product, never inside it.)

This file is a from-scratch restatement (explicit tensor algebra on torch CPU tensors, fp64 by default) of what the
reference computes on the path named in BASELINE.json; it is the *checker* for the CUDA kernels.  Only tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import it; the product package
(univtg_b200/) must never import, call or fall back to anything under oracle/.

Parity pinning: the reference ships no tests or golden vectors for this path (SURVEY.md section 4/8c: "parity unpinned"
by its own tests).  The oracle is therefore pinned against outputs of the reference (`model/univtg.py`),
stored in tests/golden/reference_pins.npz, by tests/test_oracle_vs_reference.py, and against the fixtures that
tests/golden/make_golden.py generated from the reference (tests/golden/*.npz).

Reference lines each function follows (paths relative to the UniVTG repository root):
  layer_norm / linear_layer   model/univtg.py:384-406 (LinearLayer), torch nn.LayerNorm (eps 1e-5, biased variance)
  sine_position               model/position_encoding.py:60-83
  multi_head_attention        torch F.multi_head_attention_forward as called at model/transformer_encoder_droppath.py:118
                              (q = k = x + pos, v = x, key_padding_mask, packed in_proj split in 3, q scaled by dh**-0.5)
  encoder_layer               model/transformer_encoder_droppath.py:112-126 (post-norm) and :154-167 (DropPath)
  conv1d_k3 / conv_head       model/univtg.py:367-382 (Conv), 129-136 (sigmoid, (-1,+1) sign)
  weighted_pool               model/univtg.py:22-24, 36-49
  forward                     model/univtg.py:105-155
  criterion                   model/univtg.py:195-282 (loss_spans, loss_labels, loss_saliency), 338-351;
                              utils/span_utils.py:46-73, 93-122 (temporal IoU / GIoU, diagonal only)
"""
import math

import torch
import torch.nn.functional as F

_ERF_C = 1.0 / math.sqrt(2.0)


def _ident(t):
    return t


def round_fp16(t):
    """Operand quantiser emulating the CUDA path's fp16 MMA operands (round-to-nearest-even)."""
    return t.to(torch.float16).to(t.dtype)


def round_bf16(t):
    return t.to(torch.bfloat16).to(t.dtype)


def layer_norm(x, w, b, eps=1e-5):
    xc = x - x.mean(dim=-1, keepdim=True)
    var = (xc * xc).mean(dim=-1, keepdim=True)
    return xc * torch.rsqrt(var + eps) * w + b


def gelu_erf(x):
    return 0.5 * x * (1.0 + torch.erf(x * _ERF_C))


def mm(a, w, opq, bias=None):
    """a [.., K] times w [N, K]^T (+ bias) with both operands passed through the operand quantiser."""
    a2 = opq(a).reshape(-1, a.shape[-1])
    wt = opq(w).transpose(-1, -2)
    y = torch.addmm(bias, a2, wt) if bias is not None else a2 @ wt
    return y.reshape(a.shape[:-1] + (w.shape[0],))


def sine_position(vid_mask, d, dtype):
    """pos [B, Lv, d]: normalised cumulative position, interleaved sin (even j) / cos (odd j)."""
    m = vid_mask.to(dtype)
    c = torch.cumsum(m, dim=1)
    e = c / (c[:, -1:] + 1e-6) * (2.0 * math.pi)
    j = torch.arange(d, dtype=dtype, device=vid_mask.device)
    dim_t = 10000.0 ** (2.0 * torch.floor(j / 2.0) / d)
    arg = e[:, :, None] / dim_t
    pos = torch.where((torch.arange(d, device=vid_mask.device) % 2 == 0)[None, None, :], torch.sin(arg), torch.cos(arg))
    return pos


def multi_head_attention(xq, xv, key_valid, w_in, b_in, w_out, b_out, nheads, opq):
    """xq: [B, L, d] query/key input (x + pos); xv: [B, L, d] value input; key_valid: [B, L] bool."""
    B, L, d = xq.shape
    dh = d // nheads
    q = mm(xq, w_in[:d], opq, b_in[:d])
    k = mm(xq, w_in[d:2 * d], opq, b_in[d:2 * d])
    v = mm(xv, w_in[2 * d:], opq, b_in[2 * d:])
    q = opq(q).reshape(B, L, nheads, dh).permute(0, 2, 1, 3).contiguous()
    k = opq(k).reshape(B, L, nheads, dh).permute(0, 2, 3, 1).contiguous()
    v = opq(v).reshape(B, L, nheads, dh).permute(0, 2, 1, 3).contiguous()
    s = (q @ k) * (1.0 / math.sqrt(dh))  # torch scales q before the product; the CUDA path scales the fp32 scores
    s = s.masked_fill(~key_valid[:, None, None, :], float("-inf"))
    s = s - s.amax(dim=-1, keepdim=True)
    p = torch.exp(s)
    denom = p.sum(dim=-1, keepdim=True)
    o = (opq(p) @ v) / denom  # the CUDA path rounds un-normalised probabilities, then divides by the fp32 row sum
    o = o.permute(0, 2, 1, 3).reshape(B, L, d)
    return mm(o, w_out, opq, b_out)


def encoder_layer(x, pos, key_valid, sd, pre, nheads, s1, s2, opq):
    a = multi_head_attention(x + pos, x, key_valid, sd[pre + "self_attn.in_proj_weight"], sd[pre + "self_attn.in_proj_bias"],
                             sd[pre + "self_attn.out_proj.weight"], sd[pre + "self_attn.out_proj.bias"], nheads, opq)
    # the CUDA path stores the DropPath-scaled branch as a 16-bit operand before adding it to the fp32 residual stream
    x = layer_norm(x + opq(s1[:, None, None] * a), sd[pre + "norm1.weight"], sd[pre + "norm1.bias"])
    h = gelu_erf(mm(x, sd[pre + "linear1.weight"], opq, sd[pre + "linear1.bias"]))
    f = mm(h, sd[pre + "linear2.weight"], opq, sd[pre + "linear2.bias"])
    x = layer_norm(x + opq(s2[:, None, None] * f), sd[pre + "norm2.weight"], sd[pre + "norm2.bias"])
    return x


def conv1d_k3(x, w, b, opq_x, opq_w):
    """x [B, L, C]; w [N, C, 3]; cross-correlation, zero padding 1:  y[l] = sum_t W[:, :, t] x[l + t - 1] + b."""
    B, L, C = x.shape
    xq = opq_x(x)
    z = torch.zeros(B, 1, C, dtype=x.dtype, device=x.device)
    # taps t = 0, 1, 2 read x[l-1], x[l], x[l+1]; one [B*L, 3C] x [3C, N] product
    taps = torch.cat([torch.cat([z, xq[:, :-1]], 1), xq, torch.cat([xq[:, 1:], z], 1)], dim=-1)
    w2 = opq_w(w).permute(0, 2, 1).reshape(w.shape[0], 3 * C)  # w2[n, t*C + c] = w[n, c, t]
    return torch.addmm(b, taps.reshape(B * L, 3 * C), w2.t()).reshape(B, L, -1)


def conv_head(x, sd, pre, opq):
    h = torch.relu(conv1d_k3(x, sd[pre + "layers.0.weight"], sd[pre + "layers.0.bias"], opq, opq))
    h = torch.relu(conv1d_k3(h, sd[pre + "layers.1.weight"], sd[pre + "layers.1.bias"], opq, opq))
    # the CUDA path keeps the last (1- or 2-channel) conv in fp32 weights over the 16-bit hidden activations
    return conv1d_k3(h, sd[pre + "layers.2.weight"], sd[pre + "layers.2.bias"], opq, _ident)


def input_proj(x, sd, pre, n_proj, opq, masks=None):
    """LinearLayer stack (model/univtg.py:399-406): LayerNorm -> Dropout -> Linear [-> ReLU].  masks[i]: the train-mode
    nn.Dropout multiplier of layer i (0 or 1/(1-p), same shape as the layer input) or None (eval / p = 0)."""
    for i in range(n_proj):
        p = f"{pre}{i}."
        x = layer_norm(x, sd[p + "LayerNorm.weight"], sd[p + "LayerNorm.bias"])
        if masks is not None and masks[i] is not None:
            x = x * masks[i].to(x.dtype)
        x = mm(x, sd[p + "net.1.weight"], opq, sd[p + "net.1.bias"])
        if i < n_proj - 1:
            x = torch.relu(x)
    return x


def weighted_pool(x, mask, w):
    alpha = (x @ w).squeeze(-1) + (1.0 - mask) * (-1e30)
    alpha = torch.softmax(alpha, dim=1)
    return (x * alpha[:, :, None]).sum(dim=1), alpha


def cosine(a, b, eps=1e-8):
    na = a.norm(dim=-1).clamp_min(eps)
    nb = b.norm(dim=-1).clamp_min(eps)
    return (a * b).sum(dim=-1) / (na * nb)


def forward(sd, cfg, src_txt, src_txt_mask, src_vid, src_vid_mask, dp_scale=None, dtype=torch.float64, opq=None,
            keep_intermediates=False, drop_masks=None):
    """Restatement of Model.forward (eval mode unless dp_scale [2*N, B] / drop_masks are given).

    drop_masks: train-mode input-dropout multipliers, [video layer 0..n-1, text layer 0..n-1] (model/univtg.py:394,401).
    sd: reference-named state dict; cfg: dict with hidden_dim, nheads, enc_layers, n_input_proj."""
    opq = opq or _ident
    sd = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}  # differentiable cast (autograd oracle)
    d, H, N, n_proj = cfg["hidden_dim"], cfg["nheads"], cfg["enc_layers"], cfg["n_input_proj"]
    src_txt, src_vid = src_txt.to(dtype), src_vid.to(dtype)
    tmask, vmask = src_txt_mask.to(dtype), src_vid_mask.to(dtype)
    B, Lv = src_vid.shape[:2]
    Lt = src_txt.shape[1]
    mv = drop_masks[:n_proj] if drop_masks is not None else None
    mt = drop_masks[n_proj:2 * n_proj] if drop_masks is not None else None
    x_v = input_proj(src_vid, sd, "input_vid_proj.", n_proj, opq, mv) + sd["token_type_embeddings.weight"][1]
    x_t = input_proj(src_txt, sd, "input_txt_proj.", n_proj, opq, mt) + sd["token_type_embeddings.weight"][0]
    x = torch.cat([x_v, x_t], dim=1)
    key_valid = torch.cat([vmask, tmask], dim=1) != 0
    pos = torch.cat([sine_position(vmask, d, dtype), torch.zeros(B, Lt, d, dtype=dtype, device=src_vid.device)], dim=1)
    ones = torch.ones(B, dtype=dtype, device=src_vid.device)
    inter = {}
    for l in range(N):
        s1 = dp_scale[2 * l].to(dtype) if dp_scale is not None else ones
        s2 = dp_scale[2 * l + 1].to(dtype) if dp_scale is not None else ones
        x = encoder_layer(x, pos, key_valid, sd, f"transformer.encoder.layers.{l}.", H, s1, s2, opq)
        inter[f"layer{l}"] = x
    vid_mem = x[:, :Lv]
    pred_logits = torch.sigmoid(conv_head(vid_mem, sd, "class_embed.", opq))
    spans = torch.sigmoid(conv_head(vid_mem, sd, "span_embed.", opq))
    pred_spans = spans * torch.tensor([-1.0, 1.0], dtype=dtype, device=src_vid.device)
    pooled, alpha = weighted_pool(x_t, tmask, sd["weightedpool.weight"])
    # log(mask + 1e-45): 1e-45 rounds to the smallest fp32 denormal 2**-149 in the reference
    tiny = torch.tensor(2.0 ** -149, dtype=dtype, device=src_vid.device)
    sal = cosine(x_v, pooled[:, None, :]) + torch.log(vmask + tiny)
    out = {"pred_logits": pred_logits, "pred_spans": pred_spans, "src_vid_mask": src_vid_mask, "vid_mem_proj": x_v,
           "txt_mem_proj": pooled[:, None, :], "saliency_scores": sal}
    if keep_intermediates:
        out["_memory"] = x
        out["_inter"] = inter
        out["_pos"] = pos
    return out


# ------------------------------------------------------------------------------------------------------------------
# criterion (SetCriterion for model_id=univtg: losses 'spans', 'labels', 'saliency'; the Hungarian matcher is never called)
# ------------------------------------------------------------------------------------------------------------------
def _smooth_l1(a, b):
    dlt = (a - b).abs()
    return torch.where(dlt < 1.0, 0.5 * dlt * dlt, dlt - 0.5)


def _giou_pairs(s1, s2):
    """Paired generalised temporal IoU of spans [n, 2] in (start, end) format (diagonal of the reference's N x N)."""
    inter = (torch.minimum(s1[:, 1], s2[:, 1]) - torch.maximum(s1[:, 0], s2[:, 0])).clamp(min=0)
    union = (s1[:, 1] - s1[:, 0]) + (s2[:, 1] - s2[:, 0]) - inter
    iou = inter / union
    enclose = (torch.maximum(s1[:, 1], s2[:, 1]) - torch.minimum(s1[:, 0], s2[:, 0])).clamp(min=0)
    return iou - (enclose - union) / enclose


def _log_softmax(x, dim):
    m = x.amax(dim=dim, keepdim=True)
    return x - m - torch.log(torch.exp(x - m).sum(dim=dim, keepdim=True))


def criterion(outputs, targets, eos_coef=0.1, temperature=0.07, losses=("spans", "labels", "saliency")):
    dtype = outputs["pred_spans"].dtype
    t = {k: (v.to(dtype) if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in targets.items()}
    res = {}
    if "spans" in losses:
        src = t["timestamp"] + outputs["pred_spans"]
        gt = t["span_labels_nn"]
        fg = t["timestamp_window"] != 0
        res["loss_b"] = (_smooth_l1(src, gt) * t["timestamp_window"][:, :, None]).sum() / fg.sum()
        res["loss_g"] = (1.0 - _giou_pairs(src[fg], gt[fg])).mean()
    if "labels" in losses:
        p = outputs["pred_logits"].squeeze(-1)
        valid = t["timestamp_mask"] != 0
        fg = t["timestamp_window"] != 0
        y = fg.to(dtype)
        w = torch.zeros_like(p)
        w[valid] = eos_coef
        w[fg] = 1.0
        # torch's BCE: logs clamped at -100, backward w (p - y) / max(p (1 - p), 1e-12), finite at p = 0 and p = 1.  It refuses to
        # run inside an autocast region (bench.py's bf16-autocast baseline runs this criterion), so it is evaluated outside one,
        # in fp32 or wider.
        with torch.autocast(p.device.type, enabled=False):
            pw = p if p.dtype == torch.float64 else p.float()
            bce = F.binary_cross_entropy(pw, y.to(pw.dtype), weight=w.to(pw.dtype), reduction="none")
        res["loss_f"] = (bce * valid.to(dtype)).sum() / valid.sum()
    if "saliency" in losses:
        sal = t["saliency_scores"]
        if "saliency_pos_labels" not in t or float(sal.sum()) == 0.0:
            res["loss_s_inter"] = torch.zeros((), dtype=dtype, device=sal.device)
            res["loss_s_intra"] = torch.zeros((), dtype=dtype, device=sal.device)
        else:
            xv = outputs["vid_mem_proj"]
            xt = outputs["txt_mem_proj"].squeeze(1)
            B = xv.shape[0]
            bi = torch.arange(B, device=xv.device)
            pi = t["saliency_pos_labels"][:, 0].long()
            vf = xv[bi, pi]
            a_n = vf / vf.norm(dim=1, keepdim=True).clamp_min(1e-8)
            b_n = xt / xt.norm(dim=1, keepdim=True).clamp_min(1e-8)
            sim = a_n @ b_n.t()
            li = torch.diagonal(_log_softmax(sim / temperature, 1)).sum() / B
            lj = torch.diagonal(_log_softmax(sim.t() / temperature, 1)).sum() / B
            res["loss_s_inter"] = -li - lj
            sel = sal[bi, pi][:, None]
            neg = sal < sel
            neg[bi, pi] = True
            keep = (neg & (t["timestamp_mask"] != 0)).to(dtype)
            tiny = torch.tensor(2.0 ** -149, dtype=dtype, device=xv.device)
            sim_in = cosine(xv, xt[:, None, :]) + torch.log(keep + tiny)
            ls_i = _log_softmax(sim_in / temperature, 1)
            ls_j = _log_softmax(sim_in.t() / temperature, 1)
            res["loss_s_intra"] = -(ls_i[bi, pi].sum() / B) - (ls_j[pi, bi].sum() / B)
    return res


def weighted_total(loss_dict, weight_dict):
    return sum(loss_dict[k] * weight_dict[k] for k in loss_dict if k in weight_dict)
