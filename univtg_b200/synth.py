"""Deterministic synthetic weights / inputs / targets of the shapes the reference feeds this path.

Input conventions follow the reference data pipeline: row-L2-normalised features + TEF columns
(main/dataset.py:534-540, 689-695), zero right-padding with float masks (utils/tensor_utils.py:36-53), dense per-clip
targets (main/dataset.py:501, 525-556, 1078-1098).  Seeds: weights torch.Generator(seed), data Generator(seed+1).
"""
import math
import random
import struct
from argparse import Namespace

import torch

CONFIGS = {
    # BASELINE.json configs[0]: gradio demo shapes (tmp/vid.npz 15x512(+2 TEF), tmp/txt.npz 12x512), d=256, 2 layers
    "cfg1": dict(hidden_dim=256, nheads=8, dim_feedforward=1024, enc_layers=2, n_input_proj=2, v_feat_dim=514, t_feat_dim=512,
                 batch=1, l_vid=15, l_txt=12),
    # configs[1] / [2]: QVHighlights-shaped
    "cfg2": dict(hidden_dim=1024, nheads=8, dim_feedforward=1024, enc_layers=4, n_input_proj=2, v_feat_dim=2818, t_feat_dim=512,
                 batch=32, l_vid=75, l_txt=32),
    # configs[3]: per-rank shard of the vlp_ddp pre-training batch
    "cfg4": dict(hidden_dim=1024, nheads=8, dim_feedforward=1024, enc_layers=4, n_input_proj=2, v_feat_dim=2818, t_feat_dim=512,
                 batch=32, l_vid=150, l_txt=32),
    # configs[4]: long-video stress
    "cfg5": dict(hidden_dim=1024, nheads=8, dim_feedforward=1024, enc_layers=6, n_input_proj=2, v_feat_dim=2818, t_feat_dim=512,
                 batch=8, l_vid=1200, l_txt=77),
    # small ragged parity case the oracle finishes in < 1 s
    "tiny": dict(hidden_dim=256, nheads=2, dim_feedforward=256, enc_layers=2, n_input_proj=2, v_feat_dim=194, t_feat_dim=128,
                 batch=3, l_vid=21, l_txt=9),
}


def reference_args(cfg, **over):
    """argparse.Namespace with every field reference build_model(args) reads (model/univtg.py:409-448)."""
    ns = Namespace(
        device="cpu", hidden_dim=cfg["hidden_dim"], dropout=0.0, droppath=0.1, nheads=cfg["nheads"],
        dim_feedforward=cfg["dim_feedforward"], enc_layers=cfg["enc_layers"], dec_layers=2, pre_norm=False,
        position_embedding="sine", max_q_l=max(75, cfg.get("l_txt", 32)), input_dropout=0.5, t_feat_dim=cfg["t_feat_dim"],
        v_feat_dim=cfg["v_feat_dim"], span_loss_type="l1", use_txt_pos=False, n_input_proj=cfg["n_input_proj"],
        set_cost_span=10, set_cost_giou=1, set_cost_class=4, max_v_l=max(75, cfg.get("l_vid", 75)), b_loss_coef=10.0,
        g_loss_coef=1.0, f_loss_coef=10.0, s_loss_intra_coef=0.1, s_loss_inter_coef=0.1, dset_type="vlp",
        train_path=["synthetic"], eos_coef=0.1, temperature=0.07, saliency_margin=0.2)
    for k, v in over.items():
        setattr(ns, k, v)
    return ns


def state_dict_shapes(cfg, max_q_l=None):
    """Reference state_dict keys -> shapes (SURVEY.md A.4), in the reference's registration order."""
    d, ff, N, n = cfg["hidden_dim"], cfg["dim_feedforward"], cfg["enc_layers"], cfg["n_input_proj"]
    max_q_l = max_q_l or max(75, cfg.get("l_txt", 32))
    out = {}
    for l in range(N):
        p = f"transformer.encoder.layers.{l}."
        out[p + "self_attn.in_proj_weight"] = (3 * d, d)
        out[p + "self_attn.in_proj_bias"] = (3 * d,)
        out[p + "self_attn.out_proj.weight"] = (d, d)
        out[p + "self_attn.out_proj.bias"] = (d,)
        out[p + "linear1.weight"] = (ff, d)
        out[p + "linear1.bias"] = (ff,)
        out[p + "linear2.weight"] = (d, ff)
        out[p + "linear2.bias"] = (d,)
        out[p + "norm1.weight"] = (d,)
        out[p + "norm1.bias"] = (d,)
        out[p + "norm2.weight"] = (d,)
        out[p + "norm2.bias"] = (d,)
    out["txt_position_embed.position_embeddings.weight"] = (max_q_l, d)
    out["txt_position_embed.LayerNorm.weight"] = (d,)
    out["txt_position_embed.LayerNorm.bias"] = (d,)
    out["token_type_embeddings.weight"] = (2, d)
    for head, od in (("span_embed", 2), ("class_embed", 1)):
        out[f"{head}.layers.0.weight"] = (d, d, 3)
        out[f"{head}.layers.0.bias"] = (d,)
        out[f"{head}.layers.1.weight"] = (d, d, 3)
        out[f"{head}.layers.1.bias"] = (d,)
        out[f"{head}.layers.2.weight"] = (od, d, 3)
        out[f"{head}.layers.2.bias"] = (od,)
    for name, din in (("input_txt_proj", cfg["t_feat_dim"]), ("input_vid_proj", cfg["v_feat_dim"])):
        k = din
        for i in range(n):
            out[f"{name}.{i}.LayerNorm.weight"] = (k,)
            out[f"{name}.{i}.LayerNorm.bias"] = (k,)
            out[f"{name}.{i}.net.1.weight"] = (d, k)
            out[f"{name}.{i}.net.1.bias"] = (d,)
            k = d
    out["weightedpool.weight"] = (d, 1)
    return out


def make_state_dict(cfg, seed=0, head_gain=1.0, dtype=torch.float32):
    """Seeded weights with the reference's init scales (xavier-uniform encoder matrices, U(+-1/sqrt(fan_in)) elsewhere)
    but non-trivial LayerNorm affine terms and biases, so that every parameter matters in a parity test."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd = {}
    for k, shp in state_dict_shapes(cfg).items():
        if k.endswith("LayerNorm.weight") or ".norm1.weight" in k or ".norm2.weight" in k:
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif k.endswith("LayerNorm.bias") or ".norm1.bias" in k or ".norm2.bias" in k:
            t = 0.05 * torch.randn(shp, generator=g)
        elif k == "token_type_embeddings.weight":
            t = 0.02 * torch.randn(shp, generator=g)
        elif k == "txt_position_embed.position_embeddings.weight":
            t = torch.randn(shp, generator=g)
        elif k.startswith("transformer.") and len(shp) == 2:
            bound = math.sqrt(6.0 / (shp[0] + shp[1]))
            t = (torch.rand(shp, generator=g) * 2 - 1) * bound
        elif k == "weightedpool.weight":
            bound = math.sqrt(6.0 / (shp[0] + shp[1]))
            t = (torch.rand(shp, generator=g) * 2 - 1) * bound
        elif len(shp) >= 2:
            fan_in = shp[1] * (shp[2] if len(shp) == 3 else 1)
            t = (torch.rand(shp, generator=g) * 2 - 1) / math.sqrt(fan_in)
            if k.endswith("layers.2.weight"):
                t = t * head_gain
        else:  # biases
            t = (torch.rand(shp, generator=g) * 2 - 1) * 0.05
        sd[k] = t.to(dtype)
    return sd


def make_inputs(cfg, seed=1, ragged=False, batch=None, l_vid=None, l_txt=None):
    """src_txt [B,Lt,Dt], src_txt_mask [B,Lt], src_vid [B,Lv,Dv], src_vid_mask [B,Lv] (float32, zero right-padded)."""
    B = batch or cfg["batch"]
    Lv = l_vid or cfg["l_vid"]
    Lt = l_txt or cfg["l_txt"]
    Dv, Dt = cfg["v_feat_dim"], cfg["t_feat_dim"]
    g = torch.Generator(device="cpu").manual_seed(seed)
    raw = torch.randn(B, Lv, Dv - 2, generator=g)
    split = (Dv - 2) * 9 // 11 if Dv - 2 >= 11 else (Dv - 2) // 2  # 2304 / 512 style two-backbone split
    if Dv == 2818:
        split = 2304
    parts = [raw[..., :split], raw[..., split:]] if 0 < split < Dv - 2 else [raw]
    parts = [p / (p.norm(dim=-1, keepdim=True) + 1e-5) for p in parts]
    tef = torch.stack([torch.arange(Lv) / Lv, (torch.arange(Lv) + 1) / Lv], dim=1)[None].expand(B, Lv, 2)
    src_vid = torch.cat(parts + [tef], dim=-1).float()
    src_txt = torch.randn(B, Lt, Dt, generator=g)
    src_txt = src_txt / (src_txt.norm(dim=-1, keepdim=True) + 1e-5)
    vmask = torch.ones(B, Lv)
    tmask = torch.ones(B, Lt)
    if ragged:
        lens_v = torch.randint(max(2, Lv // 5), Lv + 1, (B,), generator=g)
        lens_t = torch.randint(max(2, Lt // 5), Lt + 1, (B,), generator=g)
        lens_v[0] = Lv  # the collate pads to the longest sample
        lens_t[-1] = Lt
        vmask = (torch.arange(Lv)[None] < lens_v[:, None]).float()
        tmask = (torch.arange(Lt)[None] < lens_t[:, None]).float()
        # TEF is computed per sample over its own length before padding
        for b in range(B):
            n = int(lens_v[b])
            src_vid[b, :n, -2] = torch.arange(n) / n
            src_vid[b, :n, -1] = (torch.arange(n) + 1) / n
        src_vid = src_vid * vmask[..., None]
        src_txt = src_txt * tmask[..., None]
    return dict(src_txt=src_txt.float().contiguous(), src_txt_mask=tmask, src_vid=src_vid.float().contiguous(),
                src_vid_mask=vmask)


def make_targets(inputs, seed=2, clip_len=2.0):
    """Dense per-clip targets as DatasetMR/DatasetVLP build them: one random ground-truth window per sample."""
    vmask = inputs["src_vid_mask"]
    B, Lv = vmask.shape
    g = torch.Generator(device="cpu").manual_seed(seed)
    lens = vmask.sum(1).long()
    timestamp = torch.zeros(B, Lv, 2)
    window = torch.zeros(B, Lv)
    span_nn = torch.zeros(B, Lv, 2)
    sal = torch.zeros(B, Lv)
    pos = torch.zeros(B, 1, dtype=torch.long)
    neg = torch.zeros(B, 1, dtype=torch.long)
    for b in range(B):
        n = int(lens[b])
        centers = (torch.arange(n) + 0.5) / n  # ((l + clip_len/2) / L) with duration normalised to 1 (dataset.py:501)
        timestamp[b, :n, 0] = centers
        timestamp[b, :n, 1] = centers
        a = int(torch.randint(0, n, (1,), generator=g))
        e = int(torch.randint(a, n, (1,), generator=g))
        st, ed = a / n, (e + 1) / n
        inside = (centers >= st) & (centers <= ed)
        window[b, :n] = inside.float()
        span_nn[b, :n, 0] = st
        span_nn[b, :n, 1] = ed
        sal[b, :n] = inside.float() * (0.5 + 0.5 * torch.rand(n, generator=g))
        fg = inside.nonzero().flatten()
        pos[b, 0] = fg[int(torch.randint(0, len(fg), (1,), generator=g))]
        bg = (~inside).nonzero().flatten()
        neg[b, 0] = bg[0] if len(bg) else 0
    return dict(timestamp=timestamp, timestamp_mask=vmask.clone(), timestamp_window=window, span_labels_nn=span_nn,
                saliency_scores=sal, saliency_pos_labels=pos, saliency_neg_labels=neg)


def flops_forward(cfg, batch=None, l_vid=None, l_txt=None):
    """Algorithmic forward FLOPs (SURVEY.md 8d formulas), returns (total, encoder_only)."""
    d, ff, N = cfg["hidden_dim"], cfg["dim_feedforward"], cfg["enc_layers"]
    B = batch or cfg["batch"]
    Lv = l_vid or cfg["l_vid"]
    Lt = l_txt or cfg["l_txt"]
    L = Lv + Lt
    enc = N * (8 * L * d * d + 4 * L * d * ff + 4 * L * L * d)
    proj = 2 * Lv * (cfg["v_feat_dim"] * d + d * d) + 2 * Lt * (cfg["t_feat_dim"] * d + d * d)
    heads = 8 * Lv * 3 * d * d + 18 * Lv * d
    return B * (enc + proj + heads), B * enc


# CLIP (run_on_video/clip/model.py) shapes: ViT-B/32 as the reference's feature extractor loads it, and two small ones for goldens
CLIP_CONFIGS = {
    "vit_b32": dict(embed_dim=512, vision_width=768, vision_layers=12, patch_size=32, image_resolution=224, text_width=512,
                    text_layers=12, context_length=77, vocab_size=49408),
    "small224": dict(embed_dim=64, vision_width=128, vision_layers=2, patch_size=32, image_resolution=224, text_width=128,
                     text_layers=2, context_length=77, vocab_size=49408),
    "small64": dict(embed_dim=64, vision_width=64, vision_layers=2, patch_size=16, image_resolution=64, text_width=64,
                    text_layers=2, context_length=77, vocab_size=49408),
}
CLIP_SOT, CLIP_EOT = 49406, 49407  # <|startoftext|>, <|endoftext|> of clip.tokenize (the largest ids: argmax finds EOT)


def clip_state_dict_shapes(cfg):
    """Key -> shape of a ViT CLIP state dict (model.py:202-291), in the reference module's registration order."""
    Wv, Wt, E, P = cfg["vision_width"], cfg["text_width"], cfg["embed_dim"], cfg["patch_size"]
    grid = cfg["image_resolution"] // P

    def blocks(pre, W, n):
        out = {}
        for l in range(n):
            p = f"{pre}resblocks.{l}."
            out.update({p + "attn.in_proj_weight": (3 * W, W), p + "attn.in_proj_bias": (3 * W,), p + "attn.out_proj.weight": (W, W),
                        p + "attn.out_proj.bias": (W,), p + "ln_1.weight": (W,), p + "ln_1.bias": (W,), p + "mlp.c_fc.weight": (4 * W, W),
                        p + "mlp.c_fc.bias": (4 * W,), p + "mlp.c_proj.weight": (W, 4 * W), p + "mlp.c_proj.bias": (W,),
                        p + "ln_2.weight": (W,), p + "ln_2.bias": (W,)})
        return out

    s = {"positional_embedding": (cfg["context_length"], Wt), "text_projection": (Wt, E), "logit_scale": (),
         "visual.class_embedding": (Wv,), "visual.positional_embedding": (grid * grid + 1, Wv), "visual.proj": (Wv, E),
         "visual.conv1.weight": (Wv, 3, P, P), "visual.ln_pre.weight": (Wv,), "visual.ln_pre.bias": (Wv,)}
    s.update(blocks("visual.transformer.", Wv, cfg["vision_layers"]))
    s.update({"visual.ln_post.weight": (Wv,), "visual.ln_post.bias": (Wv,)})
    s.update(blocks("transformer.", Wt, cfg["text_layers"]))
    s.update({"token_embedding.weight": (cfg["vocab_size"], Wt), "ln_final.weight": (Wt,), "ln_final.bias": (Wt,)})
    return s


def make_clip_state_dict(cfg, seed=0, dtype=torch.float32):
    """Seeded ViT CLIP weights with the reference's keys and shapes and CLIP's init scales (model.py:209-217, 295-322), plus
    non-trivial LayerNorm affine terms and biases.  Like released checkpoints it carries the integer entries input_resolution,
    context_length and vocab_size."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    sd = {}
    for k, shp in clip_state_dict_shapes(cfg).items():
        if k == "logit_scale":
            t = torch.tensor(math.log(1 / 0.07))
        elif len(shp) == 1 and k.endswith(".weight"):  # LayerNorm scales
            t = 1.0 + 0.1 * torch.randn(shp, generator=g)
        elif len(shp) == 1 and k != "visual.class_embedding":
            t = 0.05 * torch.randn(shp, generator=g)
        elif k == "token_embedding.weight":
            t = 0.02 * torch.randn(shp, generator=g)
        elif k == "positional_embedding":
            t = 0.01 * torch.randn(shp, generator=g)
        elif k in ("visual.class_embedding", "visual.positional_embedding", "visual.proj"):
            t = cfg["vision_width"] ** -0.5 * torch.randn(shp, generator=g)
        elif k == "text_projection":
            t = cfg["text_width"] ** -0.5 * torch.randn(shp, generator=g)
        elif k == "visual.conv1.weight":
            t = (3 * cfg["patch_size"] ** 2) ** -0.5 * torch.randn(shp, generator=g)
        else:  # block matrices: in_proj / c_fc std width^-0.5, out_proj / c_proj scaled down with depth
            Wd = shp[1] if "c_proj" not in k else shp[0]
            n = cfg["vision_layers"] if k.startswith("visual.") else cfg["text_layers"]
            std = Wd ** -0.5 * ((2 * n) ** -0.5 if ("out_proj" in k or "c_proj" in k) else 1.0)
            t = std * torch.randn(shp, generator=g)
        sd[k] = t.to(dtype)
    sd["input_resolution"] = torch.tensor(cfg["image_resolution"])
    sd["context_length"] = torch.tensor(cfg["context_length"])
    sd["vocab_size"] = torch.tensor(cfg["vocab_size"])
    return sd


def make_clip_frames(cfg, n, seed=1):
    """uint8 [n, R, R, 3] RGB frames (smooth gradients plus noise, like decoded video rather than white noise)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    R = cfg["image_resolution"]
    yy, xx = torch.meshgrid(torch.linspace(0, 1, R), torch.linspace(0, 1, R), indexing="ij")
    ph = torch.rand(n, 3, generator=g)
    base = 0.5 + 0.35 * torch.sin(6.0 * (yy[None, None] * ph[:, :, None, None] + xx[None, None] * (1 - ph[:, :, None, None])) + 6.0 * ph[:, :, None, None])
    x = base + 0.1 * torch.randn(n, 3, R, R, generator=g)
    return (x.clamp(0, 1) * 255).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def make_clip_tokens(cfg, lengths, seed=2):
    """int64 [len(lengths), context_length] clip.tokenize-shaped rows: SOT, lengths[i] - 2 word ids, EOT, zero padding."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = torch.zeros(len(lengths), cfg["context_length"], dtype=torch.int64)
    for i, n in enumerate(lengths):
        assert 2 <= n <= cfg["context_length"]
        out[i, 0] = CLIP_SOT
        out[i, 1:n - 1] = torch.randint(1, CLIP_SOT, (n - 2,), generator=g)
        out[i, n - 1] = CLIP_EOT
    return out


# ---- query-focused video summarisation (main/dataset_qfvs.py) -------------------------------------------------------------
def make_qfvs_item(cfg, seed, S, Lf, seg_len, L1, L2):
    """One DatasetQFVS item (main/dataset_qfvs.py:125-208) with seeded contents: features [S, Lf, Dv - 2] zero beyond each
    segment's seg_len (segments past len(seg_len) are empty), the [S, Lf] bool mask_GT, per-shot 0/1 targets over the first
    sum(seg_len) shots of S * Lf entries (concept 1, concept 2 and the oracle summary), one positive shot index per target as
    a [1] float tensor ([0] when there is none), and two L2-normalised concept embeddings [L1, Dt] / [L2, Dt]."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    Dv, Dt = cfg["v_feat_dim"] - 2, cfg["t_feat_dim"]
    seg_len = torch.tensor(list(seg_len), dtype=torch.int64)
    mask = torch.zeros(S, Lf, dtype=torch.bool)
    for j, n in enumerate(seg_len.tolist()):
        mask[j, :n] = True
    feats = torch.randn(S, Lf, Dv, generator=g)
    feats = feats / (feats.norm(dim=-1, keepdim=True) + 1e-5) * mask[..., None]
    count = int(seg_len.sum())
    item = {"features": feats, "seg_len": seg_len, "mask_GT": mask}
    for name, key in (("concept1_GT", "saliency_pos_labels_1"), ("concept2_GT", "saliency_pos_labels_2"),
                      ("oracle_summary", "saliency_pos_labels_oracle")):
        t = torch.zeros(S * Lf)
        t[:count] = (torch.rand(count, generator=g) < 0.3).float()
        pos = torch.nonzero(t > 0).flatten()
        item[name] = t
        item[key] = torch.Tensor([float(pos[int(torch.randint(0, len(pos), (1,), generator=g))])]) if len(pos) else torch.Tensor(0)
    for key, L in (("tokens_pad1", L1), ("tokens_pad2", L2)):
        e = torch.randn(L, Dt, generator=g)
        item[key] = e / (e.norm(dim=-1, keepdim=True) + 1e-5)
    return item


def make_qfvs_batch(cfg, seed, S, Lf, seg_len, L1, L2):
    """start_end_collate_qfvs + prepare_batch_inputs_qfvs (main/dataset_qfvs.py:211-284) of make_qfvs_item(...), on the CPU:
    (inputs_1, inputs_2, inputs_oracle, targets_1, targets_2, targets_oracle, mask_GT).  The three inputs share the video
    src_vid [S, Lf, Dv] (features + the TEF columns of one Lf-frame segment, padded frames included) and src_vid_mask [S, Lf];
    the texts are concept 1 [S, L1, Dt], concept 2 [S, L2, Dt] and their concatenation [S, L1 + L2, Dt], each segment getting
    the same query.  Targets: saliency_scores [1, S * Lf], saliency_pos_labels [1, 1] (or [1, 0]), timestamp_mask = the video
    mask and timestamp_window = saliency_scores.  mask_GT: bool [1, S * Lf]."""
    it = make_qfvs_item(cfg, seed, S, Lf, seg_len, L1, L2)
    vmask = it["mask_GT"].float()
    tef_st = torch.arange(0, Lf, 1.0) / Lf
    tef = torch.stack([tef_st, tef_st + 1.0 / Lf], dim=1).repeat(S, 1, 1)
    src_vid = torch.cat([it["features"], tef], dim=-1)
    t1 = it["tokens_pad1"].float().repeat(S, 1, 1)
    t2 = it["tokens_pad2"].float().repeat(S, 1, 1)
    m1, m2 = torch.ones(S, L1), torch.ones(S, L2)
    inputs = [dict(src_vid=src_vid, src_vid_mask=vmask, src_txt=t, src_txt_mask=m)
              for t, m in ((t1, m1), (t2, m2), (torch.cat((t1, t2), dim=1), torch.cat((m1, m2), dim=1)))]
    targets = []
    for name, key in (("concept1_GT", "saliency_pos_labels_1"), ("concept2_GT", "saliency_pos_labels_2"),
                      ("oracle_summary", "saliency_pos_labels_oracle")):
        sal = it[name][None]
        targets.append(dict(saliency_scores=sal, saliency_pos_labels=it[key][None], timestamp_mask=vmask, timestamp_window=sal))
    return (*inputs, *targets, it["mask_GT"].reshape(1, -1))


# ---- evaluation submissions (eval/eval.py) --------------------------------------------------------------------------------
def _half(x):
    return struct.unpack("e", struct.pack("e", x))[0]


def _cross_iou(p, g):
    """eval/utils.py compute_temporal_iou_batch_cross for one pair, in the same double operations (0/0 -> NaN)."""
    inter = max(min(p[1], g[1]) - max(p[0], g[0]), 0.0)
    union = (p[1] - p[0]) + (g[1] - g[0]) - inter
    if union == 0:
        return math.nan
    return inter / union


def _ambiguous_gt_tie(rows, windows):
    """True when one of the first 10 predicted windows has equal IoU >= 0.5 (or NaN) with two different gt windows: the
    reference's gt visit order (numpy's default argsort) then depends on the machine."""
    for p in rows[:10]:
        seen = {}
        for g in windows:
            v = _cross_iou(p, g)
            key = "nan" if math.isnan(v) else v
            if key != "nan" and v < 0.5:
                continue
            if key in seen and seen[key] != tuple(g):
                return True
            seen[key] = tuple(g)
    return False


def make_eval_case(seed, n_queries=40, n_windows=10, durations=(150, 149, 148, 60), gt_lengths=(0, 2, 4, 10, 10, 14, 30, 30, 44, 90),
                   max_gt=4, sort_windows=True, match_number=True, tasks="mr+hl"):
    """A deterministic (Python `random`) submission / ground-truth pair in the format eval/eval.py:eval_submission reads.

    Ground truth per query: duration from `durations`; 1..max_gt windows [st, ed] on the 2 s clip grid with lengths from
    `gt_lengths` (0 = zero-length; 10 and 30 sit on the range edges), clipped to the duration; relevant_clip_ids (sometimes
    unsorted) covering the windows, with 3 annotator scores in 0..4 (some annotators all below 2 -> all-0 label columns; some
    queries cover every clip with one annotator at 4 -> all-1 columns).
    Submission per query: n_windows rows [st, ed, score] (some queries fewer than 5) rounded to 4 decimals like the decode, scores
    often multiples of 1/16 (ties), some rows copying or jittering a gt window, zero-length rows including one on a zero-length
    gt window (0/0 IoU); sorted by score (descending, stable) or, with sort_windows=False, in start order like --no_sort_results.
    pred_saliency_scores are fp16-rounded (or multiples of 1/16), sometimes longer or shorter than int(duration / 2).
    Queries whose first 10 rows tie two different gt windows at IoU >= 0.5 (or NaN) are redrawn.
    match_number=False: the two lists share only part of their qids.  tasks "mr" / "hl" leaves out pred_saliency_scores /
    pred_relevant_windows (the metrics of the other task are then skipped).
    Returns {"submission", "ground_truth", "match_number"}."""
    rng = random.Random(seed)
    sub, gt = [], []
    for qid in range(n_queries):
        while True:
            dur = rng.choice(durations)
            n_clips = int(dur / 2)
            windows = []
            for _ in range(rng.randint(1, max_gt) if rng.random() < 0.5 else 1):
                ln = min(rng.choice(gt_lengths), 2 * n_clips)
                st = 2 * rng.randint(0, (2 * n_clips - ln) // 2)
                windows.append([st, st + ln])
            if rng.random() < 0.1:
                windows.append(list(windows[0]))  # identical duplicate: harmless for the tie rule
            if rng.random() < 0.2:
                windows = [[float(s), float(e)] for s, e in windows]
            every = rng.random() < 0.06
            if every:
                clips = list(range(n_clips))
            else:
                clips = sorted({c for s, e in windows for c in range(int(s) // 2, min(int(e) // 2, n_clips))})
                if not clips:
                    clips = [rng.randrange(n_clips)]
            if rng.random() < 0.3:
                rng.shuffle(clips)
            low = rng.randrange(3) if rng.random() < 0.3 else -1
            scores = []
            for _ in clips:
                row = [rng.randint(0, 4) for _ in range(3)]
                if low >= 0:
                    row[low] = rng.randint(0, 1)
                if every:
                    row[(low + 1) % 3] = 4
                scores.append(row)
            n = rng.randint(1, 4) if rng.random() < 0.1 else n_windows
            rows = []
            for _ in range(n):
                u = rng.random()
                if u < 0.25:
                    s, e = rng.choice(windows)
                    if rng.random() < 0.5:
                        s, e = s + rng.uniform(-3, 3), e + rng.uniform(-3, 3)
                    s, e = min(max(s, 0.0), dur), min(max(e, 0.0), dur)
                    s, e = min(s, e), max(s, e)
                elif u < 0.3:
                    s = e = rng.uniform(0, dur)
                else:
                    s = rng.uniform(0, dur)
                    e = min(dur, s + rng.choice([2.0, 10.0, 30.0, rng.uniform(0, dur)]))
                sc = rng.randrange(17) / 16 if rng.random() < 0.5 else rng.random()
                rows.append([float(f"{s:.4f}"), float(f"{e:.4f}"), float(f"{sc:.4f}")])
            zero = [w for w in windows if w[0] == w[1]]
            if zero and rng.random() < 0.5:
                rows[rng.randrange(len(rows))][:2] = [float(zero[0][0]), float(zero[0][1])]  # 0/0 IoU
            if not _ambiguous_gt_tie(rows, windows):
                break
        if sort_windows:
            rows.sort(key=lambda r: -r[2])
        else:
            rows.sort(key=lambda r: r[0])
        n_sal = n_clips + (rng.choice([-3, -1, 1, 4]) if rng.random() < 0.2 else 0)
        if rng.random() < 0.3:
            sal = [rng.randrange(-16, 17) / 16 for _ in range(max(n_sal, 1))]
        else:
            sal = [_half(rng.uniform(-1, 1)) for _ in range(max(n_sal, 1))]
        gt.append(dict(qid=qid, query=f"query {qid}", duration=dur, vid=f"vid{qid}", relevant_windows=windows,
                       relevant_clip_ids=clips, saliency_scores=scores))
        pred = dict(qid=qid, query=f"query {qid}", vid=f"vid{qid}", pred_relevant_windows=rows, pred_saliency_scores=sal)
        if tasks == "mr":
            del pred["pred_saliency_scores"]
        elif tasks == "hl":
            del pred["pred_relevant_windows"]
        sub.append(pred)
    if not match_number:
        k = max(1, n_queries // 5)
        sub, gt = sub[k:], gt[:-k]
    return {"submission": sub, "ground_truth": gt, "match_number": match_number}


# ---- TVSum / YouTube highlight evaluation (main/dataset.py DatasetHL.evaluate) --------------------------------------------
class HLEvalDataset:
    """The part of the reference's DatasetHL that its evaluate() reads, in the 'val' state: dset_name, domain, label,
    get_video_id and get_saliency (the latter as main/dataset.py:828-851 computes it)."""

    def __init__(self, dset_name, domain, label, video_ids):
        self.dset_name, self.domain, self.label = dset_name, domain, label
        self.video_id = {"train": [], "val": list(video_ids)}
        self.state = "val"

    def get_video_id(self, idx):
        return self.video_id[self.state][idx]

    def get_saliency(self, idx):
        lab = self.label[self.get_video_id(idx)]
        if self.dset_name == "tvsum":
            s = torch.Tensor(lab["anno"])
            return torch.Tensor((s - s.mean()).mean(dim=1))
        return torch.Tensor([1 if s > 0 else 0 for s in lab["match"]])


def make_hl_eval_case(seed, dset_name="tvsum", n_videos=6, clips=(40, 75, 120, 17, 16, 3), shorter=0.3, batch=(1, 3),
                      tie_frac=0.5):
    """A deterministic (Python `random`) TVSum or YouTube evaluation input: the label dict of DatasetHL and the score blob
    eval_epoch collects.

    Video idx has a clip count from `clips`.  TVSum: `anno` [clips, 20] of integers 1..5 (some columns constant, so every label
    is 0; some with a few high values, so the top 5 holds few positives).  YouTube: `match` of -1 / 0 / 1 / 2 (some videos with
    no positive clip).  Blob entry idx is a [B, L] float32 tensor (B from `batch`) whose row 0 scores video idx: L is the clip
    count, or with probability `shorter` fewer clips.  With probability `tie_frac` a row's scores are multiples of 1/8 (many
    ties, in runs longer than 16 clips for long videos), else fp16-rounded uniforms.
    Returns {"dataset": HLEvalDataset, "blob": [tensor], "labels": [anno or match per video]}."""
    rng = random.Random(seed)
    label, ids, labels, blob = {}, [], [], []
    for idx in range(n_videos):
        n = clips[idx % len(clips)]
        vid = f"{dset_name}_{seed}_{idx}"
        meta = {"frames": 30 * 2 * n + rng.randrange(60), "fps": 30, "domain": "BK" if dset_name == "tvsum" else "dog"}
        if dset_name == "tvsum":
            anno = []
            kinds = [rng.random() for _ in range(20)]
            for _ in range(n):
                row = []
                for c in range(20):
                    if kinds[c] < 0.15:
                        row.append(3)
                    elif kinds[c] < 0.35:
                        row.append(5 if rng.random() < 0.1 else 1)
                    else:
                        row.append(rng.randint(1, 5))
                anno.append(row)
            meta.update(anno=anno, title=f"title {idx}")
            labels.append(anno)
        else:
            none = rng.random() < 0.15
            match = [rng.choice([-1, 0]) if none else rng.choice([-1, 0, 1, 1, 2]) for _ in range(n)]
            meta.update(match=match, clip=f"clip{idx}")
            labels.append(match)
        label[vid] = meta
        ids.append(vid)
        L = rng.randint(0, n) if rng.random() < shorter else n
        B = rng.randint(*batch)
        rows = []
        for _ in range(B):
            if rng.random() < tie_frac:
                rows.append([rng.randrange(-8, 9) / 8 for _ in range(L)])
            else:
                rows.append([_half(rng.uniform(-2, 2)) for _ in range(L)])
        blob.append(torch.tensor(rows, dtype=torch.float32).reshape(B, L))
    return {"dataset": HLEvalDataset(dset_name, "BK" if dset_name == "tvsum" else "dog", label, ids), "blob": blob,
            "labels": labels}


# ---- QFVS semantic matching (eval/qfvs.py calculate_semantic_matching) ----------------------------------------------------
def make_shot_tags(seed, n_shots, n_tags=48, max_set=31, zero_frac=0.01):
    """[n_shots, n_tags] uint8 0 / 1 with the statistics of the reference's Tags.mat: 1..max_set tags per shot, most shots with
    a few popular tags (so many pairs overlap and weights repeat), about zero_frac shots without any tag."""
    import numpy as np

    rng = random.Random(seed)
    popular = [1.0 / (c + 1) for c in range(n_tags)]
    order = list(range(n_tags))
    rng.shuffle(order)
    out = np.zeros((n_shots, n_tags), dtype=np.uint8)
    for i in range(n_shots):
        if rng.random() < zero_frac:
            continue
        k = min(max_set, 1 + int(rng.expovariate(1 / 4)))
        cols = set()
        while len(cols) < k:
            cols.add(order[rng.choices(range(n_tags), weights=popular)[0]])
        out[i, sorted(cols)] = 1
    return out


def make_qfvs_match_case(seed, n_shots, n_machine, n_gt, zero_frac=0.01):
    """Tags of one video and a machine / ground-truth summary pair (sorted shot indices, as topk + the oracle summary files
    give them; both may share shots).  Returns {"tags", "machine", "gt"}."""
    rng = random.Random(seed + 1)
    tags = make_shot_tags(seed, n_shots, zero_frac=zero_frac)
    machine = sorted(rng.sample(range(n_shots), n_machine))
    gt = sorted(rng.sample(range(n_shots), n_gt))
    return {"tags": tags, "machine": machine, "gt": gt}


def make_qfvs_permutation_case(seed, n, extra=0, n_tags=48):
    """A matching with a known optimum: n distinct non-empty tag sets built around a shared core (many pairs overlap heavily);
    the ground truth is the same n shots in a hidden order plus `extra` shots that overlap them less.  Identical pairs weigh 1
    and every other pair less, so the maximum total weight is exactly n.  Returns {"tags", "machine", "gt", "optimum"}."""
    import numpy as np

    rng = random.Random(seed)
    core = rng.sample(range(n_tags), 8)
    seen, rows = set(), []
    while len(rows) < n + extra:
        cols = frozenset(rng.sample(core, rng.randint(3, 6)) + rng.sample(range(n_tags), rng.randint(1, 6)))
        if cols not in seen:
            seen.add(cols)
            rows.append(sorted(cols))
    tags = np.zeros((n + extra, n_tags), dtype=np.uint8)
    for i, cols in enumerate(rows):
        tags[i, cols] = 1
    gt = list(range(n + extra))
    rng.shuffle(gt)
    return {"tags": tags, "machine": list(range(n)), "gt": gt, "optimum": float(n)}


# ---- CLIP-teacher pseudo labels (teacher/clip2label.py) ------------------------------------------------------------------
TEACHER_SPECIAL_NAMES = ("Sprenger's tulip", "Crème brûlée", 'A "quoted" name', "Back\\slash")


def _teacher_unsafe(feat, cls64, dup_rows, topk, th):
    """True when the CPU reference could disagree with the float64 labels on this video: a top-(k+1) class is a duplicated row
    (CPU torch.sort is not stable), two distinct top-(k+1) sums lie within 1e-5 T, or a top-(k+1) cosine (other than an exact
    0) lies within 1e-6 of a bin edge."""
    import numpy as np

    v = feat.astype(np.float64)
    v = v / np.maximum(np.linalg.norm(v, axis=1, keepdims=True), 1e-8)
    mm = v @ cls64.T
    s = mm.sum(0)
    top = np.argsort(-s, kind="stable")[:topk + 1]
    if dup_rows.intersection(top.tolist()):
        return True
    st = np.sort(s[top])
    if (np.diff(st) < 1e-5 * len(feat)).any():
        return True
    x = mm[:, top]
    edge = np.abs(x - np.round(x / th) * th)
    return bool(((edge < 1e-6) & (x != 0)).any())


def make_teacher_case(seed, n_classes=300, dim=64, n_videos=12, clips=(2, 60), lengths=(), dup=0, dup_top=False, copies=0,
                      edges=True, parallel=True, safe=False, topk=5, th=0.05):
    """Seeded inputs of the CLIP-teacher labelling: a class table, class names and videos whose clips mix a few class
    directions (Gaussian bumps over time) with noise, so the curves have peaks and windows.

    n_videos random videos with T drawn from `clips`, then one per entry of `lengths`; with `edges` also T = 1 (always
    skipped), a ramp whose maximum is only at the last clip, identical clips (all-equal curves), a video with zero rows, and
    (`parallel`) one whose clips are exact multiples of a class row (cosine 1, bin 19 at th 0.05).  `dup` class rows copy
    others (the OIDv6 list has 12 duplicated names); with `dup_top` the first video is about a duplicated row, so the copy
    and the original tie inside its top-k.  `copies` more rows copy the first video's main class.  With `safe`, videos are
    redrawn until the CPU reference cannot disagree (_teacher_unsafe), duplicated rows stay out of every top-(k+1), and
    parallel / dup_top / copies are refused.  Returns {"classes", "names", "features", "vids", "dup_rows"}."""
    import numpy as np

    if safe and (parallel and edges or dup_top or copies):
        raise ValueError("make_teacher_case: safe cases cannot have parallel clips, dup_top or copies")
    rng = np.random.default_rng(seed)
    C, D = n_classes, dim
    cls = (rng.standard_normal((C, D)) * rng.uniform(0.5, 2.0, (C, 1))).astype(np.float32)
    names = [f"class {i}" for i in range(C)]
    for i, n in enumerate(TEACHER_SPECIAL_NAMES[:C]):
        names[i] = n
    dup_rows = set()
    src_dup = None
    if dup:
        rows = rng.choice(C, 2 * dup, replace=False)
        for s, d in zip(rows[:dup], rows[dup:]):
            cls[d] = cls[s]
            names[d] = names[s]
            dup_rows.update((int(s), int(d)))
        src_dup = int(rows[0])
    main = None
    if copies:
        main = int(rng.integers(C))
        others = rng.choice(np.setdiff1d(np.arange(C), [main]), copies, replace=False)
        cls[others] = cls[main]
        for o in others:
            names[int(o)] = names[main]
    cls64 = cls.astype(np.float64)
    cls64 /= np.maximum(np.linalg.norm(cls64, axis=1, keepdims=True), 1e-8)
    unit = cls64.astype(np.float32)
    allowed = np.setdiff1d(np.arange(C), sorted(dup_rows)) if safe else np.arange(C)

    def mix(T, topics=None, noise=None):
        k = len(topics) if topics is not None else min(int(rng.integers(1, 4)), len(allowed))
        if topics is None:
            topics = rng.choice(allowed, k, replace=False)
        t = np.arange(T)[:, None]
        mu, sd = rng.uniform(0, T, k), rng.uniform(1.0, max(2.0, T / 3), k)
        w = rng.uniform(0.5, 2.0, k) * np.exp(-(t - mu) ** 2 / (2 * sd ** 2)) + rng.uniform(0.0, 0.5, k)
        sig = rng.uniform(0.3, 1.0) if noise is None else noise
        x = w @ unit[topics] + sig * rng.standard_normal((T, D)) / math.sqrt(D)
        return (x * rng.uniform(5.0, 15.0)).astype(np.float32)

    specs = [("rand", int(rng.integers(clips[0], clips[1] + 1))) for _ in range(n_videos)] + [("rand", int(T)) for T in lengths]
    if edges:
        specs += [("one", 1), ("ramp", 12), ("equal", 8), ("zero", 20)] + ([("parallel", 10)] if parallel else [])
    feats, vids = [], []
    for i, (kind, T) in enumerate(specs):
        for _ in range(200):
            if kind == "one":
                f = mix(1)
            elif kind == "ramp":
                c = rng.choice(allowed)
                f = ((np.arange(T)[:, None] + 1.0) * unit[c] + 0.3 * rng.standard_normal((T, D)) / math.sqrt(D)).astype(np.float32)
            elif kind == "equal":
                f = np.repeat(mix(1), T, axis=0)
            elif kind == "zero":
                f = mix(T)
                f[[3, 7, 8]] = 0.0
            elif kind == "parallel":
                c = int(rng.choice(allowed))
                f = mix(T, topics=np.array([c]))
                f[2:5] = cls[c] * 2.0
            elif i == 0 and dup_top:
                f = mix(T, topics=np.array([src_dup]), noise=0.3)
            elif i == 0 and copies:
                f = mix(T, topics=np.array([main]), noise=0.3)
            else:
                f = mix(T)
            if not safe or not _teacher_unsafe(f, cls64, dup_rows, topk, th):
                break
        else:
            raise RuntimeError(f"make_teacher_case: no safe draw for video {i} ({kind}, T={T})")
        feats.append(f)
        vids.append(f"v{seed}_{i:04d}_{kind}")
    return {"classes": cls, "names": names, "features": feats, "vids": vids, "dup_rows": sorted(dup_rows)}


def teacher_case_sha256(case):
    import hashlib
    import json

    h = hashlib.sha256(case["classes"].tobytes())
    h.update(json.dumps([case["names"], case["vids"]]).encode())
    for f in case["features"]:
        h.update(str(f.shape).encode())
        h.update(f.tobytes())
    return h.hexdigest()
