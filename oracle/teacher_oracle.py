"""fp64 restatement of the CLIP-teacher pseudo labelling (reference teacher/clip2label.py), written from the math.

Per video with T >= 1 clips (clip2label.py:64-65 skips T = 0):
  * sim_matrix (11-19): cos[t, c] = (v_t / max(||v_t||, 1e-8)) . (c / max(||c||, 1e-8)), here in float64;
  * the ranking key (66-68) is sum_t cos[t, c]; the top-k come from a *stable* descending sort, so equal sums keep the lower
    class index first;
  * each chosen class's curve (72-73) is float32(cos[t, c]) // th with Python's float floor division;
  * create_window (22-37) returns every run of clips equal to the curve's maximum as [i * clip_len, (j + 1) * clip_len]; a run
    that reaches the last clip is never appended, and a class without windows writes no line (86-87);
  * each line is json.dumps of the sample dict in the reference's key order (76-89).
Videos are emitted in the order given (the reference's order is that of a Python set), lines in rank order.
Works on torch tensors on any device; CUDA callers get the same float64 math on the GPU.
"""
import json

import numpy as np
import torch


def cosines(vid, cls):
    """float64 [T, C] cosine matrix of clip features vid [T, D] and class features cls [C, D]."""
    v = torch.as_tensor(vid).double()
    c = torch.as_tensor(cls).double().to(v.device)
    vn = v / v.norm(dim=1, keepdim=True).clamp_min(1e-8)
    cn = c / c.norm(dim=1, keepdim=True).clamp_min(1e-8)
    return vn @ cn.T


def create_window(score, clip_len):
    """Runs of the maximum of `score` (a list of floats) that end before the last clip."""
    mx = max(score)
    res, start = [], None
    for i, s in enumerate(score):
        if s == mx:
            if start is None:
                start = i
        elif start is not None:
            res.append([start * clip_len, i * clip_len])
            start = None
    return res


def label_video(vid_feat, cls, names, vid, topk=5, th=0.05, clip_len=2, mm=None):
    """The sample dicts of one video, in rank order (skipped classes left out)."""
    T = len(vid_feat)
    if T == 0:
        return []
    if mm is None:
        mm = cosines(vid_feat, cls)
    order = torch.sort(mm.sum(0), descending=True, stable=True)[1][:topk].tolist()
    curves = mm[:, order].float().T.cpu().tolist()
    out = []
    for c, curve in zip(order, curves):
        score = [[s // th] for s in curve]
        window = create_window([s[0] for s in score], clip_len)
        if not window:
            continue
        out.append({"qid": c, "query": names[c], "duration": float(T * clip_len), "vid": vid,
                    "relevant_clip_ids": list(range(T)), "relevant_windows": window, "saliency_scores": score})
    return out


def label(features, vids, cls, names, topk=5, th=0.05, clip_len=2):
    """Samples of every video, videos in the given order."""
    out = []
    for f, vid in zip(features, vids):
        out.extend(label_video(f, cls, names, vid, topk, th, clip_len))
    return out


def lines(samples):
    return [json.dumps(s) for s in samples]


def reference_loop_fp32(features, cls, topk=5, device="cuda"):
    """The reference's per-video device work in float32 (sim_matrix, sum, full sort, top-k) - for timing comparisons only."""
    c = torch.as_tensor(np.asarray(cls)).to(device)
    cn = c / torch.max(c.norm(dim=1)[:, None], 1e-8 * torch.ones_like(c[:, :1]))
    res = []
    for f in features:
        v = torch.as_tensor(np.asarray(f)).to(device)
        if len(v) == 0:
            continue
        vn = v / torch.max(v.norm(dim=1)[:, None], 1e-8 * torch.ones_like(v[:, :1]))
        mm = vn @ cn.T
        idx = torch.sort(mm.sum(0), descending=True)[1][:topk]
        res.append((idx.tolist(), mm.T[idx].tolist()))
    return res
