"""Restatement of the reference's QFVS evaluation epoch (main/inference_qfvs.py eval_epoch) on any device, one file at a time.

The model runs once per query variant and file (the reference runs it again for each output type of the ensemble; every model
here is deterministic, so once is the same), scores are masked_select / add / slice / torch.topk on the model's device, and
the matching is oracle.task_eval_oracle.semantic_matching (exact Hungarian; s is the float64 sum of the matched weights, so it
agrees with networkx's hash-ordered sum to the last bits only).  Returns the JSONL lines in file order and the {'F','R','P'}."""
import json
import os
import pickle

import numpy as np
import torch

from oracle import task_eval_oracle as TO
from univtg_b200 import synth
from univtg_b200.qfvs import SUMMARY_DIR, TRANSFER, l2_normalize_np_array, load_videos_tag, output_type

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_qfvs_eval.json")


def golden_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def eval_epoch(model, config, opt, root, device="cpu"):
    """Per-file epoch in the tree at root -> (lines [(file, line)], result dict)."""
    video_id = config["test_videos"][0]
    with open(os.path.join(root, f"data/qfvs/txt_clip/{config['txt_feature']}.pkl"), "rb") as f:
        emb = pickle.load(f)
    h5 = synth.h5py_stub().File(os.path.join(root, f"data/qfvs/processed/P0{video_id}_{config['vid_feature']}.h5"))
    feats = torch.from_numpy(h5["features"][()]).to(torch.float32)
    seg_len = h5["seg_len"][()]
    S, Lf = config["max_segment_num"], config["max_frame_num"]
    mask = torch.zeros(S, Lf, dtype=torch.bool)
    for j, n in enumerate(seg_len.tolist()):
        mask[j, :n] = True
    mask = mask.to(device)
    tef_st = torch.arange(0, Lf, 1.0) / Lf
    vid = torch.cat([feats, torch.stack([tef_st, tef_st + 1.0 / Lf], 1).repeat(S, 1, 1)], -1).to(device)
    vmask = mask.float()
    tags = load_videos_tag(os.path.join(root, "eval/Tags.mat"))[video_id - 1]
    mode = output_type(opt, config)
    keys = {0: ["pred_logits"], 1: ["saliency_scores"], 2: ["pred_logits", "saliency_scores"]}[mode]
    d = os.path.join(root, SUMMARY_DIR + str(video_id))
    files = [x for _, _, fs in os.walk(d) for x in fs]
    lines, f1_sum, r_sum, p_sum = [], 0, 0, 0
    for file in files:
        with open(os.path.join(d, file)) as f:
            gt = [int(x.strip()) - 1 for x in f.readlines()]
        c1, c2 = (TRANSFER.get(c, c) for c in file.split("_")[0:2])
        t1, t2 = (torch.from_numpy(l2_normalize_np_array(emb[c])).to(torch.float32).to(device) for c in (c1, c2))
        scores = []
        for t in (t1, t2, torch.cat([t1, t2])):
            out = model(src_txt=t[None].repeat(S, 1, 1), src_txt_mask=torch.ones(S, t.shape[0], device=device), src_vid=vid,
                        src_vid_mask=vmask)
            if mode == 2:
                sc = torch.zeros(int(mask.sum()), device=device)
                for k in keys:
                    sc += out[k].squeeze().masked_select(mask)
            else:
                sc = out[keys[0]].squeeze().masked_select(mask)
            scores.append(sc)
        score = scores[2] + scores[0] + scores[1] if config["qfvs_score_gather"] > 0 else scores[2]
        score = score[:min(score.shape[0], tags.shape[0])]
        _, top = score.topk(int(score.shape[0] * config["top_percent"]))
        _, s, p, r, f1 = TO.semantic_matching(top.cpu().numpy(), gt, tags)
        lines.append((file, json.dumps({"concept1": c1, "concept2": c2, "score": score.tolist(), "top_percent": config["top_percent"],
                                        "top_pred": top.tolist(), "gt": gt, "p": p, "r": r, "f1": f1, "shots": tags.shape[0]})))
        f1_sum += f1
        r_sum += r
        p_sum += p
    n = len(files)
    return lines, {"F": round(100 * f1_sum / n, 2), "R": round(100 * r_sum / n, 2), "P": round(100 * p_sum / n, 2)}


def assert_line_matches(got, want, what):
    """p, r and f1 within 1e-12 relative (NaN equal to NaN), every other field byte-identical."""
    g, w = json.loads(got), json.loads(want)
    for k in ("p", "r", "f1"):
        a, b = g.pop(k), w.pop(k)
        assert (np.isnan(a) and np.isnan(b)) or abs(a - b) <= 1e-12 * abs(b), f"{what} {k}: {a} vs {b}"
    assert json.dumps(g) == json.dumps(w), f"{what}: fields other than p, r, f1 differ"


def assert_result_matches(got, want, what):
    g, w = (json.loads(x) if isinstance(x, str) else x for x in (got, want))
    for k in ("F", "R", "P"):
        assert (np.isnan(g[k]) and np.isnan(w[k])) or g[k] == w[k], f"{what} {k}: {g[k]} vs {w[k]}"
