#!/usr/bin/env python
"""Writes tests/golden/reference_loss_edges.npz: the UNMODIFIED UniVTG SetCriterion (model/univtg.py, model_id univtg, losses
spans / labels / saliency, eos_coef as given, temperature 0.07) on CPU in fp32, on the edge batches of tests/loss_ref.mr_case:
GIoU and smooth-L1 ties, saturated pred_logits (p in {0, 1, 2^-24, 1 - 2^-24}), duplicate and masked positives, saliency ties,
B = 1, B = 33, no foreground clip, no valid clip, no saliency_pos_labels, all-zero saliency and eos_coef 0.5.

For each batch the file holds its inputs (so the pinned tests do not depend on the generator), the five losses and the gradients
of sum_k w_k loss_k (w = 10, 1, 10, 0.1, 0.1) w.r.t. pred_logits, pred_spans, vid_mem_proj and txt_mem_proj (NaN where the
reference's are).  Data only.
Usage:  python tests/golden/make_golden_loss_edges.py <path to a showlab/UniVTG checkout>"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(sys.argv[1])
sys.dont_write_bytecode = True
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from tests import loss_ref as R  # noqa: E402
from model.univtg import SetCriterion  # noqa: E402  (the reference)

# name: (B, Lv, d, seed, edges, eos_coef)
CASES = {
    "giou_ties": (2, 40, 64, 501, ("giou", "sal_ties"), 0.1),
    "bce_saturated": (2, 40, 64, 502, ("bce",), 0.1),
    "bce_saturated_eos05": (3, 24, 64, 503, ("bce", "giou"), 0.5),
    "positives": (8, 24, 64, 504, ("pos", "sal_ties"), 0.1),
    "b1": (1, 1, 64, 505, ("pos",), 0.1),
    "b1_l16": (1, 16, 64, 506, ("giou", "bce"), 0.1),
    "b33": (33, 12, 64, 507, ("pos", "giou", "bce", "sal_ties"), 0.1),
    "no_fg": (4, 24, 64, 508, ("no_fg", "pos"), 0.1),
    "no_valid": (4, 24, 64, 509, ("no_valid",), 0.1),
    "no_pos": (4, 24, 64, 510, ("no_pos", "giou"), 0.1),
    "sal_zero": (4, 24, 64, 511, ("sal_zero", "bce"), 0.1),
    "mixed_eos05": (5, 30, 128, 512, ("giou", "bce", "pos", "sal_ties"), 0.5),
}
W = dict(zip(R.LOSS_NAMES, R.TRAIN_W))

arrays, meta = {}, {"cases": {}, "weights": list(R.TRAIN_W)}
for name, (B, Lv, d, seed, edges, eos) in CASES.items():
    c = R.mr_case(B, Lv, d, seed, edges, eos)
    crit = SetCriterion(None, W, eos, ["spans", "labels", "saliency"], 0.07, "l1", 75)
    leaves = {"pred_logits": c["pred_logits"].unsqueeze(-1).clone().requires_grad_(True),
              "pred_spans": c["pred_spans"].clone().requires_grad_(True),
              "vid_mem_proj": c["vid_mem_proj"].clone().requires_grad_(True),
              "txt_mem_proj": c["txt_mem_proj"].unsqueeze(1).clone().requires_grad_(True)}
    tg = {"timestamp": c["timestamp"], "timestamp_mask": c["timestamp_mask"], "timestamp_window": c["timestamp_window"],
          "span_labels_nn": c["span_labels_nn"], "saliency_scores": c["saliency_scores"]}
    if c["pos"] is not None:
        tg["saliency_pos_labels"] = c["pos"].unsqueeze(1)
    losses = crit(dict(leaves), tg)
    total = sum(losses[k] * W[k] for k in losses)
    total.backward()
    for k, v in c.items():
        if torch.is_tensor(v):
            arrays[f"{name}/in/{k}"] = v.numpy()
    for k, v in leaves.items():
        g = v.grad if v.grad is not None else torch.zeros_like(v)  # no saliency term: vid / txt get no gradient
        arrays[f"{name}/grad/{k}"] = g.reshape(c[k].shape).numpy()  # pred_logits [B, Lv], txt_mem_proj [B, d]
    meta["cases"][name] = {"B": B, "Lv": Lv, "d": d, "seed": seed, "edges": list(edges), "eos_coef": eos,
                           "losses": {k: float(v.detach() if torch.is_tensor(v) else v) for k, v in losses.items()}}

arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
out = os.path.join(HERE, "reference_loss_edges.npz")
np.savez_compressed(out, **arrays)
print("wrote", os.path.getsize(out), "bytes")
