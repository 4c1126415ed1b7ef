#!/usr/bin/env python
"""Writes tests/golden/reference_txt_pos.npz: the UNMODIFIED UniVTG model with use_txt_pos = True (learned text positions,
model/univtg.py:123, model/position_encoding.py:19-41) on CPU:
  * eval outputs;
  * train-mode outputs and the five losses with input_dropout = 0.5 (droppath = 0, dropout = 0) after torch.manual_seed(seed);
  * the autograd gradients of that train-mode loss (weight_dict-weighted sum) w.r.t. the three txt_position_embed tensors and
    token_type_embeddings.weight.
tests/test_txt_pos_cpu.py re-draws the train-mode masks with F.dropout on ones in the reference's order (video projector layers,
text projector layers, then the text positions [B, Lt, d]) and pins tests/txt_pos_oracle.py to these numbers.  Inputs are
regenerated from seeds by univtg_b200.synth, so the file holds only reference outputs.
Usage:  python tests/golden/make_golden_txt_pos.py <path to a showlab/UniVTG checkout>"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(sys.argv[1])
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from univtg_b200 import synth  # noqa: E402
from model.univtg import build_model  # noqa: E402  (the reference)

OUT = ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj", "saliency_scores")
GRADS = ("txt_position_embed.position_embeddings.weight", "txt_position_embed.LayerNorm.weight",
         "txt_position_embed.LayerNorm.bias", "token_type_embeddings.weight")
# (config, batch, torch seed): tiny has dh = 128, cfg1 dh = 32; both with ragged masks
CASES = [("tiny", 4, 51), ("cfg1", 3, 52)]

arrays, meta = {}, {"cases": CASES}
for cfg_name, batch, seed in CASES:
    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=21)
    model, crit = build_model(synth.reference_args(cfg, use_txt_pos=True, dropout=0.0, droppath=0.0, input_dropout=0.5))
    model.load_state_dict(sd, strict=True)
    inp = synth.make_inputs(cfg, seed=22, ragged=True, batch=batch)
    tgt = synth.make_targets(inp, seed=23)
    model.eval()
    with torch.no_grad():
        ev = model(**inp)
    for k in OUT:
        arrays[f"{cfg_name}/eval/{k}"] = ev[k].detach().float().numpy()
    model.train()
    torch.manual_seed(seed)
    out = model(**inp)
    losses = crit(out, tgt)
    meta[f"{cfg_name}/losses"] = {k: v.item() for k, v in losses.items()}
    for k in OUT:
        arrays[f"{cfg_name}/train/{k}"] = out[k].detach().float().numpy()
    sum(losses[k] * crit.weight_dict[k] for k in losses).backward()
    named = dict(model.named_parameters())
    for k in GRADS:
        arrays[f"{cfg_name}/grad/{k}"] = named[k].grad.detach().float().numpy()

arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
np.savez_compressed(os.path.join(HERE, "reference_txt_pos.npz"), **arrays)
print("wrote", sorted(k for k in arrays if k != "meta"))
