#!/usr/bin/env python
"""Writes tests/golden/reference_attn_dropout.npz: the UNMODIFIED UniVTG model's train-mode outputs and five losses with
attention dropout on (args.dropout = p in nn.MultiheadAttention, model/transformer_encoder_droppath.py:93) and every other
source of randomness off (droppath = 0, input_dropout = 0), after torch.manual_seed(seed).  tests/test_attention_dropout_cpu.py
re-draws the same masks (F.dropout on ones of [B*H, L, L], one per encoder layer, in layer order) and pins the oracle's
attn_masks semantics to these outputs.  Inputs are regenerated from seeds by univtg_b200.synth, so the file holds only
reference outputs.  Usage:  python tests/golden/make_golden_attn_dropout.py <path to a showlab/UniVTG checkout>"""
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

OUT = ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj")
# (config, batch, p, torch seed): tiny has dh = 128, cfg1 dh = 32; both with ragged masks
CASES = [("tiny", 4, 0.1, 41), ("tiny", 4, 0.3, 42), ("cfg1", 3, 0.1, 43), ("cfg1", 3, 0.3, 44)]

arrays, meta = {}, {"cases": CASES}
for cfg_name, batch, p, seed in CASES:
    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=21)
    model, crit = build_model(synth.reference_args(cfg, dropout=p, droppath=0.0, input_dropout=0.0))
    model.load_state_dict(sd, strict=True)
    model.train()
    inp = synth.make_inputs(cfg, seed=22, ragged=True, batch=batch)
    tgt = synth.make_targets(inp, seed=23)
    torch.manual_seed(seed)
    with torch.no_grad():  # train mode: the dropout draws happen all the same
        out = model(**inp)
    name = f"{cfg_name}_p{p}"
    meta[f"{name}/losses"] = {k: float(v) for k, v in crit(out, tgt).items()}
    for k in OUT:
        arrays[f"{name}/{k}"] = out[k].detach().float().numpy()

arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
np.savez_compressed(os.path.join(HERE, "reference_attn_dropout.npz"), **arrays)
print("wrote", sorted(k for k in arrays if k != "meta"))
