#!/usr/bin/env python
"""Writes tests/golden/reference_qfvs.npz: the UNMODIFIED UniVTG query-focused video summarisation path on CPU, fp32.

  * the prepared inputs of a seeded DatasetQFVS item (univtg_b200.synth.make_qfvs_item) after the reference's own
    start_end_collate_qfvs + prepare_batch_inputs_qfvs (main/dataset_qfvs.py:211-284);
  * one step of main/train_qfvs.py:179-204 at the `tiny` config with S = 4 segments of Lf = 24 frames (the last one ragged),
    concept queries of L1 = 3 and L2 = 5 tokens and all dropouts 0: the three loss dicts of model/univtg_qfvs.py's
    SetCriterion, the total with qfvs_loss_gather on, and the gradients of a few named parameters;
  * criterion-only edge cases on seeded outputs (pred_logits, saliency_scores as leaves): an all-zero target, positives at and
    beyond the kept count, no saliency_pos_labels, and pred_logits exactly 0 and 1 (BCE's log clamp at -100), each with the
    losses and the gradients of both outputs.

The reference moves tensors with .cuda() and .to('cuda'); both are redirected to the CPU, nothing else is changed.  h5py and
nncore (imported by main/dataset_qfvs.py, unused here) are stubbed.  Weights and the raw item are regenerated from the seeds
below, so the file holds the reference's prepared inputs and results only.
Usage:  python tests/golden/make_golden_qfvs.py <path to a showlab/UniVTG checkout>"""
import copy
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(sys.argv[1])
sys.dont_write_bytecode = True
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from univtg_b200 import synth  # noqa: E402

CFG = "tiny"
WEIGHT_SEED, ITEM_SEED, EDGE_SEED = 31, 32, 33
S, LF, SEG_LEN, L1, L2 = 4, 24, (24, 24, 24, 10), 3, 5
GRADS = ("weightedpool.weight", "input_vid_proj.0.net.1.weight", "input_txt_proj.0.LayerNorm.weight",
         "transformer.encoder.layers.1.norm2.weight", "token_type_embeddings.weight", "class_embed.layers.2.weight")


def _stub_dataset_deps():
    sys.modules["h5py"] = types.ModuleType("h5py")
    nn_ = types.ModuleType("nncore")
    ds = types.ModuleType("nncore.dataset")

    class _Registry:
        def register(self, *a, **k):
            return lambda c: c

    ds.DATASETS = _Registry()
    par = types.ModuleType("nncore.parallel")
    par.DataContainer = object
    nn_.dataset, nn_.parallel = ds, par
    sys.modules.update({"nncore": nn_, "nncore.dataset": ds, "nncore.parallel": par})


def _cpu(a):
    return "cpu" if isinstance(a, (str, torch.device)) and str(a).startswith("cuda") else a


_to = torch.Tensor.to
torch.Tensor.cuda = lambda self, *a, **k: self
torch.Tensor.to = lambda self, *a, **k: _to(self, *[_cpu(x) for x in a], **{n: _cpu(v) for n, v in k.items()})
_stub_dataset_deps()

from main.dataset_qfvs import prepare_batch_inputs_qfvs, start_end_collate_qfvs  # noqa: E402
from model.univtg_qfvs import build_model  # noqa: E402  (the reference)

arrays, meta = {}, {"cfg": CFG, "seeds": [WEIGHT_SEED, ITEM_SEED, EDGE_SEED], "S": S, "Lf": LF, "seg_len": list(SEG_LEN),
                    "L1": L1, "L2": L2, "grads": list(GRADS)}


def _losses(d):
    return {k: float(v) for k, v in d.items()}


# ---- prepared inputs ----
cfg = synth.CONFIGS[CFG]
item = synth.make_qfvs_item(cfg, ITEM_SEED, S, LF, SEG_LEN, L1, L2)
prepared = prepare_batch_inputs_qfvs(start_end_collate_qfvs([item]), {})
inputs, targets, mask_GT = prepared[:3], prepared[3:6], prepared[6]
assert inputs[1]["src_vid"] is inputs[0]["src_vid"] and inputs[2]["src_vid"] is inputs[0]["src_vid"]
arrays["in/src_vid"] = inputs[0]["src_vid"].numpy()
arrays["in/src_vid_mask"] = inputs[0]["src_vid_mask"].numpy()
for q, inp in zip(("1", "2", "oracle"), inputs):
    arrays[f"in/{q}/src_txt"] = inp["src_txt"].numpy()
    arrays[f"in/{q}/src_txt_mask"] = inp["src_txt_mask"].numpy()
for q, tg in zip(("1", "2", "oracle"), targets):
    for k, v in tg.items():
        arrays[f"tgt/{q}/{k}"] = v.numpy()
arrays["mask_GT"] = mask_GT.numpy()

# ---- one training step (qfvs_loss_gather = 1) ----
args = synth.reference_args(cfg, dset_type="vs", dropout=0.0, droppath=0.0, input_dropout=0.0)
model, crit = build_model(args)
meta["crit_losses"] = list(crit.losses)
model.load_state_dict(synth.make_state_dict(cfg, seed=WEIGHT_SEED), strict=True)
model.train()
crit.train()
outs = [model(**inp) for inp in inputs]
dicts = [crit(o, copy.copy(t), mask_GT) for o, t in zip(outs, targets)]
meta["step/losses"] = [_losses(d) for d in dicts]
loss_dict = {k: dicts[0][k] + dicts[1][k] + dicts[2][k] for k in dicts[0]}
total = sum(loss_dict[k] * crit.weight_dict[k] for k in loss_dict.keys() if k in crit.weight_dict)
meta["step/total_gather"] = float(total)
meta["step/total_oracle_only"] = float(sum(dicts[2][k] * crit.weight_dict[k] for k in dicts[2] if k in crit.weight_dict))
total.backward()
named = dict(model.named_parameters())
for k in GRADS:
    arrays[f"grad/{k}"] = named[k].grad.numpy()

# ---- criterion-only edge cases ----
g = torch.Generator().manual_seed(EDGE_SEED)
count = int(mask_GT.sum())
base = targets[2]
edge_pl = torch.sigmoid(2.0 * torch.randn(S, LF, 1, generator=g))
edge_sal = torch.tanh(torch.randn(S, LF, generator=g)) + torch.log(inputs[0]["src_vid_mask"] + 1e-45)
kept = torch.nonzero(mask_GT.reshape(-1)).flatten()
clamp_pl = edge_pl.clone().reshape(-1)
t_or = base["saliency_scores"][0]
for j in range(4):  # exactly 0 and exactly 1 on kept positions with targets 0 and 1
    clamp_pl[kept[int(torch.nonzero(t_or[:count] == j % 2).flatten()[j])]] = float(j // 2)
beyond = torch.zeros_like(base["saliency_scores"])
beyond[0, count - 3:count + 5] = 1.0  # three positives inside the kept count, five at or beyond it
beyond[0, -1] = 1.0
CASES = {
    "all_zero": (edge_pl, dict(base, saliency_scores=torch.zeros_like(base["saliency_scores"]))),
    "beyond_count": (edge_pl, dict(base, saliency_scores=beyond)),
    "no_pos_labels": (edge_pl, {k: v for k, v in base.items() if k != "saliency_pos_labels"}),
    "clamp": (clamp_pl.reshape(S, LF, 1), base),
}
meta["edge_cases"] = list(CASES)
for name, (pl, tg) in CASES.items():
    arrays[f"edge/{name}/pred_logits"] = pl.numpy()
    arrays[f"edge/{name}/saliency_scores_target"] = tg["saliency_scores"].numpy()
    pl_leaf = pl.clone().requires_grad_(True)
    sal_leaf = edge_sal.clone().requires_grad_(True)
    d = crit({"pred_logits": pl_leaf, "saliency_scores": sal_leaf}, copy.copy(tg), mask_GT)
    meta[f"edge/{name}/losses"] = _losses(d)
    tot = sum(d[k] * crit.weight_dict[k] for k in d if k in crit.weight_dict)
    if torch.is_tensor(tot) and tot.requires_grad:
        tot.backward()
    for k, leaf in (("pred_logits", pl_leaf), ("saliency_scores", sal_leaf)):
        arrays[f"edge/{name}/grad_{k}"] = (leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)).numpy()
arrays["edge/saliency_scores"] = edge_sal.numpy()

arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
np.savez_compressed(os.path.join(HERE, "reference_qfvs.npz"), **arrays)
print("wrote", os.path.getsize(os.path.join(HERE, "reference_qfvs.npz")), "bytes:", sorted(k for k in arrays if k != "meta"))
