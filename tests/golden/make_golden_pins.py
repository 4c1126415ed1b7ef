#!/usr/bin/env python
"""Writes tests/golden/reference_pins.npz: what the UNMODIFIED UniVTG code computes for the checks that pin the oracle, the
decode restatement, the plugin boundary and the data loader to it (tests/test_oracle_vs_reference.py, tests/test_postproc.py,
tests/test_data_cpu.py).  Inputs are regenerated from seeds by univtg_b200.synth and the tests' own helpers, so the file holds
only reference outputs.  Usage:  python tests/golden/make_golden_pins.py <path to a showlab/UniVTG checkout>"""
import json
import os
import random
import sys
import tempfile
import types
from argparse import Namespace
from pathlib import Path

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.abspath(sys.argv[1])
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

from univtg_b200 import synth  # noqa: E402

OUT = ("pred_logits", "pred_spans", "saliency_scores", "vid_mem_proj", "txt_mem_proj")
arrays, meta = {}, {}


def ref_model(cfg, sd, **over):
    from model.univtg import build_model

    model, crit = build_model(synth.reference_args(cfg, **over))
    model.load_state_dict(sd, strict=True)
    return model, crit


def put(prefix, out, keys=OUT):
    for k in keys:
        arrays[f"{prefix}/{k}"] = out[k].detach().float().numpy()


def losses(ld):
    return {k: float(v) for k, v in ld.items()}


# ---- forward + losses (tests/test_oracle_vs_reference.py::test_forward_and_losses) ----
for cfg_name, ragged, batch in (("tiny", True, None), ("tiny", False, 5), ("cfg1", True, 3)):
    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=123)
    model, crit = ref_model(cfg, sd)
    model.eval()
    inp = synth.make_inputs(cfg, seed=7, ragged=ragged, batch=batch)
    tgt = synth.make_targets(inp, seed=8)
    with torch.no_grad():
        ref = model(**inp)
        meta[f"fwd_{cfg_name}_{ragged}_{batch}/losses"] = losses(crit(ref, tgt))
    put(f"fwd_{cfg_name}_{ragged}_{batch}", ref)

# ---- bool masks of the highlight path ----
cfg = synth.CONFIGS["tiny"]
sd = synth.make_state_dict(cfg, seed=11)
model, _ = ref_model(cfg, sd)
model.eval()
inp = synth.make_inputs(cfg, seed=3, ragged=True, batch=4)
as_bool = dict(inp, src_vid_mask=inp["src_vid_mask"].bool(), src_txt_mask=inp["src_txt_mask"].bool())
with torch.no_grad():
    put("bool_float", model(**inp))
    put("bool_bool", model(**as_bool))

# ---- DropPath in train mode ----
sd = synth.make_state_dict(cfg, seed=5)
model, _ = ref_model(cfg, sd, droppath=0.3, input_dropout=0.0)
model.train()
inp = synth.make_inputs(cfg, seed=9, ragged=True, batch=6)
torch.manual_seed(77)
put("droppath", model(**inp), ("pred_logits", "pred_spans"))

# ---- state_dict keys and shapes ----
for name in ("tiny", "cfg1"):
    c = synth.CONFIGS[name]
    m, _ = ref_model(c, synth.make_state_dict(c))
    meta[f"state_dict/{name}"] = [[k, list(v.shape)] for k, v in m.state_dict().items()]

# ---- input dropout in train mode ----
model, crit = ref_model(cfg, sd, droppath=0.0, input_dropout=0.5)
model.train()
tgt = synth.make_targets(inp, seed=10)
torch.manual_seed(31)
ref = model(**inp)
meta["input_dropout/losses"] = losses(crit(ref, tgt))
put("input_dropout", ref, ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj"))

# ---- highlight-detection loss list ----
model, crit = ref_model(cfg, sd, dset_type="hl")
meta["hl/crit_losses"] = list(crit.losses)
model.eval()
full = synth.make_targets(inp, seed=10)
tgt = {"saliency_scores": full["saliency_scores"], "saliency_pos_labels": full["saliency_pos_labels"],
       "timestamp_mask": full["timestamp_mask"], "timestamp_window": 1 * (full["saliency_scores"] > 0)}
with torch.no_grad():
    meta["hl/losses"] = losses(crit(model(**inp), tgt))


# ---- the evaluation loop's decode (main/inference_mr.py compute_mr_results) ----
def stub_dataset_deps():
    if "h5py" not in sys.modules:
        sys.modules["h5py"] = types.ModuleType("h5py")
    if "nncore" not in sys.modules:
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


stub_dataset_deps()
import main.inference_mr as M  # noqa: E402
sys.path.insert(0, ROOT)
from tests.test_oracle_vs_reference import decode_case  # noqa: E402

for sort in (True, False):
    outputs, ts, vmask, durs, B, Lt = decode_case()

    class FakeModel:
        def eval(self):
            return self

        def __call__(self, **kw):
            return {k: v.clone() for k, v in outputs.items()}

    Lv = vmask.shape[1]
    batch_meta = [{"qid": i, "query": "q", "vid": "v", "duration": durs[i]} for i in range(B)]
    batch = {"query_feat": (torch.zeros(B, Lt, 4), torch.ones(B, Lt)), "video_feat": (torch.zeros(B, Lv, 4), vmask),
             "timestamp": (ts, vmask), "timestamp_window": (torch.zeros(B, Lv),), "span_labels_nn": (torch.zeros(B, Lv, 2),)}
    opt = Namespace(device="cpu", pin_memory=False, span_loss_type="l1", model_id="univtg", eval_mode=None,
                    no_sort_results=not sort, debug=False, round_multiple=0, clip_length=2)
    res, _ = M.compute_mr_results(FakeModel(), [(batch_meta, batch)], opt)
    meta[f"decode/{sort}"] = [{"pred_relevant_windows": r["pred_relevant_windows"], "pred_saliency_scores": r["pred_saliency_scores"]}
                              for r in res]

# ---- main.config.setup_model with --model_id univtg: what an optimizer / scheduler / criterion built the reference way sees ----
import main.config as cfgmod  # noqa: E402


class _CpuDevice(str):  # the reference reads opt.device both as torch.device(opt.device) and as int(opt.device) >= 0
    def __int__(self):
        return -1


extra = dict(device=_CpuDevice("cpu"), gpu_id=0, lr=1e-4, wd=1e-4, lr_warmup=[10], lr_drop=400, lr_gamma=0.1, resume=None, resume_all=False)
torch.manual_seed(0)
m_ref, c_ref, o_ref, s_ref = cfgmod.setup_model(synth.reference_args(cfg, model_id="univtg", **extra))
meta["setup_model"] = {
    "named_parameters": [[n, list(p.shape)] for n, p in m_ref.named_parameters() if p.requires_grad],
    "optimizer_shapes": [list(p.shape) for p in o_ref.param_groups[0]["params"]],
    "weight_dict": {k: float(v) for k, v in c_ref.weight_dict.items()},
    "losses": list(c_ref.losses),
    "scheduler": type(s_ref).__name__,
    "optimizer": type(o_ref).__name__,
}

# ---- temporal NMS on seeded random windows (utils/temporal_nms.py) ----
from utils.temporal_nms import temporal_nms as ref_nms  # noqa: E402

rng = random.Random(3)
nms = []
for _ in range(300):
    n = rng.choice([0, 1, 2, 5, 10, 40])
    rows = []
    for _ in range(n):
        st = round(rng.uniform(0, 100), 4)
        rows.append([st, round(st + rng.choice([0.0, rng.uniform(0, 50)]), 4), round(rng.choice([0.0, rng.random()]), 4)])
    thd, ma = rng.choice([0.1, 0.5, 0.7, 0.9]), rng.choice([1, 3, 10, 100])
    nms.append({"rows": rows, "nms_thd": thd, "max_after_nms": ma, "expected": ref_nms([list(r) for r in rows], thd, ma)})
meta["nms_random"] = nms

# ---- feature preparation + collate of the data loader (main/dataset.py, utils/tensor_utils.py) ----
from utils.basic_utils import l2_normalize_np_array  # noqa: E402
from utils.tensor_utils import pad_sequences_1d  # noqa: E402

from tests.test_data_cpu import _fake_corpus  # noqa: E402

with tempfile.TemporaryDirectory() as tmp:
    v_dirs, q_dir, anns = _fake_corpus(Path(tmp), seed=5)
    ref_v, ref_q = [], []
    for ann in anns[:6]:
        fl = [l2_normalize_np_array(np.load(os.path.join(d, f"{ann['vid']}.npz"))["features"].astype(np.float32)) for d in v_dirs]
        n = min(len(e) for e in fl)
        v = torch.from_numpy(np.concatenate([e[:n] for e in fl], axis=1))
        st = torch.arange(0, n, 1.0) / n
        ref_v.append(torch.cat([v, torch.stack([st, st + 1.0 / n], dim=1)], dim=1))
        ref_q.append(torch.from_numpy(l2_normalize_np_array(
            np.load(os.path.join(q_dir, f"{ann['qid']}.npz"))["last_hidden_state"].astype(np.float32))))
    for key, seqs in (("vid", ref_v), ("txt", ref_q)):
        pad, mask = pad_sequences_1d(seqs, dtype=torch.float32, fixed_length=None)
        arrays[f"collate/{key}"] = pad.numpy()
        arrays[f"collate/{key}_mask"] = mask.numpy()

arrays["meta"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)  # UTF-8 JSON
out = os.path.join(HERE, "reference_pins.npz")
np.savez_compressed(out, **arrays)
print("wrote", out, os.path.getsize(out), "bytes")
