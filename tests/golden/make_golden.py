#!/usr/bin/env python
"""Generate tests/golden/*.npz by running the UNMODIFIED reference (model/univtg.py of a showlab/UniVTG checkout) on CPU fp32.

Usage:  python tests/golden/make_golden.py <path to a showlab/UniVTG checkout>
Weights and synthetic inputs are regenerated from seeds by univtg_b200.synth, so a fixture stores only the seeds, the
outputs, the five losses and per-parameter gradient summaries.  cfg1 additionally stores the reference's demo features
(tmp/vid.npz, tmp/txt.npz) pre-processed as main_gradio.py:58-80 does.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = os.path.abspath(sys.argv[1])
sys.path.insert(0, REF)

from univtg_b200 import synth  # noqa: E402
from model.univtg import build_model  # noqa: E402  (the reference)

OUT = os.path.dirname(os.path.abspath(__file__))
OUT_KEYS = ("pred_logits", "pred_spans", "saliency_scores", "vid_mem_proj", "txt_mem_proj")


def demo_inputs():
    """Reference demo inputs, as main_gradio.load_data prepares them."""
    vid = np.load(os.path.join(REF, "tmp", "vid.npz"))["features"].astype(np.float32)
    txt = np.load(os.path.join(REF, "tmp", "txt.npz"))["features"].astype(np.float32)
    vid = torch.from_numpy(vid)
    txt = torch.from_numpy(txt)
    vid = vid / (vid.norm(dim=-1, keepdim=True) + 1e-5)  # utils/basic_utils.py:97-99
    txt = txt / (txt.norm(dim=-1, keepdim=True) + 1e-5)
    n = vid.shape[0]
    tef = torch.stack([torch.arange(n) / n, (torch.arange(n) + 1) / n], dim=1)
    vid = torch.cat([vid, tef], dim=1)
    return dict(src_txt=txt[None].contiguous(), src_txt_mask=torch.ones(1, txt.shape[0]), src_vid=vid[None].contiguous(),
                src_vid_mask=torch.ones(1, n))


def run_case(name, cfg_name, seed, ragged, batch=None, demo=False, head_gain=1.0, with_grads=True):
    cfg = synth.CONFIGS[cfg_name]
    args = synth.reference_args(cfg, droppath=0.0, input_dropout=0.0)
    model, crit = build_model(args)
    sd = synth.make_state_dict(cfg, seed=seed, head_gain=head_gain)
    model.load_state_dict(sd, strict=True)
    inp = demo_inputs() if demo else synth.make_inputs(cfg, seed=seed + 1, ragged=ragged, batch=batch)
    tgt = synth.make_targets(inp, seed=seed + 2)
    model.eval()
    with torch.no_grad():
        out = model(**inp)
    save = {"meta_cfg": cfg_name, "meta_seed": seed, "meta_ragged": int(ragged), "meta_batch": inp["src_vid"].shape[0],
            "meta_head_gain": head_gain, "meta_demo": int(demo)}
    # keep fixtures small: large vid_mem_proj tensors are stored at every `stride`-th clip
    stride = 1 if out["vid_mem_proj"].numel() <= 200_000 else 15
    save["meta_vid_stride"] = stride
    for k in OUT_KEYS:
        v = out[k]
        save["out_" + k] = (v[:, ::stride] if k == "vid_mem_proj" else v).numpy()
    if demo:
        for k, v in inp.items():
            save["in_" + k] = v.numpy()
    # losses + gradients: train() with droppath = input_dropout = dropout = 0 is deterministic
    model.train()
    crit.train()
    out = model(**inp)
    loss = crit(out, tgt)
    for k, v in loss.items():
        save["loss_" + k] = np.float64(float(v))
    if with_grads:
        total = sum(loss[k] * crit.weight_dict[k] for k in loss if k in crit.weight_dict)
        save["loss_total"] = np.float64(float(total))
        total.backward()
        for n_, p in model.named_parameters():
            if p.grad is None:
                continue
            gflat = p.grad.flatten()
            save["gnorm_" + n_] = np.float64(float(gflat.double().norm()))
            save["ghead_" + n_] = gflat[:16].numpy().copy()
    np.savez_compressed(os.path.join(OUT, name + ".npz"), **save)
    print("wrote", name, {k: float(v) for k, v in loss.items()})


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    run_case("tiny_ragged", "tiny", seed=10, ragged=True)
    run_case("tiny_full", "tiny", seed=20, ragged=False, head_gain=4.0)
    run_case("cfg1_demo", "cfg1", seed=30, ragged=False, demo=True)
    run_case("cfg2_b4_ragged", "cfg2", seed=40, ragged=True, batch=4)
    run_case("cfg2_full", "cfg2", seed=50, ragged=False)  # the benchmarked B=32 shape, with gradient summaries
    run_case("cfg4_b4_ragged", "cfg4", seed=60, ragged=True, batch=4)  # L = 182: two key tiles in attention
