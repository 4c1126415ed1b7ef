"""Time one query-focused video summarisation training step (main/train_qfvs.py:179-204) on one GPU, in one call.

    python tools/qfvs_cost.py [--steps 10] [--warmup 3] [--json out.json]

The step: three train-mode forwards sharing one video (concept 1, concept 2 and their concatenation as queries), three criterion
calls with mask_GT, the gathered loss (qfvs_loss_gather = 1), one backward and an AdamW step.  Shape: S = 20 segments of
Lf = 200 frames (the reference's max_segment_num x max_frame_num) with the last segment ragged, cfg2 model dims.  Dv = 2818 and
L1 = L2 = 8 concept tokens are assumptions: the dims of the released QFVS features and the concept token counts are not checked.
Arms, alternated step by step after a warm-up of each: this library (univtg_b200.qfvs, FlatAdamW) and the oracle port
(oracle/univtg_oracle.py + oracle/qfvs_oracle.py) run by torch eager in fp32 on the same GPU with torch.optim.AdamW.  Each step is
timed with CUDA events; the medians are reported with the GPU's name and power limit, read in the same call.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from clip_cost import gpu_info, timed  # noqa: E402
from oracle import qfvs_oracle as QO  # noqa: E402
from oracle import univtg_oracle as O  # noqa: E402
from univtg_b200 import synth  # noqa: E402
from univtg_b200.optim import FlatAdamW  # noqa: E402
from univtg_b200.qfvs import build_model  # noqa: E402

S, LF, SEG_LEN, L1, L2 = 20, 200, (200,) * 19 + (137,), 8, 8


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "qfvs_cost.py measures on a GPU; there is no CPU measurement"
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = "cuda:0"
    cfg = synth.CONFIGS["cfg2"]
    batch = synth.make_qfvs_batch(cfg, 5, S, LF, SEG_LEN, L1, L2)
    inputs = [{k: v.to(dev) for k, v in d.items()} for d in batch[:3]]
    targets = [{k: v.to(dev) for k, v in d.items()} for d in batch[3:6]]
    mask = batch[6].to(dev)
    sd = synth.make_state_dict(cfg, seed=4)

    model, crit = build_model(synth.reference_args(cfg, device=dev, dset_type="vs", droppath=0.0, input_dropout=0.0))
    model.load_state_dict(sd, strict=True)
    model.to(dev).train()
    crit.to(dev)
    opt = FlatAdamW(model, lr=1e-6, weight_decay=1e-4, max_grad_norm=0.1)

    def ours():
        dicts = [crit(model(**inp), tg, mask) for inp, tg in zip(inputs, targets)]
        total = sum(sum(d[k] for d in dicts) * crit.weight_dict[k] for k in dicts[0])
        opt.zero_grad()
        total.backward()
        opt.step()
        return total.detach()

    params = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
    eager_opt = torch.optim.AdamW(list(params.values()), lr=1e-6, weight_decay=1e-4)

    def eager():
        dicts = [QO.criterion(O.forward(params, cfg, **inp, dtype=torch.float32), tg, mask) for inp, tg in zip(inputs, targets)]
        total = O.weighted_total(QO.gather(dicts, 1), crit.weight_dict)
        eager_opt.zero_grad()
        total.backward()
        torch.nn.utils.clip_grad_norm_(list(params.values()), 0.1)
        eager_opt.step()
        return total.detach()

    arms = {"ours": ours, "torch_fp32_eager_oracle": eager}
    first = {}
    for name, fn in arms.items():
        for i in range(args.warmup):
            v = fn()
            if i == 0:
                first[name] = float(v)
    ms = {name: [] for name in arms}
    for _ in range(args.steps):
        for name, fn in arms.items():
            ms[name].append(timed(fn)[0])
    result = {"gpu": gpu_info(), "shape": {"S": S, "Lf": LF, "seg_len_last": SEG_LEN[-1], "L1": L1, "L2": L2, "config": "cfg2"},
              "steps": args.steps, "warmup": args.warmup,
              "step_ms_median": {k: statistics.median(v) for k, v in ms.items()},
              "step_ms_min_max": {k: [min(v), max(v)] for k, v in ms.items()},
              "first_step_gathered_loss": first}
    result["speedup_vs_eager"] = result["step_ms_median"]["torch_fp32_eager_oracle"] / result["step_ms_median"]["ours"]
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
