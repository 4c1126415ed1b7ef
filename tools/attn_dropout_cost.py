#!/usr/bin/env python
"""Cost of attention dropout (args.dropout) in the training step: forward + criterion + backward + FlatAdamW at the cfg2/cfg3
shape (B = 32, Lv = 75, Lt = 32) and the cfg4 shape (Lv = 150), with p = 0 and p = 0.1 timed alternately (input dropout 0.5
and DropPath 0.1 on in both arms, as in bench.py's train line).

Per arm and round it reports the step time from CUDA events and, from one profiled step (profile_train_step), the summed time
of the attention launches (kind 2: the forward and backward attention kernels).  The GPU's name and power limit are read
(nvidia-smi query, read-only) in the same run and stored with the numbers.  Writes results/attn_dropout_cost.json.

    python tools/attn_dropout_cost.py [--rounds 3] [--steps 30] [--warmup 5]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from univtg_b200 import build_model, synth  # noqa: E402
from univtg_b200.optim import FlatAdamW  # noqa: E402


def gpu_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        info["nvidia_smi"] = q
    except (OSError, subprocess.SubprocessError, IndexError):
        info["nvidia_smi"] = "unavailable"
    return info


def make_arm(cfg, p, dev):
    model, crit = build_model(synth.reference_args(cfg, device=str(dev), dropout=p))
    model.load_state_dict(synth.make_state_dict(cfg, seed=0), strict=True)
    model.to(dev).train()
    crit.to(dev).train()
    opt = FlatAdamW(model, lr=1e-4, weight_decay=1e-4, max_grad_norm=0.1, zero_grad_after_step=True)
    return model, crit, opt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attn_dropout_cost.py needs a GPU")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    result = {"gpu": gpu_info(), "steps": args.steps, "rounds": args.rounds, "shapes": {}}
    for shape in ("cfg2", "cfg4"):
        cfg = synth.CONFIGS[shape]
        B, Lv, Lt = cfg["batch"], cfg["l_vid"], cfg["l_txt"]
        raw = [synth.make_inputs(cfg, seed=20 + i, ragged=True) for i in range(3)]
        inps = [{k: v.to(dev) for k, v in r.items()} for r in raw]
        tgts = [{k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in synth.make_targets(r, seed=21 + i).items()}
                for i, r in enumerate(raw)]
        arms = {p: make_arm(cfg, p, dev) for p in (0.0, 0.1)}

        def step(arm, i):
            model, crit, opt = arm
            out = model(**inps[i % 3])
            total = crit.weighted_total(crit(out, tgts[i % 3]))
            opt.zero_grad()
            total.backward()
            opt.step()

        for arm in arms.values():
            for i in range(args.warmup):
                step(arm, i)
        torch.cuda.synchronize()
        rec = {str(p): {"ms_per_step": [], "attention_ms": []} for p in arms}
        for _ in range(args.rounds):
            for p, arm in arms.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(args.steps):
                    step(arm, i)
                e1.record()
                torch.cuda.synchronize()
                rec[str(p)]["ms_per_step"].append(e0.elapsed_time(e1) / args.steps)
                model, crit, _ = arm

                def run():
                    out = model(**inps[0])
                    crit.weighted_total(crit(out, tgts[0])).backward()

                tl = model.profile_train_step(B, Lv, Lt, run)
                rec[str(p)]["attention_ms"].append(sum(ms for kind, ms in tl if kind == 2))
                arm[2].zero_grad()
        rec["shape"] = {"B": B, "Lv": Lv, "Lt": Lt, "L": Lv + Lt, "hidden_dim": cfg["hidden_dim"], "nheads": cfg["nheads"],
                        "enc_layers": cfg["enc_layers"]}
        result["shapes"][shape] = rec
        for p in ("0.0", "0.1"):
            print(f"{shape} p={p}: step ms {['%.3f' % v for v in rec[p]['ms_per_step']]}  attention ms "
                  f"{['%.3f' % v for v in rec[p]['attention_ms']]}")
        del arms
        torch.cuda.empty_cache()
    print("gpu:", result["gpu"])
    out_dir = os.path.join(ROOT, "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "attn_dropout_cost.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
