#!/usr/bin/env python
"""Cost of learned text positions (args.use_txt_pos): the training step (forward + criterion + backward + FlatAdamW) at the cfg2
shape (B = 32, Lv = 75, Lt = 32) and the cfg4 shape (Lv = 150), and the cfg2 eval forward, with the feature off and on timed
alternately (the reference's defaults in both arms: input dropout 0.5, DropPath 0.1, attention dropout 0.1 in training).

Times come from CUDA events around `--steps` steps per arm and round.  The GPU's name and power limit are read (nvidia-smi query,
read-only) in the same run and stored with the numbers.  Writes results/txt_pos_cost.json.

    python tools/txt_pos_cost.py [--rounds 3] [--steps 30] [--warmup 5]"""
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


def make_arm(cfg, on, dev, train):
    model, crit = build_model(synth.reference_args(cfg, device=str(dev), dropout=0.1, use_txt_pos=on))
    model.load_state_dict(synth.make_state_dict(cfg, seed=0), strict=True)
    model.to(dev).train(train)
    crit.to(dev).train(train)
    opt = FlatAdamW(model, lr=1e-4, weight_decay=1e-4, max_grad_norm=0.1, zero_grad_after_step=True) if train else None
    return model, crit, opt


def timed(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("txt_pos_cost.py needs a GPU")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    result = {"gpu": gpu_info(), "steps": args.steps, "rounds": args.rounds, "runs": {}}
    for shape, train in (("cfg2", True), ("cfg4", True), ("cfg2", False)):
        cfg = synth.CONFIGS[shape]
        raw = [synth.make_inputs(cfg, seed=20 + i, ragged=True) for i in range(3)]
        inps = [{k: v.to(dev) for k, v in r.items()} for r in raw]
        tgts = [{k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in synth.make_targets(r, seed=21 + i).items()}
                for i, r in enumerate(raw)]
        arms = {on: make_arm(cfg, on, dev, train) for on in (False, True)}

        def step(arm, i):
            model, crit, opt = arm
            if not train:
                with torch.no_grad():
                    model(**inps[i % 3])
                return
            out = model(**inps[i % 3])
            total = crit.weighted_total(crit(out, tgts[i % 3]))
            opt.zero_grad()
            total.backward()
            opt.step()

        for arm in arms.values():
            for i in range(args.warmup):
                step(arm, i)
        torch.cuda.synchronize()
        rec = {("on" if on else "off"): [] for on in arms}
        for _ in range(args.rounds):
            for on, arm in arms.items():
                rec["on" if on else "off"].append(timed(lambda i, arm=arm: step(arm, i), args.steps))
        name = f"{shape}_{'train' if train else 'eval'}"
        rec["shape"] = {"B": cfg["batch"], "Lv": cfg["l_vid"], "Lt": cfg["l_txt"], "hidden_dim": cfg["hidden_dim"],
                        "enc_layers": cfg["enc_layers"]}
        result["runs"][name] = rec
        print(f"{name}: ms off {['%.3f' % v for v in rec['off']]}  on {['%.3f' % v for v in rec['on']]}")
        del arms
        torch.cuda.empty_cache()
    print("gpu:", result["gpu"])
    out_dir = os.path.join(ROOT, "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "txt_pos_cost.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
