#!/usr/bin/env python
"""Cost of the strict inference mode (operand_format="fp16x3"): eval forwards at the cfg2 shape (B = 32) and the cfg5 shape, fp16
and fp16x3 timed alternately, beside the fp32 torch-eager forward of the oracle port (TF32 off, bench.oracle_step_fn) at cfg2 on
the same GPU - the speed a user gives up, and the only other way to reproduce the fp32 reference's numbers.

Times come from CUDA events around `--steps` forwards per arm and round.  The GPU's name and power limit are read (nvidia-smi
query, read-only) in the same run and stored with the numbers.  Writes results/strict_cost.json.

    python tools/strict_cost.py [--rounds 3] [--steps 30] [--warmup 5]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import bench  # noqa: E402
from txt_pos_cost import gpu_info, timed  # noqa: E402
from univtg_b200 import build_model, synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("strict_cost.py needs a GPU")
    dev = torch.device("cuda", 0)
    result = {"gpu": gpu_info(), "steps": args.steps, "rounds": args.rounds, "runs": {}}
    for shape in ("cfg2", "cfg5"):
        cfg = synth.CONFIGS[shape]
        inps = [{k: v.to(dev) for k, v in synth.make_inputs(cfg, seed=20 + i, ragged=True).items()} for i in range(3)]
        arms = {}
        for fmt in ("fp16", "fp16x3"):
            model, _ = build_model(synth.reference_args(cfg, device=str(dev), operand_format=fmt))
            model.load_state_dict(synth.make_state_dict(cfg, seed=0), strict=True)
            arms[fmt] = model.to(dev).eval()

        def step(model, i):
            with torch.no_grad():
                model(**inps[i % 3])

        for model in arms.values():
            for i in range(args.warmup):
                step(model, i)
        torch.cuda.synchronize()
        rec = {fmt: [] for fmt in arms}
        for _ in range(args.rounds):
            for fmt, model in arms.items():
                rec[fmt].append(timed(lambda i, m=model: step(m, i), args.steps))
        rec["shape"] = {"B": cfg["batch"], "Lv": cfg["l_vid"], "Lt": cfg["l_txt"], "hidden_dim": cfg["hidden_dim"],
                        "enc_layers": cfg["enc_layers"]}
        rec["ratio_fp16x3_over_fp16"] = min(rec["fp16x3"]) / min(rec["fp16"])
        if shape == "cfg2":
            old = torch.backends.cuda.matmul.allow_tf32
            torch.backends.cuda.matmul.allow_tf32 = False
            try:
                eager = bench.oracle_step_fn(cfg, "fwd", cfg["batch"], device=dev)
                for _ in range(3):
                    eager()
                torch.cuda.synchronize()
                rec["fp32_eager"] = [timed(lambda i: eager(), max(3, args.steps // 3)) for _ in range(args.rounds)]
            finally:
                torch.backends.cuda.matmul.allow_tf32 = old
        result["runs"][shape + "_eval"] = rec
        print(f"{shape}_eval: " + "  ".join(f"{k} {['%.3f' % v for v in rec[k]]}" for k in ("fp16", "fp16x3", "fp32_eager") if k in rec))
        del arms
        torch.cuda.empty_cache()
    print("gpu:", result["gpu"])
    out_dir = os.path.join(ROOT, "results")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "strict_cost.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
