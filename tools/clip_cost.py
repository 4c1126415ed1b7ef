"""Time the CLIP feature extractor (univtg_b200.clip) against torch fp16 eager, on one GPU, in one call.

    python tools/clip_cost.py [--reps 20] [--json out.json]

ViT-B/32 shapes with seeded weights (univtg_b200.synth).  encode_image at T = 1, 32 and 300 frames (300 = a 10-minute video at
clip_len 2) and encode_text at N = 1 and 64 queries.  The eager arm is the oracle's towers run by torch in fp16 on the same GPU
(the reference's convert_weights execution), both frame by frame - one encode_image call per frame, as vid2clip runs it - and
batched.  Every shape of every arm is warmed up first; the arms then alternate, each timed with CUDA events around one call.
Both arms' outputs are compared with the fp64 oracle at every timed size.  The GPU's name and power limit are read in the same call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import clip_oracle as CO  # noqa: E402
from univtg_b200 import clip, synth  # noqa: E402


def gpu_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # the number is still reported, marked as such
        info["power_limit"] = f"unavailable ({e})"
    return info


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def rel_err(got, ref):
    return float((got.double() - ref.double()).abs().max() / ref.double().abs().max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "clip_cost.py measures on a GPU; there is no CPU measurement"
    dev = "cuda:0"
    cfg = synth.CLIP_CONFIGS["vit_b32"]
    sd = synth.make_clip_state_dict(cfg, seed=0)
    enc = clip.ClipEncoder.from_state_dict(sd, operand_format="fp16").to(dev)
    sd16 = {k: v.to(dev, torch.float16) for k, v in sd.items() if v.is_floating_point()}
    result = {"gpu": gpu_info(), "config": "vit_b32", "operand_format": "fp16", "reps": args.reps, "image": {}, "text": {}}

    cases = []
    for T in (1, 32, 300):
        frames = synth.make_clip_frames(cfg, T, seed=T).to(dev)
        images = CO.preprocess(frames)
        arms = {
            "ours": lambda f=frames: enc.encode_image(f),
            "eager_per_frame": lambda im=images: torch.cat([CO.encode_image(sd16, cfg, im[i:i + 1], dtype=torch.float16)
                                                            for i in range(im.shape[0])]),
            "eager_batched": lambda im=images: CO.encode_image(sd16, cfg, im, dtype=torch.float16),
        }
        cases.append(("image", T, arms, lambda im=images: CO.encode_image(sd, cfg, im)))
    for N in (1, 64):
        g = torch.Generator().manual_seed(N)
        tokens = synth.make_clip_tokens(cfg, [int(x) for x in torch.randint(2, 33, (N,), generator=g)], seed=N).to(dev)
        arms = {
            "ours": lambda t=tokens: enc.encode_text(t)["pooler_output"],
            "eager_batched": lambda t=tokens: CO.encode_text(sd16, cfg, t, dtype=torch.float16)["pooler_output"],
        }
        cases.append(("text", N, arms, lambda t=tokens: CO.encode_text(sd, cfg, t)["pooler_output"]))

    with torch.no_grad():
        for _, _, arms, _ in cases:  # warm-up of every shape of every arm
            for fn in arms.values():
                fn()
                fn()
        for kind, n, arms, exact_fn in cases:
            times = {k: [] for k in arms}
            for _ in range(args.reps):
                for k, fn in arms.items():  # alternating arms
                    times[k].append(timed(fn)[0])
            exact = exact_fn()
            row = {}
            for k, fn in arms.items():
                row[k] = {"median_ms": statistics.median(times[k]), "min_ms": min(times[k]), "max_ms": max(times[k]),
                          "max_rel_err_vs_fp64": rel_err(fn(), exact)}
            ours = row["ours"]["median_ms"]
            for k in arms:
                if k != "ours":
                    row[k]["ours_speedup"] = row[k]["median_ms"] / ours
            result[kind][str(n)] = row
            print(kind, n, json.dumps(row), flush=True)
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
