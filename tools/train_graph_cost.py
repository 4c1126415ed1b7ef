"""What replaying the training step from a CUDA graph (univtg_b200.graphs.GraphedTrainStep) saves per step, on one GPU, in one call.

    python tools/train_graph_cost.py [--steps 240] [--block 20] [--json train_graph_cost.json]

Workload: the benchmark's cfg3_train (synth config "cfg2": d = 1024, 4 layers, Lv = 75) at B = 32 and at B = 8, FlatAdamW with
dynamic loss scaling, the reference's dropout defaults (input 0.5, DropPath 0.1, attention 0.1).  Text lengths are ragged:
every sample draws its length uniformly from [Lt / 5, Lt] (synth.make_inputs(ragged=True), Lt = 32) and the batch is padded
to its longest sample, as the collate does; 12 such batches rotate, so each padded length gets its own graph.

Per batch size, after one warm-up pass over every batch in both modes (which captures every graph), the two modes alternate
in blocks of --block steps until each has run --steps steps; each block is timed with CUDA events around its steps (the GPU
queue is never drained inside a block), so a block's time is what the step costs end to end: host launch work where the
GPU waits for it, GPU work otherwise.  Reported: ms per step of each mode (median block and all blocks pooled), the saving,
the capture time of each graph, the number of graphs and the bytes of the workspace they share.  The GPU's name, power
limit and SM clocks are read in the same call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from univtg_b200 import build_model, synth  # noqa: E402
from univtg_b200.graphs import GraphedTrainStep  # noqa: E402
from univtg_b200.optim import FlatAdamW  # noqa: E402


def gpu_info():
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["sm_clock"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # the numbers are still reported, marked as such
        info["power_limit"] = f"unavailable ({e})"
    return info


def make_batches(cfg, B, n, seed):
    g = torch.Generator().manual_seed(seed)
    Lt = cfg["l_txt"]
    out = []
    for i in range(n):
        lens = torch.randint(max(2, Lt // 5), Lt + 1, (B,), generator=g)
        raw = synth.make_inputs(cfg, seed=seed + i, ragged=True, batch=B, l_txt=int(lens.max()))
        tgt = synth.make_targets(raw, seed=seed + 100 + i)
        out.append(({k: v.cuda() for k, v in raw.items()}, {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in tgt.items()}))
    return out


def run(B, steps, block, n_batches=12):
    cfg = synth.CONFIGS["cfg2"]
    model, crit = build_model(synth.reference_args(cfg, device="cuda:0", dropout=0.1, droppath=0.1, input_dropout=0.5))
    model.load_state_dict(synth.make_state_dict(cfg, seed=0), strict=True)
    model.to("cuda:0").train()
    crit.to("cuda:0")
    opt = FlatAdamW(model, lr=1e-4, weight_decay=1e-4, max_grad_norm=0.1)
    batches = make_batches(cfg, B, n_batches, seed=1000 + B)
    shapes = sorted({tuple(b[0]["src_txt"].shape[:2]) for b in batches})
    gs = GraphedTrainStep(model, crit, opt, max_graphs=len(shapes))

    def eager(inp, tgt):
        out = model(**inp)
        total = crit.weighted_total(crit(out, tgt))
        opt.zero_grad()
        total.backward()
        opt.step()

    def graphed(inp, tgt):
        gs(inp, tgt)

    i = 0
    for fn in (eager, graphed, eager, graphed):  # warm-up: every shape in both modes, every graph captured
        for inp, tgt in batches:
            fn(inp, tgt)
    torch.cuda.synchronize()
    captures_warm = len(gs.captures)
    times = {"eager": [], "graphed": []}
    done = {"eager": 0, "graphed": 0}
    while min(done.values()) < steps:
        for name, fn in (("eager", eager), ("graphed", graphed)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(block):
                inp, tgt = batches[i % n_batches]
                i += 1
                fn(inp, tgt)
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b) / block)
            done[name] += block
    torch.cuda.synchronize()
    assert len(gs.captures) == captures_warm, "a graph was re-captured inside the timed window"
    res = {}
    for name, t in times.items():
        res[name] = {"ms_per_step_median_block": round(statistics.median(t), 4), "ms_per_step_pooled": round(sum(t) / len(t), 4),
                     "block_min_max": [round(min(t), 4), round(max(t), 4)], "steps": done[name]}
    e, g = res["eager"]["ms_per_step_median_block"], res["graphed"]["ms_per_step_median_block"]
    res["saving_ms_per_step"] = round(e - g, 4)
    res["saving_fraction"] = round((e - g) / e, 4)
    res["graphs"] = gs.num_graphs
    res["padded_text_lengths"] = [s[1] for s in shapes]
    res["capture_s_per_graph"] = [round(s, 3) for _, s in gs.captures]
    res["shared_workspace_bytes"] = gs.workspace_bytes()
    res["step_count"] = opt.step_count
    res["skipped_steps"] = opt.skipped_steps
    res["finite_params"] = bool(torch.isfinite(opt._flat_p).all())
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--steps", type=int, default=240, help="timed steps per mode and batch size (after warm-up)")
    ap.add_argument("--block", type=int, default=20, help="steps per timed block; the modes alternate block by block")
    ap.add_argument("--batches", type=int, nargs="+", default=[32, 8])
    ap.add_argument("--json", default="train_graph_cost.json")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_graph_cost: needs a CUDA GPU (nothing is measured on the CPU)")
    t0 = time.time()
    rec = {"gpu": gpu_info(), "workload": "cfg3_train (synth cfg2: d 1024, 4 layers, Lv 75, Lt <= 32 ragged), FlatAdamW, "
           "input dropout 0.5, DropPath 0.1, attention dropout 0.1", "block": args.block}
    for B in args.batches:
        rec[f"B{B}"] = run(B, args.steps, args.block)
        print(f"B={B}: {json.dumps(rec[f'B{B}'])}", flush=True)
    rec["gpu_after"] = gpu_info()
    rec["wall_s"] = round(time.time() - t0, 1)
    os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
    with open(args.json, "w") as f:
        json.dump(rec, f, indent=1)
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
