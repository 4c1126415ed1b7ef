#!/usr/bin/env python
"""Which framework (ATen / memcpy / memset) device operations does one cfg3 train step still issue next to the library's own
kernels?  Runs a few steps under torch.profiler and prints every CPU-side op that launched device work, with input shapes.

  python tools/probe_step_ops.py > results/step_ops.txt
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from univtg_b200 import build_model, synth  # noqa: E402
from univtg_b200.optim import FlatAdamW  # noqa: E402


def main():
    dev = torch.device("cuda", 0)
    cfg = synth.CONFIGS["cfg2"]
    model, crit = build_model(synth.reference_args(cfg, device=str(dev)))
    model.load_state_dict(synth.make_state_dict(cfg, seed=0), strict=True)
    model.to(dev)
    crit.to(dev)
    model.train()
    crit.train()
    opt = FlatAdamW(model, lr=1e-4, weight_decay=1e-4, max_grad_norm=0.1)
    inp = {k: v.to(dev) for k, v in synth.make_inputs(cfg, seed=1).items()}
    tgt = {k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in synth.make_targets(synth.make_inputs(cfg, seed=1), seed=100).items()}

    def step():
        out = model(**inp)
        ld = crit(out, tgt)
        total = crit.weighted_total(ld)
        opt.zero_grad(set_to_none=True)
        total.backward()
        opt.step()

    for _ in range(5):
        step()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA], record_shapes=True, with_stack=True) as prof:
        for _ in range(3):
            step()
        torch.cuda.synchronize()
    # device activities that are not this library's kernels, with the CPU op that issued them
    rows = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            continue
        kern = [k for k in ev.kernels] if hasattr(ev, "kernels") else []
        for k in kern:
            if "uv::" in k.name or "pack_multi" in k.name:
                continue
            key = (ev.name, str(ev.input_shapes), k.name[:70])
            r = rows.setdefault(key, [0, 0.0, ev.stack[:6] if ev.stack else []])
            r[0] += 1
            r[1] += k.duration
    for (op, shapes, kname), (n, us, stack) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
        print(f"{us / 3:8.1f} us/step  n/step={n / 3:4.1f}  {op}  {shapes}  -> {kname}")
        for fr in stack:
            if "site-packages" not in fr:
                print("             ", fr)


if __name__ == "__main__":
    main()
