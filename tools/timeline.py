#!/usr/bin/env python
"""GPU timeline (CUPTI via torch.profiler) of one steady-state forward / train step: kernel durations and the idle gaps."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch.profiler import profile, ProfilerActivity
from univtg_b200 import build_model, synth

mode = sys.argv[1] if len(sys.argv) > 1 else "fwd"
cfgname = sys.argv[2] if len(sys.argv) > 2 else "cfg2"
cfg = synth.CONFIGS[cfgname]
model, crit = build_model(synth.reference_args(cfg, device="cuda:0"))
model.load_state_dict(synth.make_state_dict(cfg, seed=0), strict=True)
model.to("cuda:0"); crit.to("cuda:0")
inp = {k: v.cuda() for k, v in synth.make_inputs(cfg, seed=1).items()}
tgt = {k: v.cuda() for k, v in synth.make_targets(synth.make_inputs(cfg, seed=1), seed=2).items()}
if mode == "train":
    model.train()
    from univtg_b200.optim import FlatAdamW
    opt = FlatAdamW(model, lr=1e-4, weight_decay=1e-4, max_grad_norm=0.1)
    def step():
        out = model(**inp); ld = crit(out, tgt)
        total = crit.weighted_total(ld)
        opt.zero_grad(set_to_none=True); total.backward()
        opt.step()
else:
    model.eval()
    def step():
        with torch.no_grad():
            model(**inp)
for _ in range(5):
    step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(3):
        step()
    torch.cuda.synchronize()
evs = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
evs.sort(key=lambda e: e.time_range.start)
# keep the last step: find the last occurrence of the first kernel name
names = [e.name for e in evs]
first = names[0]
idx = [i for i, n in enumerate(names) if n == first]
start = idx[-1] if mode == "fwd" else idx[len(idx) * 2 // 3]
evs = evs[start:]
t0 = evs[0].time_range.start
rows = []
prev_end = t0
busy = 0.0
for e in evs:
    s, d = e.time_range.start - t0, e.time_range.end - e.time_range.start
    gap = e.time_range.start - prev_end
    rows.append((s, d, gap, e.name[:60]))
    prev_end = max(prev_end, e.time_range.end)
    busy += d
span = prev_end - t0
print(f"{mode} {cfgname}: {len(rows)} kernels, span {span:.1f} us, busy {busy:.1f} us, idle {span - busy:.1f} us")
agg = {}
for s, d, gap, n in rows:
    a = agg.setdefault(n, [0, 0.0, 0.0]); a[0] += 1; a[1] += d; a[2] += max(gap, 0)
for n, a in sorted(agg.items(), key=lambda kv: -kv[1][1])[:28]:
    print(f"{a[1]:9.1f} us  n={a[0]:3d}  avg {a[1]/a[0]:7.1f}  gap_before_avg {a[2]/a[0]:5.1f}  {n}")
os.makedirs(os.path.join(ROOT, "results"), exist_ok=True)
json.dump(rows, open(os.path.join(ROOT, "results", f"timeline_{mode}_{cfgname}.json"), "w"))
