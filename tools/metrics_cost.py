"""Time univtg_b200.metrics.eval_submission at QVHighlights val size on one GPU, in one call.

    python tools/metrics_cost.py [--calls 15] [--warmup 3] [--json out.json]

Inputs: synth.make_eval_case at 1,550 queries with 75 predicted windows each (before NMS) and with 10 (after NMS), 75 saliency
scores, 1-4 gt windows and 3 annotators per query.  Reported per variant:
  * end_to_end_ms: median over --calls calls of eval_submission after --warmup calls (host packing, one host-to-device copy, the
    two kernels, one device-to-host copy, the numpy means and formatting; host clock, the call ends in a synchronising copy);
  * pack_ms: median of the host packing alone (pack_mr + pack_hl);
  * kernel_ms: univtg_eval_mr + univtg_eval_hl on inputs already on the device, CUDA events over 50 launch pairs;
  * oracle_ms: one call of the serial numpy restatement (oracle/metrics_oracle.py) on the same inputs, host clock;
and whether the two results are the same JSON string.  The GPU's name and power limit are read in the same call.
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from clip_cost import gpu_info  # noqa: E402
from oracle import metrics_oracle as M  # noqa: E402
from univtg_b200 import _lib, metrics  # noqa: E402
from univtg_b200.synth import make_eval_case  # noqa: E402


def kernel_ms(sub, gt, reps=50):
    lib = _lib.load_library()
    by = {d["qid"]: d for d in gt}
    gts = [by[d["qid"]] for d in sub]
    pred, n_pred, gwin, n_gt = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in metrics.pack_mr(sub, gts)]
    sal, n_sal, labels, n_clips = metrics.pack_hl(sub, gts)
    labels = torch.from_numpy(labels.view(np.int16)).cuda()
    sal, n_sal, n_clips = [torch.from_numpy(a).cuda() for a in (sal, n_sal, n_clips)]
    Q, C = len(sub), labels.shape[1]
    ap, r1, r5 = torch.empty(4, Q, 10, dtype=torch.float64, device="cuda"), torch.empty(4, Q, dtype=torch.float64, device="cuda"), \
        torch.empty(4, Q, dtype=torch.float64, device="cuda")
    kept = torch.empty(4, Q, dtype=torch.uint8, device="cuda")
    hap, hit = torch.empty(3, Q, 3, dtype=torch.float64, device="cuda"), torch.empty(3, Q, 3, dtype=torch.float64, device="cuda")
    scratch = torch.empty(Q * 9 * C, dtype=torch.float64, device="cuda")
    p = _lib.ptr

    def launch():
        s = _lib.stream_ptr()
        _lib.check(lib.univtg_eval_mr(p(pred), p(n_pred), p(gwin), p(n_gt), Q, gwin.shape[1], p(ap), p(r1), p(r5), p(kept), s), "mr")
        _lib.check(lib.univtg_eval_hl(p(sal), p(n_sal), p(labels), p(n_clips), Q, sal.shape[1], C, p(scratch), p(hap), p(hit), s), "hl")

    for _ in range(5):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        launch()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=15)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "metrics_cost.py measures on a GPU; there is no CPU measurement"
    result = {"gpu": gpu_info(), "queries": 1550}
    for name, n_windows in (("before_nms_75_windows", 75), ("after_nms_10_windows", 10)):
        case = make_eval_case(2024, n_queries=1550, n_windows=n_windows, durations=(150,))
        sub, gt = case["submission"], case["ground_truth"]
        for _ in range(args.warmup):
            metrics.eval_submission(sub, gt)
        e2e, pack = [], []
        for _ in range(args.calls):
            t = time.perf_counter()
            got = metrics.eval_submission(sub, gt)
            e2e.append((time.perf_counter() - t) * 1e3)
            by = {d["qid"]: d for d in gt}
            gts = [by[d["qid"]] for d in sub]
            t = time.perf_counter()
            metrics.pack_mr(sub, gts)
            metrics.pack_hl(sub, gts)
            pack.append((time.perf_counter() - t) * 1e3)
        t = time.perf_counter()
        ref = M.eval_submission(sub, gt)
        oracle_ms = (time.perf_counter() - t) * 1e3
        result[name] = {"end_to_end_ms": statistics.median(e2e), "end_to_end_min_max_ms": [min(e2e), max(e2e)],
                        "pack_ms": statistics.median(pack), "kernel_ms": kernel_ms(sub, gt), "oracle_ms": oracle_ms,
                        "same_json_as_oracle": json.dumps(got) == json.dumps(ref)}
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
