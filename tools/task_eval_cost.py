"""Time the device drop-ins of the reference's highlight (TVSum / YouTube) and QFVS evaluations on one GPU, in one call.

    python tools/task_eval_cost.py [--calls 20] [--warmup 3] [--json out.json]

Inputs (synthetic, univtg_b200.synth):
  * tvsum: 10 videos (a TVSum domain's val split is about 10) of 100-700 clips x 20 annotators, top-5 mAP;
  * youtube: 30 videos of 20-300 clips, full-list mAP;
  * qfvs_<n>: one summary pair at each real Tags.mat size - 43, 73, 71 and 55 shots per side out of 2152, 3692, 3588 and 2783;
  * qfvs_1024: the size bound, 1024 x 1024 shots.
Reported per input: end_to_end_ms (median over --calls calls of evaluate_hl / calculate_semantic_matching after --warmup calls:
host packing, copies, the kernel, the host means; host clock, each call ends in a synchronising copy), kernel_ms (the kernel
alone on inputs already on the device, CUDA events over 20 launches), oracle_ms (one call of the plain-Python oracle, host
clock; for qfvs the exact Fraction Hungarian, skipped at 1024) and whether the results agree (hl: the same mAP dict; qfvs: s
within 1e-12 of the exact optimum).  The GPU's name and power limit are read in the same call.
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
from oracle import task_eval_oracle as T  # noqa: E402
from univtg_b200 import _lib, metrics, qfvs, synth  # noqa: E402


def _median_ms(fn, calls, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(calls):
        t = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t) * 1e3)
    return statistics.median(times), [min(times), max(times)]


def _events_ms(launch, reps=20):
    for _ in range(3):
        launch()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        launch()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def hl_kernel_ms(case):
    lib = _lib.load_library()
    rows = [b[0] for b in case["blob"]]
    labels, n_label, n_cut, median = metrics.pack_hl_labels(case["dataset"], len(rows), [r.numel() for r in rows])
    V, C, A = labels.shape
    S = max(r.numel() for r in rows)
    scores = torch.zeros(V, S, device="cuda")
    for v, r in enumerate(rows):
        scores[v, :r.numel()] = r.cuda()
    n_score = torch.tensor([r.numel() for r in rows], dtype=torch.int32, device="cuda")
    d_cut, d_lab, d_nl = [torch.from_numpy(x).cuda() for x in (n_cut, labels, n_label)]
    ap = torch.empty(V, A, dtype=torch.float64, device="cuda")
    p = _lib.ptr
    return _events_ms(lambda: _lib.check(lib.univtg_eval_hl_topk(p(scores), p(n_score), p(d_cut), p(d_lab), p(d_nl), V, S, C, A,
                                                                 median, p(ap), _lib.stream_ptr()), "hl_topk"))


def qfvs_kernel_ms(a, b):
    lib = _lib.load_library()
    da, db = torch.from_numpy(a.view(np.int64)).cuda(), torch.from_numpy(b.view(np.int64)).cuda()
    ao = torch.tensor([0, len(a)], dtype=torch.int32, device="cuda")
    bo = torch.tensor([0, len(b)], dtype=torch.int32, device="cuda")
    s = torch.empty(1, dtype=torch.float64, device="cuda")
    p = _lib.ptr
    return _events_ms(lambda: _lib.check(lib.univtg_qfvs_match(p(da), p(ao), p(db), p(bo), 1, max(len(a), len(b)), p(s),
                                                               _lib.stream_ptr()), "qfvs_match"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "task_eval_cost.py measures on a GPU; there is no CPU measurement"
    result = {"gpu": gpu_info()}
    for name, dset, n, clips in (("tvsum", "tvsum", 10, (100, 250, 400, 700)), ("youtube", "youtube", 30, (20, 60, 120, 300))):
        case = synth.make_hl_eval_case(2024, dset, n_videos=n, clips=clips, shorter=0.0, tie_frac=0.0)
        blob = [b.cuda() for b in case["blob"]]
        got = metrics.evaluate_hl(case["dataset"], blob)
        e2e, span = _median_ms(lambda: metrics.evaluate_hl(case["dataset"], blob), args.calls, args.warmup)
        t = time.perf_counter()
        ref = T.evaluate_hl(dset, case["labels"], case["blob"])
        oracle_ms = (time.perf_counter() - t) * 1e3
        result[name] = {"videos": n, "end_to_end_ms": e2e, "end_to_end_min_max_ms": span, "kernel_ms": hl_kernel_ms(case),
                        "oracle_ms": oracle_ms, "same_as_oracle": got == ref}
    for seed, (shots, k) in enumerate(((2152, 43), (3692, 73), (3588, 71), (2783, 55), (4000, 1024))):
        c = synth.make_qfvs_match_case(500 + seed, shots, k, k)
        top = torch.tensor(c["machine"], device="cuda")
        tags = [c["tags"]]
        e2e, span = _median_ms(lambda: qfvs.calculate_semantic_matching(top, c["gt"], tags, 0), args.calls, args.warmup)
        masks = (qfvs.tag_masks(c["tags"][c["machine"]]), qfvs.tag_masks(c["tags"][c["gt"]]))
        rec = {"shots": shots, "per_side": k, "end_to_end_ms": e2e, "end_to_end_min_max_ms": span, "kernel_ms": qfvs_kernel_ms(*masks)}
        if k <= 128:
            s = float(qfvs.match_sums([masks])[0])
            t = time.perf_counter()
            opt = float(T.semantic_matching(c["machine"], c["gt"], c["tags"])[0])
            rec["oracle_ms"] = (time.perf_counter() - t) * 1e3
            rec["s_within_1e-12_of_exact"] = abs(s - opt) <= 1e-12 * max(opt, 1.0)
        result[f"qfvs_{k}"] = rec
    print(json.dumps(result))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
