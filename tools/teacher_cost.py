"""Time the CLIP-teacher pseudo labelling (univtg_b200.teacher) on one GPU, in one call.

    python tools/teacher_cost.py [--videos 10000] [--json out.json]

Inputs (synthetic, univtg_b200.synth.make_teacher_case): C = 19,994 classes (the OIDv6 list) of D = 512 (ViT-B/32), and
--videos videos with T drawn uniformly from 5..75 clips.  That T range is an assumption; it has not been checked against the
VideoCC features.  Reported, all per 1,000 videos:
  * kernel_ms: univtg_teacher_label alone on inputs already on the device, chunks of 1,000 videos, CUDA events;
  * memory_ms: PseudoLabeler.lines from numpy arrays in memory (packing, one copy each way, the kernels, the JSONL text),
    host clock, median of 3 runs over every video after a warm-up;
  * npz_ms: write_pseudo_labels from one .npz file per video in a temporary directory (the files were just written, so they
    are likely in the page cache), host clock, one run;
  * reference_loop_ms: the reference's per-video device work (oracle.teacher_oracle.reference_loop_fp32: fp32 sim_matrix, sum,
    full sort, the .tolist() syncs) on the same GPU with TF32 off, over the first 1,000 videos, host clock;
  * fallback_videos over all videos, and whether the lines of the first 300 videos equal the float64 oracle's.
The GPU's name and power limit are read in the same call.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from clip_cost import gpu_info  # noqa: E402
from oracle import teacher_oracle as O  # noqa: E402
from univtg_b200 import _lib, synth, teacher  # noqa: E402


def kernel_ms(lab, feats, chunk=1000, reps=3):
    """CUDA-event time of univtg_teacher_label per `chunk` videos (inputs packed on the device beforehand)."""
    lib = _lib.load_library()
    K, D = lab.topk, lab.D
    jobs = []
    for s in range(0, len(feats) - chunk + 1, chunk):
        part = feats[s:s + chunk]
        off = np.zeros(chunk + 1, np.int32)
        np.cumsum([len(f) for f in part], out=off[1:])
        S = int(off[-1])
        x = torch.from_numpy(np.concatenate(part)).cuda()
        o = torch.from_numpy(off).cuda()
        ws = torch.empty(lib.univtg_teacher_chunk_bytes(chunk, S, lab.C, D), dtype=torch.uint8, device="cuda")
        out = torch.empty(2 * chunk * K + 2 * S * K + 1, dtype=torch.int32, device="cuda")
        jobs.append((x, o, S, ws, out))

    def run():
        for x, o, S, ws, out in jobs:
            _lib.check(lib.univtg_teacher_label(_lib.ptr(lab._cls), _lib.ptr(lab._cls_ws), lab.C, D, _lib.ptr(x), _lib.ptr(o), chunk, S,
                                                K, lab.th, _lib.ptr(ws), ws.numel(), _lib.ptr(out), _lib.stream_ptr()), "label")

    run()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        run()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / (reps * len(jobs)) * (1000 / chunk)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--videos", type=int, default=10000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    info = gpu_info()
    t = time.perf_counter()
    case = synth.make_teacher_case(7, n_classes=19994, dim=512, n_videos=args.videos, clips=(5, 75), edges=False)
    gen_s = time.perf_counter() - t
    feats, vids = case["features"], case["vids"]
    n = len(feats)
    per = 1000.0 / n
    cls = torch.from_numpy(case["classes"]).cuda()
    torch.cuda.synchronize()
    t = time.perf_counter()
    lab = teacher.PseudoLabeler(cls, case["names"])
    torch.cuda.synchronize()
    prep_ms = (time.perf_counter() - t) * 1e3

    k_ms = kernel_ms(lab, feats)
    lab.lines(feats[:500], vids[:500])  # warm-up
    times = []
    for _ in range(3):
        t = time.perf_counter()
        lines = lab.lines(feats, vids)
        times.append((time.perf_counter() - t) * 1e3)
    fallback = lab.fallback_videos
    with tempfile.TemporaryDirectory() as tmp:
        clip_dir = os.path.join(tmp, "vid_clip")
        os.makedirs(clip_dir)
        for f, v in zip(feats, vids):
            np.savez(os.path.join(clip_dir, v + ".npz"), features=f)
        t = time.perf_counter()
        n_lines = teacher.write_pseudo_labels(os.path.join(tmp, "out.jsonl"), clip_dir, lab)
        npz_ms = (time.perf_counter() - t) * 1e3
    m = min(1000, n)
    torch.cuda.synchronize()
    t = time.perf_counter()
    O.reference_loop_fp32(feats[:m], case["classes"])
    torch.cuda.synchronize()
    ref_ms = (time.perf_counter() - t) * 1e3 * (1000 / m)
    q = min(300, n)
    agree = lab.lines(feats[:q], vids[:q]) == O.lines(O.label(feats[:q], vids[:q], cls, case["names"]))
    res = {"gpu": info, "classes": 19994, "dim": 512, "videos": n, "clips": int(sum(len(f) for f in feats)), "clips_per_video": [5, 75],
           "lines": len(lines), "npz_lines": n_lines, "prepare_classes_ms": round(prep_ms, 3),
           "per_1000_videos": {"kernel_ms": round(k_ms, 3), "memory_ms": round(statistics.median(times) * per, 3),
                               "memory_ms_min_max": [round(min(times) * per, 3), round(max(times) * per, 3)],
                               "npz_ms": round(npz_ms * per, 3), "reference_loop_ms": round(ref_ms, 3)},
           "fallback_videos": fallback, "oracle_agrees_first_300": agree, "synth_s": round(gen_s, 1)}
    print(json.dumps(res, indent=1))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
