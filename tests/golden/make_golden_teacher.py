#!/usr/bin/env python
"""Writes tests/golden/reference_teacher.json: the lines the unmodified reference teacher/clip2label.py writes for the seeded
cases of univtg_b200.synth.make_teacher_case, so the float64 oracle (oracle/teacher_oracle.py) and the device labels stay
pinned without the reference.  The inputs are not stored: each case keeps its seed, parameters and the sha256 of its inputs
(tests regenerate them and check the hash), plus the reference's lines grouped by video in the order it wrote them (rank order).

The script runs with runpy as __main__ in a temporary directory laid out as it expects (see `layout`), with torch.Tensor.cuda
stubbed to the identity so it runs on the CPU.  Every case is drawn with safe=True: no top-(k+1) cosine near a bin edge, no
near-tied top-(k+1) sums and no duplicated row in a top-(k+1), so the reference's float32 arithmetic and CPU sort cannot
disagree with the float64 labels.

Usage: python tests/golden/make_golden_teacher.py <path to a showlab/UniVTG checkout>"""
import json
import os
import runpy
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from univtg_b200 import synth  # noqa: E402

CASES = [
    dict(seed=1),
    dict(seed=2, n_classes=2000, dim=512, n_videos=20, clips=(2, 120), dup=12),
    dict(seed=3, n_classes=50, dim=32, n_videos=30, clips=(2, 20)),
    dict(seed=4, n_classes=19994, dim=512, n_videos=8, clips=(5, 75), dup=12),
    dict(seed=5, n_classes=4, dim=16, n_videos=6, clips=(2, 30)),
]


def make_case(params):
    return synth.make_teacher_case(**params, safe=True, parallel=False)


def layout(case, root):
    """clip2label.py's inputs under root: data/videocc/vid_clip/{vid}.npz ('features'), data/videocc/vid_slowfast/{vid}.npz
    (only listed), teacher/oidv6-class-descriptions.json and data/commonsense/clip_txt/class_text.npz ('pooler_output').  The
    last video has no slowfast file (it is left out), and one extra video has no clips (it is skipped).  Returns the clip
    directory and the slowfast directory."""
    clip_dir = os.path.join(root, "data", "videocc", "vid_clip")
    sf_dir = os.path.join(root, "data", "videocc", "vid_slowfast")
    for d in (clip_dir, sf_dir, os.path.join(root, "teacher"), os.path.join(root, "data", "commonsense", "clip_txt")):
        os.makedirs(d, exist_ok=True)
    D = case["classes"].shape[1]
    items = list(zip(case["vids"], case["features"])) + [("zz_empty", np.zeros((0, D), np.float32))]
    for i, (vid, f) in enumerate(items):
        np.savez(os.path.join(clip_dir, vid + ".npz"), features=f)
        if i != len(case["vids"]) - 1:
            np.savez(os.path.join(sf_dir, vid + ".npz"), features=np.zeros((1, 1), np.float32))
    with open(os.path.join(root, "teacher", "oidv6-class-descriptions.json"), "w") as f:
        json.dump(case["names"], f)
    np.savez(os.path.join(root, "data", "commonsense", "clip_txt", "class_text.npz"), pooler_output=case["classes"])
    return clip_dir, sf_dir


def run_reference(script, case):
    import torch

    cuda = torch.Tensor.cuda
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        layout(case, tmp)
        torch.Tensor.cuda = lambda self, *a, **k: self
        try:
            os.chdir(tmp)
            runpy.run_path(script, run_name="__main__")
            with open(os.path.join(tmp, "curve_5_window.jsonl")) as f:
                text = f.read()
        finally:
            os.chdir(cwd)
            torch.Tensor.cuda = cuda
    by_vid = {}
    for line in text.splitlines():
        by_vid.setdefault(json.loads(line)["vid"], []).append(line)
    return by_vid


def main():
    import torch

    script = os.path.join(os.path.abspath(sys.argv[1]), "teacher", "clip2label.py")
    cases = []
    for params in CASES:
        case = make_case(params)
        cases.append({"params": params, "sha256": synth.teacher_case_sha256(case), "lines": run_reference(script, case)})
    out = {"torch": torch.__version__, "numpy": np.__version__, "topk": 5, "th": 0.05, "clip_len": 2, "cases": cases}
    path = os.path.join(HERE, "reference_teacher.json")
    with open(path, "w") as f:
        json.dump(out, f)
    print("wrote", path, len(cases), "cases,", sum(sum(len(v) for v in c["lines"].values()) for c in cases), "lines")


if __name__ == "__main__":
    main()
