#!/usr/bin/env python
"""Writes tests/golden/postproc_nms.json: inputs and outputs of the reference `utils.temporal_nms.temporal_nms` on seeded random
windows, so the oracle's restatement stays pinned without the reference.
Usage: python tests/golden/make_golden_postproc.py <path to a showlab/UniVTG checkout>"""
import json
import os
import random
import sys

sys.path.insert(0, os.path.abspath(sys.argv[1]))
from utils.temporal_nms import temporal_nms  # noqa: E402

rng = random.Random(7)
cases = []
for n in (0, 1, 2, 3, 10, 10, 37, 75):
    for thd in (0.3, 0.5, 0.7, 0.0):
        rows = []
        for _ in range(n):
            st = round(rng.uniform(0, 140), 4)
            ed = round(min(150.0, st + rng.choice([0.0, 2.0, rng.uniform(0, 60)])), 4)
            sc = round(rng.choice([0.0, rng.random(), 0.5]), 4)
            rows.append([st, ed, sc])
        for max_after in (10, 3):
            ref = temporal_nms([list(r) for r in rows], nms_thd=thd, max_after_nms=max_after)
            cases.append({"rows": rows, "nms_thd": thd, "max_after_nms": max_after, "expected": ref})
out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "postproc_nms.json")
with open(out, "w") as f:
    json.dump(cases, f)
print("wrote", out, len(cases), "cases")
