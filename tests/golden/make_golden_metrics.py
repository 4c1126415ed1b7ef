#!/usr/bin/env python
"""Writes tests/golden/reference_metrics.json: the live reference `eval.eval.eval_submission` on the seeded cases of
univtg_b200.synth.make_eval_case, so the metrics oracle (oracle/metrics_oracle.py) stays pinned without the reference or
scikit-learn.  The inputs are not stored: each case keeps its seed and parameters and a sha256 of its JSON-serialised inputs
(tests regenerate them and check the hash).  Per case the file holds json.dumps of the returned dict, the per-query
compute_average_precision_detection arrays of every length range (as compute_mr_ap builds its triples) and the per-tuple
get_ap values of every min score (as compute_hl_ap builds its tuples); floats are stored as JSON numbers (repr-exact).
Every case has at most 50 queries, so compute_mr_ap's single imap_unordered chunk keeps submission order.
Usage: python tests/golden/make_golden_metrics.py <path to a showlab/UniVTG checkout>"""
import contextlib
import hashlib
import io
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, os.path.abspath(sys.argv[1]))
import sklearn  # noqa: E402
from eval import eval as E  # noqa: E402
from eval.utils import compute_average_precision_detection  # noqa: E402

from univtg_b200.synth import make_eval_case  # noqa: E402

CASES = [
    dict(seed=1),
    dict(seed=2, n_queries=30, n_windows=20, sort_windows=False),
    dict(seed=3, n_queries=30, durations=(149,), gt_lengths=(14, 20, 30, 44)),
    dict(seed=4, n_queries=36, match_number=False),
    dict(seed=5, n_queries=8, durations=(1200, 1201), gt_lengths=(10, 30, 60, 150, 400)),
    dict(seed=6, n_queries=30, gt_lengths=(0, 2, 4, 10), max_gt=6),
    dict(seed=7, n_queries=30, n_windows=3, max_gt=6),
    dict(seed=8, n_queries=20, tasks="mr"),
    dict(seed=9, n_queries=20, tasks="hl"),
]


def input_hash(case):
    blob = json.dumps([case["submission"], case["ground_truth"], case["match_number"]], sort_keys=True)
    return hashlib.sha256(blob.encode()).hexdigest()


def per_query_ap(sub, gt):
    """{range name: [[qid, ap list], ...]} with the reference's own get_data_by_range and triple construction."""
    out = {}
    thds = [float(f"{e:.2f}") for e in np.linspace(0.5, 0.95, 10)]
    for rng_, name in zip([[0, 10], [10, 30], [30, float("inf")], [0, float("inf")]], ["short", "middle", "long", "full"]):
        s, g = E.get_data_by_range(sub, gt, rng_)
        gt_by = {d["qid"]: d for d in g}
        rows = []
        for d in s:
            preds = [{"video-id": d["qid"], "t-start": w[0], "t-end": w[1], "score": w[2]} for w in d["pred_relevant_windows"][:10]]
            gts = [{"video-id": d["qid"], "t-start": w[0], "t-end": w[1]} for w in gt_by[d["qid"]]["relevant_windows"]]
            rows.append([d["qid"], [float(x) for x in compute_average_precision_detection(gts, preds, tiou_thresholds=thds)]])
        out[name] = rows
    return out


def per_tuple_ap(sub, gt):
    """{min score: [[qid, [ap per annotator]], ...]} with the reference's mk_gt_scores and compute_ap_from_tuple."""
    gt_by = {d["qid"]: E.mk_gt_scores(d) for d in gt}
    out = {}
    for m in (2, 3, 4):
        rows = []
        for d in sub:
            binary = (gt_by[d["qid"]] >= m).astype(float)
            rows.append([d["qid"], [float(E.compute_ap_from_tuple((0, a, binary[:, a], np.array(d["pred_saliency_scores"])))[2])
                                    for a in range(3)]])
        out[str(m)] = rows
    return out


def main():
    records = []
    for params in CASES:
        case = make_eval_case(**params)
        sub, gt = case["submission"], case["ground_truth"]
        with contextlib.redirect_stdout(io.StringIO()):
            res = E.eval_submission(sub, gt, verbose=False, match_number=case["match_number"])
        if not case["match_number"]:
            shared = {d["qid"] for d in sub} & {d["qid"] for d in gt}
            sub = [d for d in sub if d["qid"] in shared]
            gt = [d for d in gt if d["qid"] in shared]
        rec = {"params": params, "sha256": input_hash(case), "result": json.dumps(res)}
        if "pred_relevant_windows" in sub[0]:
            rec["ap_detection"] = per_query_ap(sub, gt)
        if "pred_saliency_scores" in sub[0]:
            rec["get_ap"] = per_tuple_ap(sub, gt)
        records.append(rec)
    out = {"numpy": np.__version__, "scikit-learn": sklearn.__version__, "cases": records}
    path = os.path.join(HERE, "reference_metrics.json")
    with open(path, "w") as f:
        json.dump(out, f)
    print("wrote", path, len(records), "cases")


if __name__ == "__main__":
    main()
