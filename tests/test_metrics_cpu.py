"""Metrics oracle (oracle/metrics_oracle.py) pinned to the live reference eval_submission through
tests/golden/reference_metrics.json, numpy's summation order, and the input checks of univtg_b200.metrics (which run on the
host, before any launch)."""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import metrics_oracle as M
from tests.helpers import GOLDEN
from univtg_b200 import metrics
from univtg_b200.synth import make_eval_case


def _golden():
    with open(os.path.join(GOLDEN, "reference_metrics.json")) as f:
        return json.load(f)


def _shared(case):
    sub, gt = case["submission"], case["ground_truth"]
    shared = {d["qid"] for d in sub} & {d["qid"] for d in gt}
    return [d for d in sub if d["qid"] in shared], [d for d in gt if d["qid"] in shared]


def test_golden_records_versions_and_cases():
    g = _golden()
    assert g["numpy"] and g["scikit-learn"]
    assert len(g["cases"]) == 9


@pytest.mark.parametrize("i", range(9))
def test_regenerated_inputs_hash_to_the_golden_sha256(i):
    rec = _golden()["cases"][i]
    case = make_eval_case(**rec["params"])
    blob = json.dumps([case["submission"], case["ground_truth"], case["match_number"]], sort_keys=True)
    assert hashlib.sha256(blob.encode()).hexdigest() == rec["sha256"], "make_eval_case drifted from the golden inputs"


@pytest.mark.parametrize("i", range(9))
def test_oracle_reproduces_reference_eval_submission(i):
    rec = _golden()["cases"][i]
    case = make_eval_case(**rec["params"])
    got = M.eval_submission(case["submission"], case["ground_truth"], verbose=False, match_number=case["match_number"])
    assert json.dumps(got) == rec["result"]


@pytest.mark.parametrize("i", range(9))
def test_oracle_per_query_values_are_bit_exact(i):
    """Every compute_average_precision_detection array (per range; an empty range is the full set) and every get_ap value."""
    rec = _golden()["cases"][i]
    sub, gt = _shared(make_eval_case(**rec["params"]))
    pq = M.per_query(sub, gt, mr="ap_detection" in rec, hl="get_ap" in rec)
    row = {d["qid"]: q for q, d in enumerate(sub)}
    n = 0
    for r, (name, _, _) in enumerate(M.RANGES):
        src = r if pq.get("kept", np.zeros((4, 1), bool))[r].any() else 3
        for qid, ap in rec.get("ap_detection", {}).get(name, []):
            assert pq["ap"][src, row[qid]].tolist() == ap, (name, qid)
            n += 1
    for lv, m in enumerate(("2", "3", "4")):
        for qid, aps in rec.get("get_ap", {}).get(m, []):
            assert pq["hl_ap"][lv, row[qid]].tolist() == aps, (m, qid)
            n += 1
    assert n > 0


def _ap_lengths(case):
    """Lengths of the vectors the reference sums per query: AP terms of interpolated_precision_recall, get_ap's mean."""
    sub, gt = _shared(case)
    gt_by = {d["qid"]: d for d in gt}
    lens = set()
    for d in sub:
        if "pred_relevant_windows" in d:
            lens.update(range(1, min(len(d["pred_relevant_windows"]), 10) + 2))
        if "pred_saliency_scores" in d and "relevant_clip_ids" in gt_by[d["qid"]]:
            full = M.gt_scores(gt_by[d["qid"]])
            for m in (2, 3, 4):
                for a in range(3):
                    y = (full[:, a] >= m).astype(float)
                    if 0 < y.sum() < len(y):
                        n = len(y)
                        s = np.zeros(n)
                        p = np.asarray(d["pred_saliency_scores"][:n], float)
                        s[:len(p)] = p
                        _, recall, _ = M.precision_recall_curve(y, s)
                        lens.add(int(np.count_nonzero(np.diff(recall.astype(np.float32)))))
    return lens


def test_numpy_sum_follows_the_pairwise_rule_for_the_lengths_that_occur():
    lens = set(range(1, 12))
    for rec in _golden()["cases"]:
        lens |= _ap_lengths(make_eval_case(**rec["params"]))
    assert max(lens) > 128, "no case exercises the recursive part of numpy's pairwise sum"
    rng = np.random.default_rng(0)
    for n in sorted(lens):
        for scale in (1.0, 1e-8, 1e8):
            for _ in range(20):
                x = rng.random(n) * rng.choice([1.0, scale], n)
                assert float(np.sum(x)) == M.pairwise_sum(x), n
                assert float(np.mean(x)) == M.pairwise_sum(x) / n, n


def test_oracle_tie_rule_locks_the_higher_gt_index():
    """One prediction with IoU 0.5 to two different gt windows: the higher index is locked, so the second prediction (IoU 1 with
    that window) finds it taken."""
    preds = [[0.0, 20.0, 0.9], [10.0, 20.0, 0.8]]
    assert M.ap_detection([[0, 10], [10, 20]], preds)[0] == 0.5
    assert M.ap_detection([[10, 20], [0, 10]], preds)[0] == 1.0


def _small():
    return make_eval_case(1, n_queries=4)


def _bad(mutate, match_number=True):
    case = _small()
    mutate(case["submission"], case["ground_truth"])
    return case["submission"], case["ground_truth"], match_number


@pytest.mark.parametrize("mutate,match", [
    (lambda s, g: (s.clear(), g.clear()), "empty submission"),
    (lambda s, g: s.append(dict(s[0])), "duplicate qids"),
    (lambda s, g: g.append(dict(g[0])), "duplicate qids"),
    (lambda s, g: s[1].update(pred_relevant_windows=[]), "no predicted window"),
    (lambda s, g: g[2].update(relevant_windows=[]), "no relevant_windows"),
    (lambda s, g: g[2].pop("relevant_windows"), "no relevant_windows"),
    (lambda s, g: g[0].update(relevant_windows=[[0, 2]] * 65), "more than 64"),
    (lambda s, g: g[1].update(duration=1.5), "int\\(duration / 2\\)"),
    (lambda s, g: g[1].update(duration=2 * 4097), "int\\(duration / 2\\)"),
    (lambda s, g: g[3].update(relevant_clip_ids=[-1] + g[3]["relevant_clip_ids"][1:]), "outside"),
    (lambda s, g: g[3].update(relevant_clip_ids=[int(g[3]["duration"] / 2)] + g[3]["relevant_clip_ids"][1:]), "outside"),
    (lambda s, g: g[3].update(relevant_clip_ids=[], saliency_scores=[]), "relevant_clip_ids"),
    (lambda s, g: s[0].update(pred_saliency_scores=[]), "empty pred_saliency_scores"),
    (lambda s, g: s[0].update(pred_saliency_scores=[float("nan")] + s[0]["pred_saliency_scores"][1:]), "non-finite"),
])
def test_inputs_the_reference_cannot_evaluate_raise_value_error(mutate, match):
    sub, gt, mn = _bad(mutate)
    with pytest.raises(ValueError, match=match):
        metrics.eval_submission(sub, gt, match_number=mn)


def test_qid_mismatch_raises_the_reference_exception():
    case = _small()
    with pytest.raises(AssertionError):
        metrics.eval_submission(case["submission"][1:], case["ground_truth"])
    with pytest.raises(ValueError, match="no qid shared"):
        metrics.eval_submission(case["submission"][:2], case["ground_truth"][2:], match_number=False)


def test_packing_keeps_submission_order_and_the_first_ten_windows():
    case = make_eval_case(2, n_queries=6, n_windows=20, sort_windows=False)
    sub, gt = case["submission"], case["ground_truth"]
    gts = [{d["qid"]: d for d in gt}[d["qid"]] for d in reversed(sub)]
    pred, n_pred, gwin, n_gt = metrics.pack_mr(list(reversed(sub)), gts)
    for q, d in enumerate(reversed(sub)):
        rows = d["pred_relevant_windows"][:10]
        assert n_pred[q] == len(rows) and pred[q, :len(rows)].tolist() == rows
        assert gwin[q, :n_gt[q]].tolist() == [[float(x) for x in w] for w in gts[q]["relevant_windows"]]
    sal, n_sal, labels, n_clips = metrics.pack_hl(sub, gt)
    for q, g in enumerate(gt):
        full = M.gt_scores(g)
        assert n_clips[q] == len(full)
        for lv in range(3):
            for a in range(3):
                assert (((labels[q, :n_clips[q]] >> (3 * lv + a)) & 1) == (full[:, a] >= 2 + lv)).all()
        assert sal[q, :n_sal[q]].tolist() == sub[q]["pred_saliency_scores"]
