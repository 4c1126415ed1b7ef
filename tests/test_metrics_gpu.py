"""univtg_eval_mr / univtg_eval_hl (csrc/metrics.cu) and univtg_b200.metrics.eval_submission: per-query values bit-exact
against the metrics oracle, the returned dict equal to the live reference's (tests/golden/reference_metrics.json)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import metrics_oracle as M
from tests.helpers import GOLDEN
from univtg_b200 import metrics
from univtg_b200.synth import make_eval_case

pytestmark = pytest.mark.gpu


def _golden():
    with open(os.path.join(GOLDEN, "reference_metrics.json")) as f:
        return json.load(f)["cases"]


def _shared(case):
    sub, gt = case["submission"], case["ground_truth"]
    shared = {d["qid"] for d in sub} & {d["qid"] for d in gt}
    return [d for d in sub if d["qid"] in shared], [d for d in gt if d["qid"] in shared]


def _device_per_query(sub, gt):
    by = {d["qid"]: d for d in gt}
    gts = [by[d["qid"]] for d in sub]
    mr = metrics.pack_mr(sub, gts) if "pred_relevant_windows" in sub[0] else None
    hl = metrics.pack_hl(sub, gts) if "pred_saliency_scores" in sub[0] else None
    return metrics.per_query(mr, hl)


def _assert_bit_exact(dev, ref):
    if "ap" in ref:
        assert (dev["kept"] == ref["kept"]).all()
        k = ref["kept"]
        for name in ("ap", "iou_r1", "iou_r5"):
            d, r = dev[name][k], ref[name][k]
            assert d.view(np.int64).tolist() == r.view(np.int64).tolist(), (name, np.argwhere(d != r)[:5])
    if "hl_ap" in ref:
        for name in ("hl_ap", "hit"):
            d, r = dev[name], ref[name]
            assert d.view(np.int64).tolist() == r.view(np.int64).tolist(), (name, np.argwhere(d != r)[:5])


@pytest.mark.parametrize("i", range(9))
def test_device_per_query_values_equal_the_oracle_on_golden_cases(i):
    sub, gt = _shared(make_eval_case(**_golden()[i]["params"]))
    ref = M.per_query(sub, gt, mr="pred_relevant_windows" in sub[0], hl="pred_saliency_scores" in sub[0])
    _assert_bit_exact(_device_per_query(sub, gt), ref)


@pytest.mark.parametrize("i", range(9))
def test_eval_submission_equals_the_reference_json(i):
    rec = _golden()[i]
    case = make_eval_case(**rec["params"])
    got = metrics.eval_submission(case["submission"], case["ground_truth"], verbose=False, match_number=case["match_number"])
    assert json.dumps(got) == rec["result"]


@pytest.mark.parametrize("params", [
    dict(seed=101, n_queries=1550, n_windows=75, durations=(150,)),  # QVHighlights val size, before NMS
    dict(seed=102, n_queries=1550, n_windows=10, durations=(150,)),  # after NMS
    dict(seed=103, n_queries=40, durations=(1200, 1201, 1202), gt_lengths=(30, 400, 600, 1200), max_gt=8),  # 600 clips
], ids=["qvh_val_75", "qvh_val_10", "long_video"])
def test_device_per_query_values_equal_the_oracle_on_random_cases(params):
    case = make_eval_case(**params)
    sub, gt = case["submission"], case["ground_truth"]
    ref = M.per_query(sub, gt)
    _assert_bit_exact(_device_per_query(sub, gt), ref)
    assert json.dumps(metrics.eval_submission(sub, gt)) == json.dumps(M.eval_submission(sub, gt))


def test_tie_rule_locks_the_higher_gt_index():
    """A prediction at IoU 0.5 with two different gt windows locks the higher index; the next prediction (IoU 1 with that window)
    then finds it taken.  Swapping the gt order makes both predictions hits."""
    pred = [[0.0, 20.0, 0.9], [10.0, 20.0, 0.8]]
    for gt_windows, expect in (([[0, 10], [10, 20]], 0.5), ([[10, 20], [0, 10]], 1.0)):
        pq = metrics.per_query(metrics.pack_mr([{"qid": 0, "pred_relevant_windows": pred}],
                                               [{"qid": 0, "relevant_windows": gt_windows}]), None)
        assert pq["ap"][3, 0, 0] == expect
        assert pq["ap"][3, 0, 0] == M.ap_detection(gt_windows, pred)[0]


def test_nan_iou_counts_as_a_match_and_r5_zeroes_it():
    """Zero-length prediction on a zero-length gt window: IoU 0/0 = NaN, which numpy's comparisons treat as a hit."""
    pred = [[4.0, 4.0, 0.9], [0.0, 2.0, 0.5]]
    gt_windows = [[0, 6], [4, 4]]
    pq = metrics.per_query(metrics.pack_mr([{"qid": 0, "pred_relevant_windows": pred}], [{"qid": 0, "relevant_windows": gt_windows}]),
                           None)
    ref = M.per_query([{"qid": 0, "pred_relevant_windows": pred}], [{"qid": 0, "relevant_windows": gt_windows}], hl=False)
    _assert_bit_exact(pq, ref)
    assert pq["ap"][3, 0, -1] > 0  # the NaN pair is a true positive even at IoU 0.95


def test_compose_submission_feeds_eval_submission():
    from univtg_b200 import postproc

    B, Lv = 12, 75
    g = torch.Generator().manual_seed(5)
    logits = (torch.rand(B, Lv, 1, generator=g) * 16).round() / 16
    spans = torch.stack([-torch.rand(B, Lv, generator=g), torch.rand(B, Lv, generator=g)], dim=-1) * 0.1
    mask = torch.ones(B, Lv)
    mask[3:, 60:] = 0
    ts = ((torch.arange(Lv, dtype=torch.float32) + 0.5) / Lv)[None, :, None].expand(B, Lv, 2).contiguous()
    sal = torch.randn(B, Lv, generator=g)
    gt = make_eval_case(9, n_queries=B, durations=(150,))["ground_truth"]
    meta = [{"qid": d["qid"], "query": d["query"], "vid": d["vid"], "duration": d["duration"]} for d in gt]
    outputs = {"pred_logits": logits.cuda(), "pred_spans": spans.cuda(), "saliency_scores": sal.cuda()}
    for thd in (-1, 0.7):
        sub = postproc.compose_submission(meta, outputs, {"timestamp": ts.cuda(), "timestamp_mask": mask.cuda()},
                                          {"src_vid_mask": mask.cuda()}, nms_thd=thd)
        got = metrics.eval_submission(sub, gt)
        assert json.dumps(got) == json.dumps(M.eval_submission(sub, gt))
        assert list(got["brief"])[0] == "MR-full-R1@0.3-key"
