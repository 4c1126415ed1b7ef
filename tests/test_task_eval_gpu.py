"""univtg_eval_hl_topk / univtg_qfvs_match (csrc/task_eval.cu) and their drop-ins univtg_b200.metrics.evaluate_hl and
univtg_b200.qfvs.calculate_semantic_matching: per-(video, annotator) APs bit-exact against the oracle, the matching optimum
within 1e-12 of the exact one, the returned values equal to the live reference's (tests/golden/reference_task_eval.json)."""
import hashlib
import json
import math
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import task_eval_oracle as T
from tests.golden.make_golden_task_eval import hl_inputs
from tests.helpers import GOLDEN
from univtg_b200 import metrics, qfvs, synth

pytestmark = pytest.mark.gpu


def _golden():
    with open(os.path.join(GOLDEN, "reference_task_eval.json")) as f:
        return json.load(f)


def _device_ap(case, k=5, device="cuda"):
    ds, blob = case["dataset"], case["blob"]
    rows = [b[0].to(device) for b in blob]
    labels, n_label, n_cut, median = metrics.pack_hl_labels(ds, len(rows), [r.numel() for r in rows], k)
    return metrics.hl_topk_ap(rows, labels, n_label, n_cut, median)


def _assert_ap_bit_exact(case, k=5, device="cuda"):
    dev = _device_ap(case, k, device)
    ref = np.array(T.per_video_ap(case["dataset"].dset_name, case["labels"], case["blob"], k), dtype=np.float64)
    assert dev.shape == ref.shape
    assert dev.view(np.int64).tolist() == ref.view(np.int64).tolist(), np.argwhere(dev != ref)[:5]
    return dev


@pytest.mark.parametrize("i", range(9))
def test_evaluate_hl_equals_the_reference_on_golden_cases(i, tmp_path):
    rec = _golden()["hl"][i]
    case, k = hl_inputs(rec["params"])
    ds = case["dataset"]
    dev = _assert_ap_bit_exact(case, k)
    name = ds.dset_name
    values = []
    for v in range(len(dev)):
        collected = [sum([a]) / 1 for a in dev[v].tolist()] if name == "tvsum" else [dev[v, 0].item()]
        values.append(sum(collected) / len(collected))
    assert values == rec["per_video"]
    cuda_blob = [b.cuda() for b in case["blob"]]
    (tmp_path / name).mkdir()
    assert metrics.evaluate_hl(ds, cuda_blob, k=k, save_dir=str(tmp_path)) == rec["result"]
    data = (tmp_path / name / f"{ds.domain}.jsonl").read_bytes()
    assert hashlib.sha256(data).hexdigest() == rec["jsonl_sha256"]
    assert metrics.evaluate_hl(ds, case["blob"], k=k) == rec["result"]  # CPU entries


@pytest.mark.parametrize("dset", ["tvsum", "youtube"])
def test_device_ap_equals_the_oracle_over_many_seeds(dset):
    for seed in range(40):
        clips = [(5, 16, 17, 40), (75, 120, 200), (1, 2, 3, 300)][seed % 3]
        k = [5, 1, 20, 500, 0][seed % 5]
        case = synth.make_hl_eval_case(100 + seed, dset, n_videos=5, clips=clips, shorter=0.3, tie_frac=[0.0, 0.5, 1.0][seed % 3])
        _assert_ap_bit_exact(case, k, device="cuda" if seed % 2 else "cpu")
        assert metrics.evaluate_hl(case["dataset"], case["blob"], k=k) == T.evaluate_hl(dset, case["labels"], case["blob"], k)


@pytest.mark.parametrize("dset", ["tvsum", "youtube"])
def test_device_ap_at_4096_clips_with_ties(dset):
    case = synth.make_hl_eval_case(7, dset, n_videos=3, clips=(4096, 4095, 2049), shorter=0.0, tie_frac=1.0)
    ap = _assert_ap_bit_exact(case, k=4096)
    assert ap.shape == (3, 20 if dset == "tvsum" else 1)
    # scores in equal pairs along an organ pipe: the introsort falls back to heap sort
    case["blob"][0] = torch.tensor([[float(min(i, 4095 - i) // 2) for i in range(4096)]])
    _assert_ap_bit_exact(case, k=4096)


def test_fp16_scores_rank_as_the_reference_ranks_them():
    case = synth.make_hl_eval_case(8, "youtube", n_videos=4, clips=(300, 40), shorter=0.0, tie_frac=0.5)
    case["blob"] = [b.half() for b in case["blob"]]
    _assert_ap_bit_exact(case)
    assert metrics.evaluate_hl(case["dataset"], [b.cuda() for b in case["blob"]]) == \
        T.evaluate_hl("youtube", case["labels"], case["blob"])


# ---- QFVS semantic matching --------------------------------------------------------------------------------------------------
def _masks(case):
    return qfvs.tag_masks(case["tags"][case["machine"]]), qfvs.tag_masks(case["tags"][case["gt"]])


def test_matching_sum_is_the_exact_optimum_at_the_real_sizes():
    cases = [synth.make_qfvs_match_case(200 + i, n, m, m) for i, (n, m) in enumerate(((2152, 43), (3692, 73), (3588, 71), (2783, 55)))]
    cases += [synth.make_qfvs_match_case(300 + i, 500, a, b, zero_frac=0.1) for i, (a, b) in enumerate(((1, 7), (7, 1), (30, 12),
                                                                                                         (12, 30), (64, 64)))]
    got = qfvs.match_sums([_masks(c) for c in cases])
    for c, s in zip(cases, got.tolist()):
        opt = float(T.semantic_matching(c["machine"], c["gt"], c["tags"])[0])
        assert abs(s - opt) <= 1e-12 * max(opt, 1.0), (s, opt)


@pytest.mark.parametrize("n,extra", [(1024, 0), (1000, 24), (257, 700)])
def test_matching_finds_a_hidden_permutation_at_the_size_bound(n, extra):
    c = synth.make_qfvs_permutation_case(5, n, extra)
    s = qfvs.match_sums([_masks(c)])[0]
    assert s == c["optimum"]
    p, r, f1 = qfvs.calculate_semantic_matching(c["machine"], c["gt"], [c["tags"]], 0)
    assert (p, r) == (1.0, n / (n + extra))


def test_matching_of_random_1024_shot_summaries_against_scipy():
    scipy_opt = pytest.importorskip("scipy.optimize")
    c = synth.make_qfvs_match_case(9, 4000, 1024, 1024)
    a, b = c["tags"][c["machine"]].astype(np.int64), c["tags"][c["gt"]].astype(np.int64)
    inter, union = a @ b.T, a.shape[1] - (1 - a) @ (1 - b).T
    w = np.where(union > 0, inter / np.maximum(union, 1), 0.0)
    ri, ci = scipy_opt.linear_sum_assignment(w, maximize=True)
    s = qfvs.match_sums([_masks(c)])[0]
    assert s == pytest.approx(float(w[ri, ci].sum()), rel=1e-12, abs=0)


def test_all_zero_weights_give_nan_f1():
    c = synth.make_qfvs_match_case(18, 120, 20, 20, zero_frac=1.0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        p, r, f1 = qfvs.calculate_semantic_matching(c["machine"], c["gt"], [c["tags"]], 0)
    assert (p, r) == (0.0, 0.0) and math.isnan(f1)
    assert all(isinstance(x, np.float64) for x in (p, r, f1))


@pytest.mark.parametrize("i", range(8))
def test_calculate_semantic_matching_equals_the_reference(i):
    rec = _golden()["qfvs"][i]
    c = synth.make_qfvs_match_case(**rec["params"])
    top_index = torch.tensor(c["machine"], device="cuda")  # what score.topk returns, passed as it is
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        got = qfvs.calculate_semantic_matching(top_index, c["gt"], [c["tags"]], 0)
    for x, ref in zip(got, rec["prf"]):
        assert isinstance(x, np.float64)
        if ref is None:
            assert math.isnan(x)
        else:
            assert x == pytest.approx(ref, rel=1e-12, abs=0)
