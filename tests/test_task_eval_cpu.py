"""Task-evaluation oracle (oracle/task_eval_oracle.py) pinned to the live reference's DatasetHL.evaluate and
calculate_semantic_matching through tests/golden/reference_task_eval.json; the ranking rule univtg_eval_hl_topk implements; the
input checks of univtg_b200.metrics.evaluate_hl and univtg_b200.qfvs.calculate_semantic_matching (host side, before any launch)."""
import hashlib
import json
import math
import os
import random

import numpy as np
import pytest
import torch

from oracle import task_eval_oracle as T
from tests.golden.make_golden_task_eval import hl_hash, hl_inputs, qfvs_hash
from tests.helpers import GOLDEN
from univtg_b200 import metrics, qfvs, synth


def _golden():
    with open(os.path.join(GOLDEN, "reference_task_eval.json")) as f:
        return json.load(f)


def _video_value(dset_name, aps):
    """What evaluate() returns unrounded for a one-video blob, from that video's per-annotator APs."""
    if dset_name == "tvsum":
        collected = [sum([a]) / 1 for a in aps]
    else:
        collected = [aps[0]]
    return sum(collected) / len(collected)


def test_golden_records_versions_and_cases():
    g = _golden()
    assert g["torch"] and g["networkx"] and g["scikit-learn"]
    assert len(g["hl"]) == 9 and len(g["qfvs"]) == 8


@pytest.mark.parametrize("i", range(9))
def test_hl_inputs_hash_to_the_golden_sha256(i):
    rec = _golden()["hl"][i]
    case, k = hl_inputs(rec["params"])
    assert hl_hash(case, k) == rec["sha256"], "make_hl_eval_case drifted from the golden inputs"


@pytest.mark.parametrize("i", range(8))
def test_qfvs_inputs_hash_to_the_golden_sha256(i):
    rec = _golden()["qfvs"][i]
    assert qfvs_hash(synth.make_qfvs_match_case(**rec["params"])) == rec["sha256"], "make_qfvs_match_case drifted"


@pytest.mark.parametrize("i", range(9))
def test_oracle_reproduces_the_reference_hl_evaluation(i):
    rec = _golden()["hl"][i]
    case, k = hl_inputs(rec["params"])
    name = case["dataset"].dset_name
    assert T.evaluate_hl(name, case["labels"], case["blob"], k) == rec["result"]
    aps = T.per_video_ap(name, case["labels"], case["blob"], k)
    assert [_video_value(name, a) for a in aps] == rec["per_video"]  # bit-exact floats


@pytest.mark.parametrize("i", range(8))
def test_oracle_reproduces_the_reference_semantic_matching(i):
    rec = _golden()["qfvs"][i]
    case = synth.make_qfvs_match_case(**rec["params"])
    opt, s, p, r, f1 = T.semantic_matching(case["machine"], case["gt"], case["tags"])
    assert abs(float(opt) - float(s)) <= 1e-12 * max(1.0, float(opt))
    for got, ref in zip((p, r, f1), rec["prf"]):
        assert isinstance(got, np.float64)
        if ref is None:
            assert math.isnan(got)
        else:
            assert got == pytest.approx(ref, rel=1e-12, abs=0)


# ---- ranking: torch.argsort(descending=True) on the CPU is libstdc++'s std::sort ---------------------------------------------
def _std_sort_order(x):
    """libstdc++ std::sort (introsort: threshold 16, median-of-three pivot, heap sort past depth 2*lg n, final insertion sort)
    of (value, index) pairs with comp = "a > b" -> the index order.  univtg_eval_hl_topk runs the same steps."""
    a = [(v, i) for i, v in enumerate(x)]
    less = lambda p, q: a[p][0] > a[q][0]  # noqa: E731

    def swap(p, q):
        a[p], a[q] = a[q], a[p]

    def adjust_heap(first, hole, n, val):
        top, child = hole, hole
        while child < (n - 1) // 2:
            child = 2 * (child + 1)
            if less(first + child, first + child - 1):
                child -= 1
            a[first + hole] = a[first + child]
            hole = child
        if n % 2 == 0 and child == (n - 2) // 2:
            child = 2 * (child + 1)
            a[first + hole] = a[first + child - 1]
            hole = child - 1
        parent = (hole - 1) // 2
        while hole > top and a[first + parent][0] > val[0]:
            a[first + hole] = a[first + parent]
            hole = parent
            parent = (hole - 1) // 2
        a[first + hole] = val

    def heap_sort(first, last):
        n = last - first
        if n >= 2:
            for parent in range((n - 2) // 2, -1, -1):
                adjust_heap(first, parent, n, a[first + parent])
        while last - first > 1:
            last -= 1
            val = a[last]
            a[last] = a[first]
            adjust_heap(first, 0, last - first, val)

    def introsort(first, last, depth):
        while last - first > 16:
            if depth == 0:
                heap_sort(first, last)
                return
            depth -= 1
            p, q, r = first + 1, first + (last - first) // 2, last - 1
            if less(p, q):
                m = q if less(q, r) else (r if less(p, r) else p)
            else:
                m = p if less(p, r) else (r if less(q, r) else q)
            swap(first, m)
            lo, hi = first + 1, last
            while True:
                while less(lo, first):
                    lo += 1
                hi -= 1
                while less(first, hi):
                    hi -= 1
                if not lo < hi:
                    break
                swap(lo, hi)
                lo += 1
            introsort(lo, last, depth)
            last = lo

    def linear_insert(i):
        val, j = a[i], i - 1
        while val[0] > a[j][0]:
            a[j + 1] = a[j]
            j -= 1
        a[j + 1] = val

    n = len(a)
    if n > 1:
        introsort(0, n, 2 * (n.bit_length() - 1))
        for i in range(1, min(n, 16)):
            if less(i, 0):
                val = a[i]
                a[1:i + 1] = a[0:i]
                a[0] = val
            else:
                linear_insert(i)
        for i in range(16, n):
            linear_insert(i)
    return [i for _, i in a]


def test_ties_come_out_in_index_order_up_to_16_elements():
    x = torch.tensor([.5, .1, .5, .5, .2, .5])
    assert torch.argsort(x, descending=True).tolist() == [0, 2, 3, 5, 4, 1]
    g = torch.Generator().manual_seed(0)
    for n in range(1, 17):
        for _ in range(20):
            x = torch.randint(0, 3, (n,), generator=g).float()
            assert torch.argsort(x, descending=True).tolist() == sorted(range(n), key=lambda j: (-x[j].item(), j))


def test_ties_beyond_16_elements_follow_std_sort_not_index_order():
    """Above 16 elements the CPU sort is an introsort: equal scores do not stay in index order.  The kernel runs the same
    introsort, so the reference's order is reproduced for every length up to 4,096 (and the heap-sort fallback too)."""
    x = torch.zeros(17)
    assert torch.argsort(x, descending=True).tolist() == [8, 16, 15, 14, 13, 12, 11, 10, 9, 0, 7, 6, 5, 4, 3, 2, 1]
    assert torch.argsort(x, descending=True, stable=True).tolist() == list(range(17))
    rng = random.Random(0)
    sizes = [17, 18, 31, 32, 33, 64, 100, 255, 256, 257, 1000, 1024, 2047, 2048, 4095, 4096]
    for n in sizes:
        for t in range(6):
            levels = [2, 3, 8, n // 4 + 1, n][t % 5]
            x = torch.tensor([rng.randrange(levels) / 8 for _ in range(n)], dtype=torch.float32)
            if t == 5:
                x = torch.tensor([0.0 if rng.random() < 0.5 else -0.0 for _ in range(n)])
            assert torch.argsort(x, descending=True).tolist() == _std_sort_order(x.tolist()), (n, t)
    # an organ-pipe sequence with pairs of equal values drives the introsort past its depth limit, into the heap-sort fallback
    x = torch.tensor([float(min(i, 4095 - i) // 2) for i in range(4096)])
    assert torch.argsort(x, descending=True).tolist() == _std_sort_order(x.tolist())


# ---- input checks (host side, before any launch) ----------------------------------------------------------------------------
def _hl(dset="tvsum", **kw):
    case = synth.make_hl_eval_case(3, dset, n_videos=3, clips=(10, 20, 30), shorter=0.0, **kw)
    return case["dataset"], case["blob"]


def test_hl_inputs_the_reference_cannot_evaluate():
    ds, blob = _hl()
    with pytest.raises(IndexError):
        metrics.evaluate_hl(ds, [torch.zeros(1, 11)] + blob[1:])  # 11 scores, 10 labelled clips
    ds.label[ds.get_video_id(1)]["anno"] = [row[:19] for row in ds.label[ds.get_video_id(1)]["anno"]]
    with pytest.raises(IndexError):
        metrics.evaluate_hl(ds, blob)
    with pytest.raises(ZeroDivisionError):
        metrics.evaluate_hl(ds, [])
    ds, blob = _hl("youtube")
    with pytest.raises(IndexError):
        metrics.evaluate_hl(ds, blob[:2] + [torch.zeros(2, 31)])
    ds.dset_name = "qvhighlight"
    with pytest.raises(NotImplementedError):
        metrics.evaluate_hl(ds, blob)


def test_hl_inputs_outside_the_domain_raise_value_error():
    ds, blob = _hl()
    bad = blob[0].clone()
    bad[0, 3] = float("nan")
    with pytest.raises(ValueError, match="non-finite scores"):
        metrics.evaluate_hl(ds, [bad] + blob[1:])
    with pytest.raises(ValueError, match="float32"):
        metrics.evaluate_hl(ds, [blob[0].double()] + blob[1:])
    with pytest.raises(ValueError, match="one score row"):
        metrics.evaluate_hl(ds, [blob[0][None]] + blob[1:])
    ds.label[ds.get_video_id(2)]["anno"][0][4] = float("inf")
    with pytest.raises(ValueError, match="non-finite labels"):
        metrics.evaluate_hl(ds, blob)
    big = synth.make_hl_eval_case(1, "youtube", n_videos=1, clips=(4097,), shorter=0.0, tie_frac=1.0)
    with pytest.raises(ValueError, match="4096"):
        metrics.evaluate_hl(big["dataset"], big["blob"])


def test_qfvs_inputs_the_reference_cannot_evaluate():
    case = synth.make_qfvs_match_case(5, 100, 10, 10)
    tags = [case["tags"]]
    with pytest.raises(ValueError, match="0 sample"):
        qfvs.calculate_semantic_matching([], case["gt"], tags, 0)
    with pytest.raises(ValueError, match="0 sample"):
        qfvs.calculate_semantic_matching(case["machine"], [], tags, 0)
    with pytest.raises(IndexError):
        qfvs.calculate_semantic_matching(case["machine"] + [100], case["gt"], tags, 0)
    with pytest.raises(IndexError):
        qfvs.calculate_semantic_matching(case["machine"], case["gt"], tags, 1)


def test_qfvs_inputs_outside_the_domain_raise_value_error():
    case = synth.make_qfvs_match_case(5, 2000, 10, 10)
    t = case["tags"].copy()
    t[case["machine"][0], 0] = 2
    with pytest.raises(ValueError, match="0 or 1"):
        qfvs.calculate_semantic_matching(case["machine"], case["gt"], [t], 0)
    wide = np.zeros((2000, 65), dtype=np.uint8)
    with pytest.raises(ValueError, match="64 tag columns"):
        qfvs.calculate_semantic_matching(case["machine"], case["gt"], [wide], 0)
    with pytest.raises(ValueError, match="1024"):
        qfvs.calculate_semantic_matching(list(range(1025)), case["gt"], [case["tags"]], 0)


def test_tag_masks_pack_each_column_into_its_bit():
    rng = np.random.default_rng(0)
    t = (rng.random((50, 48)) < 0.2).astype(np.uint8)
    m = qfvs.tag_masks(t)
    assert m.dtype == np.uint64 and m.shape == (50,)
    for row, mask in zip(t, m.tolist()):
        assert mask == sum(1 << c for c in np.flatnonzero(row).tolist())


def test_entry_points_raise_without_cuda(monkeypatch):
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    ds, blob = _hl()
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.evaluate_hl(ds, blob)
    case = synth.make_qfvs_match_case(5, 100, 10, 10)
    with pytest.raises(RuntimeError, match="CUDA"):
        qfvs.calculate_semantic_matching(case["machine"], case["gt"], [case["tags"]], 0)


def test_save_dir_file_is_written_first_with_the_reference_bytes(tmp_path, monkeypatch):
    """The reference writes <save_dir>/<dset_name>/<domain>.jsonl before it evaluates; so does evaluate_hl, byte for byte."""
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    for rec in (_golden()["hl"][0], _golden()["hl"][6]):
        case, k = hl_inputs(rec["params"])
        ds = case["dataset"]
        (tmp_path / ds.dset_name).mkdir()
        with pytest.raises(RuntimeError, match="CUDA"):
            metrics.evaluate_hl(ds, case["blob"], k=k, save_dir=str(tmp_path))
        data = (tmp_path / ds.dset_name / f"{ds.domain}.jsonl").read_bytes()
        assert hashlib.sha256(data).hexdigest() == rec["jsonl_sha256"]
