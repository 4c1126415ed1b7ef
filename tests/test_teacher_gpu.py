"""univtg_teacher_* (csrc/teacher.cu) through univtg_b200.teacher: the live reference's lines (tests/golden/reference_teacher.json)
byte for byte, the float64 oracle's labels exactly at the real class-table size, the tie and edge cases (duplicated class rows,
a video that needs the exhaustive fallback, parallel clips, zero rows, T = 1, trailing maxima, all-equal curves), chunking, and
the argument checks."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import teacher_oracle as O
from tests.golden.make_golden_teacher import layout, make_case
from tests.helpers import GOLDEN
from univtg_b200 import _lib, synth, teacher

pytestmark = pytest.mark.gpu


def _golden():
    with open(os.path.join(GOLDEN, "reference_teacher.json")) as f:
        return json.load(f)


def _labeler(case, **kw):
    return teacher.PseudoLabeler(torch.from_numpy(case["classes"]).cuda(), case["names"], **kw)


def _oracle(case, **kw):
    cls = torch.from_numpy(case["classes"]).cuda()
    return O.label(case["features"], case["vids"], cls, case["names"], **kw)


def _by_vid(lines):
    out = {}
    for line in lines:
        out.setdefault(json.loads(line)["vid"], []).append(line)
    return out


@pytest.mark.parametrize("i", range(len(_golden()["cases"])))
def test_golden_lines_byte_for_byte(i, tmp_path):
    g = _golden()["cases"][i]
    case = make_case(g["params"])
    assert synth.teacher_case_sha256(case) == g["sha256"]
    lab = _labeler(case)
    got = _by_vid(lab.lines(case["features"][:-1], case["vids"][:-1]))
    assert got == g["lines"]
    assert lab.fallback_videos == 0
    # the script's __main__: the same directory layout, videos sorted by name
    clip_dir, sf_dir = layout(case, str(tmp_path))
    out = tmp_path / "curve_5_window.jsonl"
    n = teacher.write_pseudo_labels(str(out), clip_dir, lab, slowfast_dir=sf_dir, batch_videos=7)
    want = [line for vid in sorted(g["lines"]) for line in g["lines"][vid]]
    assert out.read_text().splitlines() == want and n == len(want)


def test_real_size_equals_oracle():
    case = synth.make_teacher_case(21, n_classes=19994, dim=512, n_videos=2000, clips=(1, 300), lengths=(4096, 4096, 4096),
                                   dup=12)
    lab = _labeler(case)
    got = lab(case["features"], case["vids"])
    assert lab.fallback_videos == 0
    want = _oracle(case)
    assert len(want) > 4000
    assert got == want
    assert lab.lines(case["features"], case["vids"]) == O.lines(want)


def test_duplicated_classes_inside_the_top_k():
    case = synth.make_teacher_case(22, n_classes=19994, dim=512, n_videos=40, dup=12, dup_top=True)
    lab = _labeler(case)
    got = lab.lines(case["features"], case["vids"])
    want = O.lines(_oracle(case))
    assert got == want
    cls = torch.from_numpy(case["classes"]).cuda()
    mm = O.cosines(case["features"][0], cls)
    top = torch.sort(mm.sum(0), descending=True, stable=True)[1][:5].tolist()
    pair = [c for c in top if c in case["dup_rows"]]
    assert len(pair) >= 2 and torch.equal(cls[pair[0]], cls[pair[1]]) and pair[0] < pair[1]


def test_uncertifiable_video_falls_back_to_every_class():
    case = synth.make_teacher_case(23, n_classes=19994, dim=512, n_videos=30, copies=40)
    lab = _labeler(case)
    got = lab(case["features"], case["vids"])
    assert lab.fallback_videos > 0
    assert got == _oracle(case)
    first = [s["qid"] for s in got if s["vid"] == case["vids"][0]]
    assert first == sorted(first)  # five copies of one row: the lowest indices, in index order


def test_edge_videos_equal_oracle():
    case = synth.make_teacher_case(24, n_classes=3000, dim=512, n_videos=10, dup=12)
    lab = _labeler(case)
    got = lab(case["features"], case["vids"])
    want = _oracle(case)
    assert got == want
    assert lab.lines(case["features"], case["vids"]) == O.lines(want)
    vids = {s["vid"] for s in got}
    assert not any(v.endswith(("_one", "_equal")) for v in vids)
    par = [s for s in got if s["vid"].endswith("_parallel")]
    assert any(s["saliency_scores"][2] == [19.0] for s in par)
    zero = [s for s in got if s["vid"].endswith("_zero")]
    assert zero and all(s["saliency_scores"][3] == [0.0] for s in zero)


def test_small_class_tables():
    for C in (1, 3, 16, 17, 40):
        case = synth.make_teacher_case(30 + C, n_classes=C, dim=24, n_videos=8)
        for topk in (1, 5, 16):
            lab = _labeler(case, topk=topk, th=0.1, clip_len=1.5)
            assert lab(case["features"], case["vids"]) == _oracle(case, topk=topk, th=0.1, clip_len=1.5), (C, topk)


def test_cuda_sort_orders_ties_by_index():
    g = torch.Generator().manual_seed(5)
    x = torch.randn(19994, generator=g)
    dst = torch.randperm(19994, generator=g)[:200]
    x[dst[100:]] = x[dst[:100]]
    x[:50] = 0.25
    idx = torch.sort(x.cuda(), descending=True)[1].cpu()
    assert torch.equal(idx, torch.sort(x, descending=True, stable=True)[1])


def test_chunking_gives_identical_output():
    case = synth.make_teacher_case(25, n_classes=2000, dim=512, n_videos=60, clips=(1, 90))
    feats = case["features"]
    feats[5] = np.zeros((0, 512), np.float32)
    lab = _labeler(case)
    whole = lab.lines(feats, case["vids"])
    cuts = [0, 1, 8, 9, 30, 31, len(feats)]
    parts = [x for a, b in zip(cuts[:-1], cuts[1:]) for x in lab.lines(feats[a:b], case["vids"][a:b])]
    single = [x for f, v in zip(feats, case["vids"]) for x in lab.lines([f], [v])]
    lab._max_videos, lab._max_clips = 7, 200
    small = lab.lines(feats, case["vids"])
    on_device = lab.lines([torch.from_numpy(f).cuda() for f in feats], case["vids"])
    assert whole == parts == single == small == on_device
    assert not any(json.loads(x)["vid"] == case["vids"][5] for x in whole)


def test_bad_arguments_raise_before_any_launch():
    lib = _lib.load_library()
    cls = torch.randn(30, 16, device="cuda")
    names = [str(i) for i in range(30)]
    n0 = lib.univtg_launch_count()
    for kw in (dict(topk=0), dict(topk=17), dict(th=0.0), dict(th=-0.05), dict(th=float("nan")), dict(clip_len=0)):
        with pytest.raises(ValueError):
            teacher.PseudoLabeler(cls, names, **kw)
    with pytest.raises(ValueError):
        teacher.PseudoLabeler(cls, names[:-1])
    with pytest.raises(ValueError):
        teacher.PseudoLabeler(cls.double(), names)
    with pytest.raises(ValueError):
        teacher.PseudoLabeler(torch.randn(30, 2048, device="cuda"), names)
    assert lib.univtg_launch_count() == n0
    lab = teacher.PseudoLabeler(cls, names)
    n0 = lib.univtg_launch_count()
    ok = np.zeros((4, 16), np.float32)
    for feats in ([ok.astype(np.float64)], [np.zeros((4, 15), np.float32)], [np.zeros((65536, 16), np.float32)], [ok.tolist()]):
        with pytest.raises(ValueError):
            lab(feats, ["v"])
    with pytest.raises(ValueError):
        lab([ok, ok], ["v"])
    with pytest.raises(RuntimeError, match="CUDA"):
        lab([torch.from_numpy(ok)], ["v"])
    assert lib.univtg_launch_count() == n0
