"""CLIP-teacher pseudo labels without a GPU: the float64 oracle (oracle/teacher_oracle.py) against the live reference's lines
(tests/golden/reference_teacher.json), the host build of the curves' floor division (univtg_debug_py_floordiv, the function the
kernel runs) against Python's //, and the argument checks of univtg_b200.teacher."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import teacher_oracle as O
from tests.golden.make_golden_teacher import make_case
from tests.helpers import GOLDEN
from univtg_b200 import _lib, synth, teacher


def _golden():
    with open(os.path.join(GOLDEN, "reference_teacher.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("i", range(len(_golden()["cases"])))
def test_oracle_lines_equal_reference(i):
    g = _golden()["cases"][i]
    case = make_case(g["params"])
    assert synth.teacher_case_sha256(case) == g["sha256"]
    cls = torch.from_numpy(case["classes"])
    kept = case["vids"][:-1]  # the last video has no slowfast file
    for vid, f in zip(case["vids"][:-1], case["features"][:-1]):
        got = O.lines(O.label_video(f, cls, case["names"], vid))
        assert got == g["lines"].get(vid, []), vid
    assert set(g["lines"]) <= set(kept)


def test_golden_covers_the_edge_cases():
    g = _golden()
    n_lines = sum(len(v) for c in g["cases"] for v in c["lines"].values())
    assert n_lines > 200
    lines = [json.loads(x) for c in g["cases"] for v in c["lines"].values() for x in v]
    assert any(len(x["relevant_windows"]) > 1 for x in lines)
    assert any(x["query"] in synth.TEACHER_SPECIAL_NAMES for x in lines)
    vids = {v for c in g["cases"] for v in c["lines"]}
    assert not any(v.endswith("_one") or v.endswith("_equal") for v in vids)  # T = 1 and all-equal curves write no line


def _floordiv(x, th):
    lib = _lib.load_library()
    x = np.ascontiguousarray(x, dtype=np.float64)
    out = np.empty_like(x)
    _lib.check(lib.univtg_debug_py_floordiv(x.ctypes.data, x.size, th, out.ctypes.data), "univtg_debug_py_floordiv")
    return out


def _same(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


@pytest.mark.parametrize("th", [0.05, 0.1, 0.03])
def test_floordiv_equals_python_near_every_bin_edge(th):
    edges = np.float32(np.arange(-int(1 / th) - 1, int(1 / th) + 2) * th)
    edges = edges[np.abs(edges) <= 1.0]
    bits = edges.view(np.int32).astype(np.int64)
    vals = []
    for b, e in zip(bits, edges):
        if e == 0:
            pos = np.arange(0, 2001, dtype=np.int64)
            vals += [pos.astype(np.int32).view(np.float32), (pos | 0x80000000).astype(np.uint32).view(np.float32)]
        else:
            vals.append((b + np.arange(-2000, 2001)).astype(np.int32).view(np.float32))
    rng = np.random.default_rng(int(th * 1000))
    vals.append(rng.uniform(-1.0, 1.0, 10 ** 6).astype(np.float32))
    x = np.concatenate(vals).astype(np.float64)
    got = _floordiv(x, th)
    ref = np.array([v // th for v in x.tolist()])
    bad = np.flatnonzero(got.view(np.int64) != ref.view(np.int64))
    assert bad.size == 0, [(x[i], got[i], ref[i]) for i in bad[:5]]


def test_floordiv_known_values():
    x = [0.25, 0.5, 0.75, 1.0, -0.0, 0.0, -1e-10, -1.0, 0.049999999999999996]
    assert _same(_floordiv(x, 0.05), [4.0, 9.0, 14.0, 19.0, -0.0, 0.0, -1.0, -20.0, 0.0])
    assert _same(_floordiv(x, 0.05), [v // 0.05 for v in x])
    assert np.floor(1.0 / 0.05) == 20.0  # what a naive port would give


def test_oracle_tie_rule_and_windows():
    cls = torch.tensor([[1.0, 0.0], [0.0, 1.0], [1.0, 0.0], [1.0, 1.0]])
    feats = np.array([[1.0, 0.0], [0.0, 1.0], [1.0, 0.0], [0.5, 0.5]], np.float32)
    s = O.label_video(feats, cls, ["a", "b", "a2", "ab"], "v", topk=4)
    # sums: 3 > 0 == 2 > 1; class 3's maximum (a parallel clip, 1.0 // 0.05 = 19) is only at the last clip: no line
    assert [x["qid"] for x in s] == [0, 2, 1]
    assert s[0]["saliency_scores"] == [[19.0], [0.0], [19.0], [14.0]]
    assert s[0]["relevant_windows"] == [[0, 2], [4, 6]] and s[2]["relevant_windows"] == [[2, 4]]
    assert O.create_window([1, 3, 3, 0, 3], 2) == [[2, 6]]
    assert O.create_window([3, 3, 3], 2) == []
    assert O.create_window([3, 1, 3, 3, 1, 2], 2) == [[0, 2], [4, 8]]


def test_bad_arguments_raise_before_any_launch():
    lib = _lib.load_library()
    n0 = lib.univtg_launch_count()
    with pytest.raises(RuntimeError, match="CUDA"):
        teacher.PseudoLabeler(torch.zeros(10, 8), ["x"] * 10)
    assert lib.univtg_launch_count() == n0
    assert lib.univtg_teacher_label(None, None, 10, 8, None, None, 1, 1, 5, 0.05, None, 0, None, None) != 0
    assert "bad argument" in _lib.last_error()
    x = np.zeros(4)
    assert lib.univtg_teacher_label(x.ctypes.data, x.ctypes.data, 10, 8, x.ctypes.data, x.ctypes.data, 1, 1, 17, 0.05,
                                    x.ctypes.data, 1 << 20, x.ctypes.data, None) != 0
    assert lib.univtg_teacher_label(x.ctypes.data, x.ctypes.data, 10, 8, x.ctypes.data, x.ctypes.data, 1, 1, 5, 0.0,
                                    x.ctypes.data, 1 << 20, x.ctypes.data, None) != 0
    assert lib.univtg_teacher_label(x.ctypes.data, x.ctypes.data, 10, 2048, x.ctypes.data, x.ctypes.data, 1, 1, 5, 0.05,
                                    x.ctypes.data, 1 << 20, x.ctypes.data, None) != 0
    assert lib.univtg_teacher_class_bytes(10, 2048) == 0
    assert lib.univtg_launch_count() == n0


def test_class_names_from_csv_and_json(tmp_path):
    csv_path = tmp_path / "oidv6-class-descriptions.csv"
    csv_path.write_text('LabelName,DisplayName\n/m/01,Ball\n/m/02,"Sprenger\'s, tulip"\n/m/03,Crème brûlée\n', encoding="utf-8")
    assert teacher.read_class_names(str(csv_path)) == ["Ball", "Sprenger's, tulip", "Crème brûlée"]
    js = tmp_path / "names.json"
    js.write_text(json.dumps(["a", "b"]))
    assert teacher.read_class_names(str(js)) == ["a", "b"]
