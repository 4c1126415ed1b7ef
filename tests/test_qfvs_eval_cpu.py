"""The QFVS evaluation epoch on the host: the restatement (tests/qfvs_eval_oracle.py) against the live reference's lines and
dicts (tests/golden/reference_qfvs_eval.json), the refusals of univtg_b200.qfvs.eval_epoch and of univtg_qfvs_eval_select
(raised before any launch), and the ptxas record of the selection kernel."""
import json
import os
import re
import subprocess
import sys
import tempfile

import pytest

import __graft_entry__ as G
from tests import qfvs_eval_oracle as O
from tests.golden import make_golden_qfvs_eval as M
from univtg_b200 import _lib, qfvs, synth

CASES = O.golden_cases()
OK = [c for c in CASES if c["error"] is None]


def test_golden_covers_the_branches():
    p = [c["params"] for c in CASES]
    assert {(x["f_coef"] == 0, x["s_coef"] == 0, x["ensemble"]) for x in p} >= {(False, False, 1), (False, False, 0), (True, False, 1),
                                                                              (False, True, 1)}
    assert {x["gather"] for x in p} == {0, 1}
    ks = {len(json.loads(next(iter(c["lines"].values())))["top_pred"]) for c in OK}
    assert 1 in ks and max(ks) > 10
    assert any(c["error"] == "ValueError" and c["jsonl_on_error"] == "" for c in CASES)
    assert any(len({len(json.loads(x)["score"]) for x in c["lines"].values()}) == 1 and json.loads(next(iter(c["lines"].values())))["shots"] <
               sum(c["params"]["seg_len"]) for c in OK)


@pytest.mark.parametrize("case", OK, ids=[c["params"]["name"] for c in OK])
def test_restatement_reproduces_the_reference(case):
    p = case["params"]
    with tempfile.TemporaryDirectory() as tmp:
        M.build_tree(p, tmp)
        lines, res = O.eval_epoch(synth.QFVSReplayModel(p["seed"]), M.case_config(p), M.case_opt(p), tmp)
    assert sorted(f for f, _ in lines) == sorted(case["lines"])
    for f, line in lines:
        O.assert_line_matches(line, case["lines"][f], f"{p['name']} {f}")
    O.assert_result_matches(res, case["inference"], p["name"])
    O.assert_result_matches(res, case["train"], p["name"] + " train")


def _refusal_tree(tmp, what):
    p = M.case_params({"name": what})
    if what == "k0":
        p["top_percent"] = 0.001
    if what == "gt_index":
        p["gt_extra"] = ((61,), (), ())
    if what == "empty_gt":
        p["gt_sizes"], p["gt_extra"] = (0, 3, 3), ()
    if what == "seg_len":
        p["seg_len"] = (16, 16, 16, 17)
    M.build_tree(p, tmp)
    cfg, opt = M.case_config(p), M.case_opt(p)
    if what == "shape":
        cfg["max_frame_num"] = p["Lf"] + 1
    if what == "side":  # k = 2,000 machine shots, over the matching's 1,024
        p["shots"] = (2000, 60, 60, 60)
        p["S"], p["Lf"], p["seg_len"], p["top_percent"] = 20, 100, (100,) * 20, 1.0
        M.build_tree(p, tmp)
        cfg = M.case_config(p)
    return cfg, opt


@pytest.mark.parametrize("what,exc", [("k0", ValueError), ("gt_index", IndexError), ("empty_gt", ValueError), ("seg_len", IndexError),
                                      ("shape", RuntimeError), ("side", ValueError), ("cpu", RuntimeError)])
def test_refusals_raise_before_the_model_runs(what, exc, monkeypatch):
    monkeypatch.setitem(sys.modules, "h5py", synth.h5py_stub())
    model = synth.QFVSReplayModel(1)
    with tempfile.TemporaryDirectory() as tmp:
        cfg, opt = _refusal_tree(tmp, what)
        monkeypatch.chdir(tmp)
        with pytest.raises(exc):
            qfvs.eval_epoch(model, cfg, opt)
        assert open(os.path.join(tmp, "plot", "qfvs", "1.jsonl")).read() == ""
    assert model.calls == 0


def test_select_rejects_bad_arguments_without_launching():
    lib = _lib.load_library()
    fake = _lib.c_void_p(0x1000)
    good = dict(F=2, N=64, n=50, k=5, mode=2, gather=1, q0=0)
    for over in ({"n": 0}, {"n": 65}, {"k": 0}, {"k": 51}, {"mode": 3}, {"gather": 2}, {"q0": -1}, {"N": 9000, "n": 8193}):
        a = dict(good, **over)
        rc = lib.univtg_qfvs_eval_select(*[fake] * 8, a["F"], a["N"], a["n"], a["k"], a["mode"], a["gather"], a["q0"], fake, fake, fake,
                                         None)
        assert rc == 1 and "univtg_qfvs_eval_select: bad argument" in _lib.last_error(), over
    # variant 1 and 2 outputs are read only with gather = 1; the logits only in modes 0 and 2
    rc = lib.univtg_qfvs_eval_select(fake, fake, None, fake, fake, fake, fake, fake, 2, 64, 50, 5, 0, 1, 0, fake, fake, fake, None)
    assert rc == 1
    # without gather, saliency mode reads only the both-concepts saliency (F = 0: accepted, nothing launched)
    rc = lib.univtg_qfvs_eval_select(None, None, None, None, None, fake, fake, fake, 0, 64, 50, 5, 1, 0, 0, fake, fake, fake, None)
    assert rc == 0


def _ptxas_select():
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [G._nvcc()] + G.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(G.CSRC, "task_eval.cu"), "-o", os.path.join(tmp, "t.o")]
        log = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    lines = log.splitlines()
    i = next(j for j, x in enumerate(lines) if "Function properties for" in x and "qfvs_eval_select_kernel" in x)
    return lines[i + 1] + "\n" + lines[i + 2]


def test_select_kernel_does_not_spill():
    rec = _ptxas_select()
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", rec)
    assert m and m.groups() == ("0", "0", "0"), rec
    assert int(re.search(r"Used (\d+) registers", rec).group(1)) <= 64, rec  # 1,024 threads per block
