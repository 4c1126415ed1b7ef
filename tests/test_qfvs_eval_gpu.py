"""univtg_b200.qfvs.eval_epoch on the device: against the live reference's lines and dicts (tests/golden/reference_qfvs_eval.json)
with the replaying model, against the per-file restatement (tests/qfvs_eval_oracle.py) with the real model (batched forwards
equal per-file forwards bit for bit), the tie rule of univtg_qfvs_eval_select against torch.topk on CUDA, refusals before any
launch, and no host synchronisation in a select call."""
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

from tests import qfvs_eval_oracle as O
from tests.golden import make_golden_qfvs_eval as M
from univtg_b200 import _lib, qfvs, synth
from univtg_b200.qfvs import build_model

pytestmark = pytest.mark.gpu
CASES = O.golden_cases()


def _run(model, p, tmp, monkeypatch, **kw):
    monkeypatch.setitem(sys.modules, "h5py", synth.h5py_stub())
    monkeypatch.chdir(tmp)
    res = qfvs.eval_epoch(model, M.case_config(p), M.case_opt(p), **kw)
    path = os.path.join(tmp, M.jsonl_path(p))
    text = open(path).read() if os.path.exists(path) else None
    return res, text


@pytest.mark.parametrize("case", CASES, ids=[c["params"]["name"] for c in CASES])
@pytest.mark.parametrize("rows", [qfvs.ROWS_PER_FORWARD, 4])  # one forward per variant, and one file per forward
def test_device_epoch_matches_the_reference(case, rows, monkeypatch):
    p = case["params"]
    model = synth.QFVSReplayModel(p["seed"]).cuda()
    with tempfile.TemporaryDirectory() as tmp:
        M.build_tree(p, tmp)
        if case["error"]:
            with pytest.raises({"ValueError": ValueError, "IndexError": IndexError}[case["error"]]):
                _run(model, p, tmp, monkeypatch, rows_per_forward=rows)
            assert open(os.path.join(tmp, M.jsonl_path(p))).read() == case["jsonl_on_error"]
            assert model.calls == 0
            return
        res, text = _run(model, p, tmp, monkeypatch, rows_per_forward=rows)
        res_train, _ = _run(model, p, tmp, monkeypatch, write_jsonl=False, rows_per_forward=rows)
    got = M.lines_by_file(p, text)
    assert sorted(got) == sorted(case["lines"])
    for f, line in got.items():
        O.assert_line_matches(line, case["lines"][f], f"{p['name']} {f}")
    O.assert_result_matches(res, case["inference"], p["name"])
    O.assert_result_matches(res_train, case["train"], p["name"] + " train")


@pytest.mark.parametrize("name,over", [("ensemble_gather", {}), ("logits_no_gather", {"ensemble": 0, "gather": 0}),
                                       ("saliency", {"f_coef": 0.0})])
def test_real_model_epoch_equals_per_file_forwards(name, over, monkeypatch):
    cfg = synth.CONFIGS["tiny"]
    p = M.case_params(dict(over, name=name, seed=31, S=6, Lf=40, seg_len=(40,) * 5 + (17,), files=M.FILES6, shots=(200,) * 4,
                           top_percent=0.1))
    model, _ = build_model(synth.reference_args(cfg, device="cuda", dset_type="vs"))
    model.load_state_dict(synth.make_state_dict(cfg, seed=5), strict=True)
    model.cuda().eval()
    with tempfile.TemporaryDirectory() as tmp:
        synth.write_qfvs_eval_tree(tmp, p["seed"], S=p["S"], Lf=p["Lf"], seg_len=p["seg_len"], dv=cfg["v_feat_dim"] - 2,
                                   dt=cfg["t_feat_dim"], shots=p["shots"], files=p["files"], gt_sizes=(9, 12, 4))
        with torch.no_grad():
            want, want_res = O.eval_epoch(model, M.case_config(p), M.case_opt(p), tmp, device="cuda")
        res, text = _run(model, p, tmp, monkeypatch, rows_per_forward=3 * p["S"])  # two chunks per token-count group at most
    got = M.lines_by_file(p, text)
    assert sorted(got) == sorted(f for f, _ in want)
    for f, line in want:
        O.assert_line_matches(got[f], line, f"{name} {f}")
    O.assert_result_matches(res, want_res, name)


def _select(scores, k, pos=None):
    """univtg_qfvs_eval_select in saliency mode, no gather, on [F, N] scores -> (score [F, n], top [F, k], tag masks [F, k])."""
    lib = _lib.load_library()
    F, N = scores.shape
    pos = torch.arange(N, dtype=torch.int32, device="cuda") if pos is None else pos
    n = pos.numel()
    tags = torch.arange(n, dtype=torch.int64, device="cuda") * 3 + 1
    out = (torch.empty(F, n, device="cuda"), torch.empty(F, k, dtype=torch.int32, device="cuda"),
           torch.empty(F, k, dtype=torch.int64, device="cuda"))
    _lib.check(lib.univtg_qfvs_eval_select(None, None, None, None, None, _lib.ptr(scores), _lib.ptr(pos), _lib.ptr(tags), F, N, n, k,
                                           1, 0, 0, *[_lib.ptr(t) for t in out], _lib.stream_ptr()), "univtg_qfvs_eval_select")
    return out, tags


@pytest.mark.parametrize("n,k", [(7, 3), (9, 8), (40, 9), (300, 17), (4000, 32), (4000, 33), (100, 100), (1000, 37), (4000, 80),
                                 (8192, 500), (5000, 5000)])
def test_ties_and_nan_order_as_torch_topk_on_cuda(n, k):
    """Up to k = 32 torch.topk sorts its selection with an unstable bitonic network, above that stably (ties by index)."""
    g = torch.Generator().manual_seed(n + k)
    F = 3
    s = (torch.randint(-4, 5, (F, n), generator=g).float() / 4)  # a handful of values: ties everywhere
    s[0, torch.randint(0, n, (max(1, n // 50),), generator=g)] = float("nan")
    s[1, torch.randint(0, n, (max(1, n // 50),), generator=g)] = float("-inf")
    s[2, :] = 0.0
    s = s.cuda()
    (score, top, a), tags = _select(s, k)
    for f in range(F):
        _, want = s[f].topk(k)
        assert torch.equal(top[f].long(), want), f"row {f}: {top[f][:20].tolist()} vs {want[:20].tolist()}"
        assert torch.equal(a[f], tags[want])
    assert torch.equal(score.view(torch.int32), s.view(torch.int32))


def test_cuda_topk_orders_ties_of_large_results_by_index():
    x = torch.zeros(4000, device="cuda")
    x[::7] = 1.0
    _, idx = x.topk(1000)
    ones = torch.arange(0, 4000, 7, device="cuda")
    assert torch.equal(idx[:len(ones)], ones)
    assert torch.equal(idx[len(ones):], torch.tensor([i for i in range(4000) if i % 7], device="cuda")[:1000 - len(ones)])


def test_select_does_not_synchronise():
    s = torch.randn(20, 4000, device="cuda")
    _select(s, 80)  # library load, function attributes
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)  # ~50 ms at the H100's clocks
    ev = torch.cuda.Event()
    ev.record()
    _select(s, 80)
    pending = not ev.query()
    torch.cuda.synchronize()
    assert pending, "the select call waited for the GPU"


@pytest.mark.parametrize("what,exc", [("k0", ValueError), ("gt_index", IndexError), ("shape", RuntimeError), ("side", ValueError),
                                      ("cpu", RuntimeError)])
def test_refusals_launch_nothing(what, exc, monkeypatch):
    from tests.test_qfvs_eval_cpu import _refusal_tree

    lib = _lib.load_library()
    model = synth.QFVSReplayModel(1)
    if what != "cpu":
        model = model.cuda()
    torch.cuda.synchronize()
    before = lib.univtg_launch_count()
    with tempfile.TemporaryDirectory() as tmp:
        cfg, opt = _refusal_tree(tmp, what)
        monkeypatch.setitem(sys.modules, "h5py", synth.h5py_stub())
        monkeypatch.chdir(tmp)
        with pytest.raises(exc):
            qfvs.eval_epoch(model, cfg, opt)
    assert model.calls == 0 and lib.univtg_launch_count() == before
