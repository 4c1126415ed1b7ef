#!/usr/bin/env python
"""Writes tests/golden/reference_eval_epoch.json: what the live reference `main.inference_mr.eval_epoch` writes and returns on the
seeded cases below, so the evaluation-epoch restatement (tests/eval_epoch_oracle.py) and the device path
(univtg_b200/evaluation.py) stay pinned without the reference.

Each case runs the unmodified eval_epoch on CPU tensors (h5py / nncore stubbed, opt.device = "cpu") with
univtg_b200.synth.EvalEpochDataset, univtg_b200.synth.ReplayEvalModel and, when the case has a criterion, the reference's
SetCriterion (model/univtg.py, the weights and losses build_model gives an mr run).  Stored per case: its parameters, the
sha256 and size of every file written to results_dir, the returned metrics / metrics_nms (as json.dumps strings, key order included), the
returned paths relative to results_dir, the loss-meter fields, every tb_writer.add_scalar call and every batch's loss values
(float(v) of the criterion's fp32 results).

Usage: python tests/golden/make_golden_eval_epoch.py <path to a showlab/UniVTG checkout>"""
import hashlib
import json
import os
import sys
import tempfile
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from univtg_b200 import synth  # noqa: E402

WEIGHTS = {"loss_b": 10, "loss_g": 1, "loss_f": 10, "loss_s_intra": 0.1, "loss_s_inter": 0.1}  # main/config.py defaults
BASE = dict(seed=1, n_queries=37, lv=(6, 75), lt=(3, 32), eval_bsz=8, eval_mode=None, round_multiple=1, clip_length=2.0,
            nms_thd=-1, max_before_nms=10, max_after_nms=10, no_sort_results=False, debug=False, eval_split_name="val",
            criterion=True, epoch_i=3, tb=True)
CASES = [
    dict(name="default"),
    dict(name="add_norm_nms", seed=2, eval_mode="add", round_multiple=-1, nms_thd=0.7),
    dict(name="add_mr_nms_20_5", seed=3, eval_mode="add_mr", nms_thd=0.7, max_before_nms=20, max_after_nms=5),
    dict(name="none_norm", seed=3, eval_mode=None, round_multiple=-1, nms_thd=0.7, max_before_nms=20, max_after_nms=5),
    dict(name="clip1_nms", seed=4, clip_length=1.0, nms_thd=0.7),
    dict(name="clip1.5_add", seed=5, clip_length=1.5, eval_mode="add", eval_bsz=5, n_queries=23),
    dict(name="clip0.2_nms", seed=6, clip_length=0.2, nms_thd=0.7, eval_mode="add"),
    dict(name="unsorted_nms", seed=7, no_sort_results=True, nms_thd=0.7),
    dict(name="unsorted_nms_20_5", seed=8, no_sort_results=True, nms_thd=0.7, max_before_nms=20, max_after_nms=5, clip_length=1.5),
    dict(name="debug_add", seed=9, debug=True, eval_mode="add", nms_thd=0.7),
    dict(name="test_split_nms", seed=10, eval_split_name="test", nms_thd=0.7),
    dict(name="test_split", seed=11, eval_split_name="test"),
    dict(name="other_split_nms", seed=12, eval_split_name="test_public", nms_thd=0.7, criterion=False),
    dict(name="no_tb_bsz32", seed=13, n_queries=70, eval_bsz=32, tb=False, round_multiple=-1, nms_thd=0.5),
    dict(name="no_epoch", seed=14, epoch_i=None, eval_mode="add", nms_thd=0.7),
]


def case_params(c):
    p = dict(BASE)
    p.update(c)
    return p


def case_opt(p, results_dir, device):
    return synth.eval_epoch_opt(eval_bsz=p["eval_bsz"], eval_mode=p["eval_mode"], round_multiple=p["round_multiple"],
                                clip_length=p["clip_length"], nms_thd=p["nms_thd"], max_before_nms=p["max_before_nms"],
                                max_after_nms=p["max_after_nms"], no_sort_results=p["no_sort_results"], debug=p["debug"],
                                eval_split_name=p["eval_split_name"], results_dir=results_dir, device=device)


def case_dataset(p):
    return synth.EvalEpochDataset(p["seed"], n_queries=p["n_queries"], lv=tuple(p["lv"]), lt=tuple(p["lt"]))


def submission_name(p):
    return "inference_fake_{}_{}_preds.jsonl".format(p["eval_split_name"], p["name"])


class TbRecorder:
    def __init__(self):
        self.calls = []

    def add_scalar(self, tag, value, step):
        self.calls.append([tag, value, step])


def read_results(results_dir):
    """{file name: [sha256 of its bytes, size]} of every file in results_dir."""
    out = {}
    for name in sorted(os.listdir(results_dir)):
        with open(os.path.join(results_dir, name), "rb") as f:
            data = f.read()
        out[name] = [hashlib.sha256(data).hexdigest(), len(data)]
    return out


def stub_reference_deps():
    sys.modules.setdefault("h5py", types.ModuleType("h5py"))
    if "nncore" not in sys.modules:
        nn_ = types.ModuleType("nncore")
        ds = types.ModuleType("nncore.dataset")

        class _Registry:
            def register(self, *a, **k):
                return lambda c: c

        ds.DATASETS = _Registry()
        par = types.ModuleType("nncore.parallel")
        par.DataContainer = object
        nn_.dataset, nn_.parallel = ds, par
        sys.modules.update({"nncore": nn_, "nncore.dataset": ds, "nncore.parallel": par})


def main():
    sys.path.insert(0, os.path.abspath(sys.argv[1]))
    stub_reference_deps()
    import torch

    torch.Tensor.cuda = lambda self, *a, **k: self  # every tensor stays on the CPU
    import main.inference_mr as M
    from model.univtg import SetCriterion

    class Recording(torch.nn.Module):
        def __init__(self, crit):
            super().__init__()
            self.crit, self.weight_dict, self.batches = crit, crit.weight_dict, []

        def forward(self, outputs, targets):
            out = self.crit(outputs, targets)
            self.batches.append({k: float(v) for k, v in out.items()})
            return out

    cases = []
    for c in CASES:
        p = case_params(c)
        ds = case_dataset(p)
        model = synth.ReplayEvalModel(p["seed"])
        crit = None
        if p["criterion"]:
            crit = Recording(SetCriterion(matcher=None, weight_dict=dict(WEIGHTS), eos_coef=0.1, losses=["spans", "labels", "saliency"],
                                          temperature=0.07, span_loss_type="l1", max_v_l=75))
        tb = TbRecorder() if p["tb"] else None
        with tempfile.TemporaryDirectory() as tmp:
            opt = case_opt(p, tmp, "cpu")
            metrics, metrics_nms, meters, paths = M.eval_epoch(model, ds, opt, submission_name(p), epoch_i=p["epoch_i"], criterion=crit,
                                                               tb_writer=tb)
            files = read_results(tmp)
            rel = [os.path.relpath(x, tmp) for x in paths]
        cases.append({
            "params": p, "files": files, "paths": rel,
            "metrics": None if metrics is None else json.dumps(metrics), "metrics_nms": None if metrics_nms is None else json.dumps(metrics_nms),
            "meters": {k: {f: getattr(m, f) for f in ("val", "avg", "sum", "count", "max", "min")} for k, m in meters.items()},
            "tb": tb.calls if tb else None, "batch_losses": crit.batches if crit else None, "weight_dict": WEIGHTS,
        })
        print(p["name"], "files:", sorted(files), "batches:", len(crit.batches) if crit else 0)
    out = {"torch": torch.__version__, "cases": cases}
    path = os.path.join(HERE, "reference_eval_epoch.json")
    with open(path, "w") as f:
        json.dump(out, f)
    print("wrote", path, len(cases), "cases")


if __name__ == "__main__":
    main()
