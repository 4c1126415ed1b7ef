#!/usr/bin/env python
"""Writes tests/golden/reference_task_eval.json: the live reference's DatasetHL.evaluate (main/dataset.py) and
calculate_semantic_matching (eval/qfvs.py) on the seeded cases of univtg_b200.synth, so the task-evaluation oracle
(oracle/task_eval_oracle.py) stays pinned without the reference, networkx or scikit-learn.  The inputs are not stored: each
case keeps its seed and parameters and a sha256 of its inputs (tests regenerate them and check the hash).

  * highlight cases: DatasetHL is built with __new__ (nncore and h5py stubbed) and given dset_name, domain, state, video_id and
    label; its evaluate() gives the {'mAP'} dict of the whole blob, and with main.dataset's `round` shadowed by the identity,
    the unrounded value of every one-video blob (TVSum: the mean of the 20 annotator APs in the reference's order; YouTube:
    the video's AP).  The sha256 of the jsonl file evaluate(save_dir=...) writes is kept too.
  * QFVS cases: calculate_semantic_matching's (p, r, f1) as floats (f1 may be NaN, stored as null).

Usage: python tests/golden/make_golden_task_eval.py <path to a showlab/UniVTG checkout>"""
import hashlib
import json
import math
import os
import sys
import tempfile
import types
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from univtg_b200 import synth  # noqa: E402

HL_CASES = [
    dict(seed=1, dset_name="tvsum"),
    dict(seed=2, dset_name="tvsum", n_videos=10, clips=(200, 96, 33, 150), tie_frac=0.8),
    dict(seed=3, dset_name="tvsum", n_videos=4, clips=(4, 2, 5, 1), shorter=0.5),
    dict(seed=4, dset_name="tvsum", n_videos=3, clips=(700, 400, 1000), k=20),
    dict(seed=5, dset_name="tvsum", n_videos=5, k=0),
    dict(seed=6, dset_name="tvsum", n_videos=5, k=-3),
    dict(seed=7, dset_name="youtube"),
    dict(seed=8, dset_name="youtube", n_videos=12, clips=(60, 18, 250, 33, 90), tie_frac=0.9),
    dict(seed=9, dset_name="youtube", n_videos=4, clips=(1, 2, 16, 17), shorter=0.5),
]
QFVS_CASES = [  # the four Tags.mat videos' shot counts with their summary sizes, then smaller and edge cases
    dict(seed=11, n_shots=2152, n_machine=43, n_gt=43),
    dict(seed=12, n_shots=3692, n_machine=73, n_gt=73),
    dict(seed=13, n_shots=3588, n_machine=71, n_gt=71),
    dict(seed=14, n_shots=2783, n_machine=55, n_gt=55),
    dict(seed=15, n_shots=400, n_machine=30, n_gt=12),
    dict(seed=16, n_shots=400, n_machine=9, n_gt=25, zero_frac=0.3),
    dict(seed=17, n_shots=50, n_machine=1, n_gt=1),
    dict(seed=18, n_shots=120, n_machine=20, n_gt=20, zero_frac=1.0),  # every weight 0
]


def hl_inputs(params):
    params = dict(params)
    k = params.pop("k", 5)
    return synth.make_hl_eval_case(**params), k


def hl_hash(case, k):
    ds = case["dataset"]
    h = hashlib.sha256(json.dumps([ds.dset_name, ds.domain, ds.video_id["val"], ds.label, k], sort_keys=True).encode())
    for t in case["blob"]:
        h.update(str(list(t.shape)).encode())
        h.update(t.numpy().tobytes())
    return h.hexdigest()


def qfvs_hash(case):
    h = hashlib.sha256(np.ascontiguousarray(case["tags"]).tobytes())
    h.update(json.dumps([case["machine"], case["gt"]]).encode())
    return h.hexdigest()


def stub_dataset_deps():
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


def reference_dataset(D, case):
    fake = case["dataset"]
    ds = D.DatasetHL.__new__(D.DatasetHL)
    ds.dset_name, ds.domain, ds.state = fake.dset_name, fake.domain, "val"
    ds.video_id = {"train": [], "val": list(fake.video_id["val"])}
    ds.label = fake.label
    return ds


def main():
    sys.path.insert(0, os.path.abspath(sys.argv[1]))
    stub_dataset_deps()
    import networkx
    import sklearn
    import torch

    import main.dataset as D
    from eval.qfvs import calculate_semantic_matching

    hl = []
    for params in HL_CASES:
        case, k = hl_inputs(params)
        ds = reference_dataset(D, case)
        res = ds.evaluate(case["blob"], k=k)
        with tempfile.TemporaryDirectory() as tmp:
            os.makedirs(os.path.join(tmp, ds.dset_name))
            ds.evaluate(case["blob"], k=k, save_dir=tmp)
            with open(os.path.join(tmp, ds.dset_name, ds.domain + ".jsonl"), "rb") as f:
                jsonl = hashlib.sha256(f.read()).hexdigest()
        per_video = []
        D.round = lambda x, n=None: x  # the unrounded mean of one-video blobs
        try:
            for idx, score in enumerate(case["blob"]):
                one = reference_dataset(D, case)
                one.video_id["val"] = [one.video_id["val"][idx]]
                per_video.append(one.evaluate([score], k=k)["mAP"])
        finally:
            del D.round
        hl.append({"params": params, "sha256": hl_hash(case, k), "result": res, "per_video": per_video, "jsonl_sha256": jsonl})

    qfvs = []
    for params in QFVS_CASES:
        case = synth.make_qfvs_match_case(**params)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)  # 0/0 of the all-zero case, as in the reference
            p, r, f1 = calculate_semantic_matching(list(case["machine"]), list(case["gt"]), [case["tags"]], 0)
        qfvs.append({"params": params, "sha256": qfvs_hash(case),
                     "prf": [None if math.isnan(float(x)) else float(x) for x in (p, r, f1)],
                     "types": [type(x).__name__ for x in (p, r, f1)]})

    out = {"torch": torch.__version__, "networkx": networkx.__version__, "scikit-learn": sklearn.__version__, "numpy": np.__version__,
           "hl": hl, "qfvs": qfvs}
    path = os.path.join(HERE, "reference_task_eval.json")
    with open(path, "w") as f:
        json.dump(out, f)
    print("wrote", path, len(hl), "highlight cases,", len(qfvs), "QFVS cases")


if __name__ == "__main__":
    main()
