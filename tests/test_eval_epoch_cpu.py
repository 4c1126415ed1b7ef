"""The evaluation-epoch restatement (tests/eval_epoch_oracle.py) against the live reference's eval_epoch
(tests/golden/reference_eval_epoch.json, tests/golden/make_golden_eval_epoch.py): files byte for byte, returned metrics, paths,
loss meters and TensorBoard scalars exactly.  No GPU."""
import json
import os

import pytest

from tests import eval_epoch_oracle as O
from tests.golden import make_golden_eval_epoch as G
from univtg_b200 import synth

CASES = O.golden_cases()


def test_golden_covers_the_options():
    ps = [c["params"] for c in CASES]
    assert {p["eval_mode"] for p in ps} == {None, "add", "add_mr"}
    assert {p["round_multiple"] for p in ps} == {1, -1}
    assert {p["clip_length"] for p in ps} == {2.0, 1.0, 1.5, 0.2}
    assert {p["nms_thd"] for p in ps} >= {-1, 0.7}
    assert {(p["max_before_nms"], p["max_after_nms"]) for p in ps} == {(10, 10), (20, 5)}
    assert {p["eval_split_name"] for p in ps} == {"val", "test", "test_public"}
    assert any(p["no_sort_results"] for p in ps) and any(p["debug"] for p in ps)
    assert any(p["n_queries"] % p["eval_bsz"] for p in ps)


def test_add_mr_equals_no_eval_mode():
    """eval_mode "add_mr" rebinds prob after the scores were taken: the reference's files equal those of eval_mode None."""
    by = {c["params"]["name"]: c for c in CASES}
    a, b = by["add_mr_nms_20_5"], by["none_norm"]
    assert a["params"]["seed"] == b["params"]["seed"]
    # none_norm skips round_multiple, so only the highlight lists may be compared through the metrics' HL keys
    ma, mb = json.loads(a["metrics"]), json.loads(b["metrics"])
    assert {k: v for k, v in ma.items() if k.startswith("HL")} == {k: v for k, v in mb.items() if k.startswith("HL")}


@pytest.mark.parametrize("case", CASES, ids=[c["params"]["name"] for c in CASES])
def test_oracle_epoch_matches_reference(case, tmp_path):
    p = case["params"]
    ds = G.case_dataset(p)
    model = synth.ReplayEvalModel(p["seed"])
    crit = O.ReplayCriterion(case["batch_losses"], case["weight_dict"]) if p["criterion"] else None
    tb = G.TbRecorder() if p["tb"] else None
    opt = G.case_opt(p, str(tmp_path), "cpu")
    metrics, metrics_nms, meters, paths = O.eval_epoch(model, ds, opt, G.submission_name(p), epoch_i=p["epoch_i"], criterion=crit,
                                                       tb_writer=tb)
    assert O.file_digests(str(tmp_path)) == case["files"]
    assert [os.path.relpath(x, str(tmp_path)) for x in paths] == case["paths"]
    assert (None if metrics is None else json.dumps(metrics)) == case["metrics"]
    assert (None if metrics_nms is None else json.dumps(metrics_nms)) == case["metrics_nms"]
    assert O.meter_fields(meters) == case["meters"]
    assert (tb.calls if tb else None) == case["tb"]
    if crit is not None:
        assert crit.calls == len(case["batch_losses"])
