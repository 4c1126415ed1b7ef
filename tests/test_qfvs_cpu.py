"""Query-focused video summarisation without a GPU: the synthetic batch restates the reference's input preparation, the fp64
oracle (oracle/qfvs_oracle.py) reproduces the reference's losses and gradients (tests/golden/reference_qfvs.npz, written by
tests/golden/make_golden_qfvs.py), and malformed criterion inputs are refused before anything is launched."""
import json
import os

import numpy as np
import pytest
import torch

from univtg_b200 import synth
from univtg_b200.qfvs import QFVSCriterion, build_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
Q = ("1", "2", "oracle")


@pytest.fixture(scope="module")
def golden():
    z = dict(np.load(os.path.join(ROOT, "tests", "golden", "reference_qfvs.npz")))
    meta = json.loads(bytes(z.pop("meta")).decode())
    return z, meta


def _batch(meta):
    cfg = synth.CONFIGS[meta["cfg"]]
    return cfg, synth.make_qfvs_batch(cfg, meta["seeds"][1], meta["S"], meta["Lf"], meta["seg_len"], meta["L1"], meta["L2"])


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_synthetic_batch_equals_the_reference_preparation(golden):
    z, meta = golden
    _, batch = _batch(meta)
    inputs, targets, mask_GT = batch[:3], batch[3:6], batch[6]
    for q, inp in zip(Q, inputs):
        assert torch.equal(inp["src_vid"], torch.from_numpy(z["in/src_vid"]))
        assert torch.equal(inp["src_vid_mask"], torch.from_numpy(z["in/src_vid_mask"]))
        assert torch.equal(inp["src_txt"], torch.from_numpy(z[f"in/{q}/src_txt"]))
        assert torch.equal(inp["src_txt_mask"], torch.from_numpy(z[f"in/{q}/src_txt_mask"]))
    for q, tg in zip(Q, targets):
        assert sorted(tg) == sorted(k.split("/")[2] for k in z if k.startswith(f"tgt/{q}/"))
        for k, v in tg.items():
            ref = torch.from_numpy(z[f"tgt/{q}/{k}"])
            assert v.dtype == ref.dtype and torch.equal(v, ref), (q, k)
    assert mask_GT.dtype == torch.bool and torch.equal(mask_GT, torch.from_numpy(z["mask_GT"]))


def _close(got, ref, tol=1e-6):
    got = float(got.detach()) if torch.is_tensor(got) else float(got)
    return abs(got - ref) <= tol * max(abs(ref), 1e-30) or (ref == 0.0 and got == 0.0)


def test_oracle_train_step_matches_the_reference(golden):
    from oracle import qfvs_oracle as QO
    from oracle import univtg_oracle as O

    z, meta = golden
    cfg, batch = _batch(meta)
    inputs, targets, mask_GT = batch[:3], batch[3:6], batch[6]
    sd = synth.make_state_dict(cfg, seed=meta["seeds"][0])
    leaves = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    dicts = [QO.criterion(O.forward(leaves, cfg, **inp), tg, mask_GT) for inp, tg in zip(inputs, targets)]
    for got, ref in zip(dicts, meta["step/losses"]):
        assert sorted(got) == sorted(ref)
        for k in ref:
            assert _close(got[k], ref[k]), (k, float(got[k]), ref[k])
    wd = synth.reference_args(cfg)
    wd = {"loss_f": wd.f_loss_coef, "loss_s_intra": wd.s_loss_intra_coef, "loss_s_inter": wd.s_loss_inter_coef}
    assert _close(O.weighted_total(QO.gather(dicts, 0), wd), meta["step/total_oracle_only"])
    total = O.weighted_total(QO.gather(dicts, 1), wd)
    assert _close(total, meta["step/total_gather"])
    total.backward()
    for k in meta["grads"]:
        assert _rel(leaves[k].grad, torch.from_numpy(z["grad/" + k]).double()) < 1e-5, k


def test_oracle_edge_cases_match_the_reference(golden):
    from oracle import qfvs_oracle as QO

    z, meta = golden
    _, batch = _batch(meta)
    base, mask_GT = batch[5], batch[6]
    assert meta["edge_cases"] == ["all_zero", "beyond_count", "no_pos_labels", "clamp"]
    for name in meta["edge_cases"]:
        tg = dict(base, saliency_scores=torch.from_numpy(z[f"edge/{name}/saliency_scores_target"]))
        if name == "no_pos_labels":
            del tg["saliency_pos_labels"]
        pl = torch.from_numpy(z[f"edge/{name}/pred_logits"]).double().requires_grad_(True)
        sal = torch.from_numpy(z["edge/saliency_scores"]).double().requires_grad_(True)
        got = QO.criterion({"pred_logits": pl, "saliency_scores": sal}, tg, mask_GT)
        ref = meta[f"edge/{name}/losses"]
        for k in ref:
            assert _close(got[k], ref[k]), (name, k, float(got[k]), ref[k])
        total = got["loss_f"] * 10.0 + got["loss_s_intra"] * 0.1
        if total.requires_grad:
            total.backward()
        for k, leaf in (("pred_logits", pl), ("saliency_scores", sal)):
            g = leaf.grad if leaf.grad is not None else torch.zeros_like(leaf)
            ref_g = torch.from_numpy(z[f"edge/{name}/grad_{k}"]).double()
            if float(ref_g.abs().max()) == 0.0:
                assert float(g.abs().max()) == 0.0, (name, k)
            else:
                assert _rel(g, ref_g) < 1e-5, (name, k, _rel(g, ref_g))
    assert all(v == 0.0 for v in meta["edge/all_zero/losses"].values())
    assert meta["edge/no_pos_labels/losses"]["loss_s_intra"] == 0.0


def test_build_model_reads_the_reference_args():
    cfg = synth.CONFIGS["tiny"]
    model, crit = build_model(synth.reference_args(cfg, dset_type="vs"))
    assert isinstance(crit, QFVSCriterion) and crit.losses == ["labels", "saliency"] and crit.temperature == 0.07
    assert sorted(model.state_dict()) == sorted(synth.state_dict_shapes(cfg))
    _, crit_mr = build_model(synth.reference_args(cfg, dset_type="mr"))
    assert "spans" in crit_mr.losses


def _cpu_case(S=3, Lf=8, d=16):
    outputs = {"pred_logits": torch.full((S, Lf, 1), 0.5), "pred_spans": torch.zeros(S, Lf, 2), "vid_mem_proj": torch.randn(S, Lf, d),
               "txt_mem_proj": torch.randn(S, 1, d), "src_vid_mask": torch.ones(S, Lf)}
    targets = {"saliency_scores": torch.zeros(1, S * Lf), "saliency_pos_labels": torch.zeros(1, 1)}
    return outputs, targets, torch.ones(1, S * Lf, dtype=torch.bool)


def test_qfvs_criterion_refuses_malformed_inputs_before_launching():
    cfg = synth.CONFIGS["tiny"]
    _, crit = build_model(synth.reference_args(cfg, dset_type="vs"))
    outputs, targets, mask = _cpu_case()
    with pytest.raises(ValueError, match="mask_GT"):
        crit(outputs, targets)
    with pytest.raises(ValueError, match="mask_GT"):
        crit(outputs, targets, mask[:, :-1])
    with pytest.raises(ValueError, match="saliency_scores"):
        crit(outputs, {**targets, "saliency_scores": torch.zeros(1, 23)}, mask)
    with pytest.raises(ValueError, match="saliency_scores"):
        crit(outputs, {**targets, "saliency_scores": torch.zeros(24)}, mask)
    _, crit_mr = build_model(synth.reference_args(cfg, dset_type="mr"))
    with pytest.raises(ValueError, match="spans"):
        crit_mr(outputs, targets, mask)
    with pytest.raises(RuntimeError, match="CUDA"):  # well-formed: only the device is wrong
        crit(outputs, {**targets, "saliency_scores": torch.zeros(1, 30)}, mask)


def test_mr_criterion_refuses_mis_shaped_targets_before_launching():
    from univtg_b200 import build_model as build_mr_model

    cfg = synth.CONFIGS["tiny"]
    _, crit = build_mr_model(synth.reference_args(cfg, dset_type="vlp"))
    inp = synth.make_inputs(cfg, seed=1, ragged=True, batch=3)
    tgt = synth.make_targets(inp, seed=2)
    B, Lv = inp["src_vid_mask"].shape
    outputs = {"pred_logits": torch.zeros(B, Lv, 1), "pred_spans": torch.zeros(B, Lv, 2), "vid_mem_proj": torch.zeros(B, Lv, 8),
               "txt_mem_proj": torch.zeros(B, 1, 8), "src_vid_mask": inp["src_vid_mask"]}
    bad = {"saliency_pos_labels": tgt["saliency_pos_labels"][:1], "timestamp_mask": tgt["timestamp_mask"][:, :-1],
           "timestamp_window": tgt["timestamp_window"].reshape(1, -1)}
    for k, v in bad.items():
        with pytest.raises(ValueError, match=k):
            crit(outputs, {**tgt, k: v})
    with pytest.raises(RuntimeError, match="CUDA"):  # valid targets get as far as the device check
        crit(outputs, tgt)
