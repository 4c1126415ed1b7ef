"""univtg_b200.evaluation.eval_epoch on the device against the live reference's eval_epoch (tests/golden/reference_eval_epoch.json)
and against the CPU restatement (tests/eval_epoch_oracle.py) fed with the same device outputs.

Files are compared byte for byte (sha256), metrics as json.dumps strings.  The loss meters come from the device criterion: they
must equal the restatement's meters computed from the device criterion's own per-batch fp32 values exactly, and each per-batch
loss must lie within the criterion kernels' error bound (tests/loss_ref.py mr_bounds, doubled: the reference's fp32 values carry
their own rounding error) of the reference's value."""
import json
import os

import pytest
import torch

from tests import eval_epoch_oracle as O
from tests import loss_ref as R
from tests.bounds import U, cfac
from tests.golden import make_golden_eval_epoch as G
from tests.helpers import load_golden
from univtg_b200 import build_model, evaluation, postproc, synth
from univtg_b200.criterion import SetCriterion

pytestmark = pytest.mark.gpu
CASES = O.golden_cases()


class RecordingCriterion(torch.nn.Module):
    """The device criterion; keeps every batch's loss dict and its inputs (CPU copies) for the checks below."""

    def __init__(self, weight_dict):
        super().__init__()
        self.crit = SetCriterion(dict(weight_dict), 0.1, ["spans", "labels", "saliency"], 0.07, "l1", 75)
        self.weight_dict = self.crit.weight_dict
        self.batches, self.cases = [], []

    def forward(self, outputs, targets):
        out = self.crit(outputs, targets)
        self.batches.append({k: v.detach().clone() for k, v in out.items()})
        cpu = lambda t: t.detach().float().cpu()  # noqa: E731
        self.cases.append({"pred_logits": cpu(outputs["pred_logits"][..., 0]), "pred_spans": cpu(outputs["pred_spans"]),
                           "vid_mem_proj": cpu(outputs["vid_mem_proj"]), "txt_mem_proj": cpu(outputs["txt_mem_proj"][:, 0]),
                           "timestamp": cpu(targets["timestamp"]), "timestamp_mask": cpu(targets["timestamp_mask"]),
                           "timestamp_window": cpu(targets["timestamp_window"]), "span_labels_nn": cpu(targets["span_labels_nn"]),
                           "saliency_scores": cpu(targets["saliency_scores"]),
                           "pos": targets["saliency_pos_labels"][:, 0].cpu(), "eos_coef": 0.1})
        return out


def _run_device(p, tmp, model, crit=None, tb=None, **opt_over):
    opt = G.case_opt(p, tmp, "cuda")
    for k, v in opt_over.items():
        setattr(opt, k, v)
    return evaluation.eval_epoch(model, G.case_dataset(p), opt, G.submission_name(p), epoch_i=p["epoch_i"], criterion=crit,
                                 tb_writer=tb, collate_fn=O.start_end_collate_mr, prepare_batch=O.prepare_batch_inputs_mr)


@pytest.mark.parametrize("case", CASES, ids=[c["params"]["name"] for c in CASES])
def test_device_epoch_matches_reference(case, tmp_path):
    p = case["params"]
    model = synth.ReplayEvalModel(p["seed"]).cuda()
    crit = RecordingCriterion(case["weight_dict"]) if p["criterion"] else None
    tb = G.TbRecorder() if p["tb"] else None
    metrics, metrics_nms, meters, paths = _run_device(p, str(tmp_path), model, crit, tb)
    assert O.file_digests(str(tmp_path)) == case["files"]
    assert [os.path.relpath(x, str(tmp_path)) for x in paths] == case["paths"]
    assert (None if metrics is None else json.dumps(metrics)) == case["metrics"]
    assert (None if metrics_nms is None else json.dumps(metrics_nms)) == case["metrics_nms"]
    if crit is None:
        assert dict(meters) == {} and (tb is None or tb.calls == [])
        return
    # exactly the reference's meter arithmetic on the device criterion's own fp32 values
    want = O.meter_fields(O.loss_meters([{k: v.cpu() for k, v in b.items()} for b in crit.batches], crit.weight_dict))
    assert O.meter_fields(meters) == want
    assert list(want) == list(case["meters"])
    if tb is not None and p["epoch_i"] is None:
        assert tb.calls == case["tb"] == []
    elif tb is not None:
        assert tb.calls == [[f"Eval/{k}", want[k]["avg"], p["epoch_i"] + 1] for k in want]
        assert [c[0] for c in tb.calls] == [c[0] for c in case["tb"]]
    # each batch's losses within the criterion's error bound of the reference's fp32 values
    assert len(crit.batches) == len(case["batch_losses"])
    for got, ref, c in zip(crit.batches, case["batch_losses"], crit.cases):
        lb, _ = R.mr_bounds(c, R.TRAIN_W)
        for k in R.LOSS_NAMES:
            S, K, E = lb[k]
            bound = 2 * (cfac(K) * U * float(S) + float(E))
            assert abs(float(got[k]) - ref[k]) <= bound, (p["name"], k, float(got[k]), ref[k], bound)


class DeviceReplay(torch.nn.Module):
    """Returns recorded outputs in call order (already on the right device)."""

    def __init__(self, outputs):
        super().__init__()
        self.outputs, self.calls = outputs, 0
        self.register_buffer("anchor", torch.zeros(1))

    def forward(self, **inputs):
        out = self.outputs[self.calls]
        self.calls += 1
        return out


class Recording(torch.nn.Module):
    def __init__(self, model):
        super().__init__()
        self.model, self.outputs = model, []

    def forward(self, **inputs):
        out = self.model(**inputs)
        self.outputs.append({k: v.detach().cpu().clone() for k, v in out.items()})
        return out


def _golden_dataset(name):
    """The golden batch as per-sample items (each cut to its own length, so the collate re-pads every batch) and ground truth."""
    cfg, sd, inp, tgt, _ = load_golden(name)
    ds = synth.EvalEpochDataset(0, n_queries=0)
    lv, lt = inp["src_vid_mask"].sum(1).long().tolist(), inp["src_txt_mask"].sum(1).long().tolist()
    for b in range(len(lv)):
        dur = 2.0 * lv[b] - 0.7
        mi = {"query_feat": inp["src_txt"][b, :lt[b]], "video_feat": inp["src_vid"][b, :lv[b]],
              "timestamp": tgt["timestamp"][b, :lv[b]], "timestamp_window": tgt["timestamp_window"][b, :lv[b]],
              "span_labels_nn": tgt["span_labels_nn"][b, :lv[b]], "saliency_scores": tgt["saliency_scores"][b, :lv[b]],
              "saliency_pos_labels": [int(tgt["saliency_pos_labels"][b, 0])], "saliency_neg_labels": [int(tgt["saliency_neg_labels"][b, 0])]}
        ds.items.append({"meta": {"qid": b, "query": f"q{b}", "vid": f"v{b}", "duration": dur}, "model_inputs": mi})
        ids = list(range(0, max(1, int(dur / 2) // 3)))
        ds.data.append({"qid": b, "query": f"q{b}", "vid": f"v{b}", "duration": dur, "relevant_windows": [[0, 2 * len(ids)]],
                        "relevant_clip_ids": ids, "saliency_scores": [[4, 2, 3]] * len(ids)})
    model, _ = build_model(synth.reference_args(cfg, device="cuda:0"))
    model.load_state_dict(sd, strict=True)
    return ds, model.to("cuda:0").eval()


@pytest.mark.parametrize("name", ["tiny_ragged", "cfg2_b4_ragged"])
def test_real_model_epoch_matches_oracle_on_device_outputs(name, tmp_path):
    ds, model = _golden_dataset(name)
    rec = Recording(model)
    d_dev, d_ref = tmp_path / "device", tmp_path / "oracle"
    d_dev.mkdir()
    d_ref.mkdir()
    opt = synth.eval_epoch_opt(eval_bsz=2, eval_mode="add", round_multiple=1, clip_length=2.0, nms_thd=0.7, results_dir=str(d_dev))
    got = evaluation.eval_epoch(rec, ds, opt, "preds.jsonl", collate_fn=O.start_end_collate_mr, prepare_batch=O.prepare_batch_inputs_mr)
    assert len(rec.outputs) == 2
    opt.results_dir, opt.device = str(d_ref), "cpu"
    ref = O.eval_epoch(DeviceReplay(rec.outputs), ds, opt, "preds.jsonl")
    assert O.file_digests(str(d_dev)) == O.file_digests(str(d_ref))
    assert json.dumps(got[0]) == json.dumps(ref[0]) and json.dumps(got[1]) == json.dumps(ref[1])
    with open(d_dev / "preds.jsonl") as f:
        sub = [json.loads(line) for line in f]
    assert len(sub) == len(ds) and all(len(e["pred_saliency_scores"]) == len(ds.items[i]["model_inputs"]["video_feat"])
                                       for i, e in enumerate(sub))


def test_no_host_sync_per_batch():
    """One batch's step (forward, decode into the pool, criterion) returns while an earlier ~50 ms sleep kernel still runs."""
    p = G.case_params({"name": "sync", "seed": 21})
    ds = G.case_dataset(p)
    opt = synth.eval_epoch_opt(pin_memory=True, eval_mode="add", round_multiple=1, nms_thd=0.7)
    loader = torch.utils.data.DataLoader(ds, collate_fn=O.start_end_collate_mr, batch_size=8, pin_memory=True)
    batches = list(loader)[:2]
    outs = []
    for b in batches:  # outputs resident on the device before the timed step: the model itself does no copies
        mi, _ = O.prepare_batch_inputs_mr(b[1], "cpu")
        with torch.no_grad():
            outs.append(synth.ReplayEvalModel(21).cuda()(**mi))
    torch.cuda.synchronize()
    model = DeviceReplay(outs).cuda()
    crit = SetCriterion({"loss_b": 10, "loss_g": 1, "loss_f": 10, "loss_s_intra": 0.1, "loss_s_inter": 0.1}, 0.1,
                        ["spans", "labels", "saliency"], 0.07, "l1", 75)
    state = evaluation.EpochState(torch.device("cuda", torch.cuda.current_device()), len(ds), opt)
    with torch.no_grad():
        evaluation.step(model, crit, state, batches[0], O.prepare_batch_inputs_mr, opt)  # warm-up: library load, pool allocation
        torch.cuda.synchronize()
        torch.cuda._sleep(100_000_000)  # ~50 ms at the H100's clocks
        ev = torch.cuda.Event()
        ev.record()
        evaluation.step(model, crit, state, batches[1], O.prepare_batch_inputs_mr, opt)
        pending = not ev.query()
    torch.cuda.synchronize()
    assert pending, "the step waited for the GPU"
    assert len(state.meta) == 16 and len(state.losses) == 2


@pytest.mark.parametrize("eval_mode,round_multiple,clip,thd,sort", [("add", 1, 2.0, 0.7, True), ("add_mr", 1, 1.5, -1, True),
                                                                    (None, 1, 0.2, 0.5, False), ("add", -1, 2.0, 0.7, True)])
def test_compose_submission_new_kwargs_match_oracle(eval_mode, round_multiple, clip, thd, sort):
    from oracle import postproc_oracle as P

    g = torch.Generator().manual_seed(33)
    B, Lv = 6, 75
    logits = torch.sigmoid(torch.randn(B, Lv, 1, generator=g))
    logits[:, ::5] = 0.5  # ties
    spans = torch.stack([-0.2 * torch.rand(B, Lv, generator=g), 0.2 * torch.rand(B, Lv, generator=g)], -1)
    lens = torch.randint(5, Lv + 1, (B,), generator=g)
    mask = (torch.arange(Lv)[None] < lens[:, None]).float()
    ts = ((torch.arange(Lv, dtype=torch.float32) + 0.5) / Lv)[None, :, None].expand(B, Lv, 2).contiguous()
    sal = torch.randn(B, Lv, generator=g)
    dur = [64.0, 150.0, 97.3, 40.0, 128.0, 33.33]
    meta = [{"qid": i, "query": f"q{i}", "vid": f"v{i}", "duration": dur[i]} for i in range(B)]
    outputs = {"pred_logits": logits.cuda(), "pred_spans": spans.cuda(), "saliency_scores": sal.cuda()}
    sub = postproc.compose_submission(meta, outputs, {"timestamp": ts.cuda(), "timestamp_mask": mask.cuda()},
                                      {"src_vid_mask": mask.cuda()}, nms_thd=thd, sort=sort, eval_mode=eval_mode,
                                      round_multiple=round_multiple, clip_length=clip)
    rows = P.decode_mr(logits, spans, ts, mask, dur, sort=sort)
    if round_multiple > 0:
        rows = [O.round_multiple(r, clip) for r in rows]
    if thd != -1:
        rows = [O.reference_temporal_nms(r[:10], thd, 10) for r in rows]
    hl = O.highlight_lists(sal, logits, mask, mask, eval_mode)
    assert [e["pred_relevant_windows"] for e in sub] == rows
    assert [e["pred_saliency_scores"] for e in sub] == hl


@pytest.mark.parametrize("what", ["moment_detr", "ce", "cpu", "two_class"])
def test_refusals_raise_before_launch(what, tmp_path):
    p = G.case_params({"name": "refuse", "n_queries": 9})
    model = synth.ReplayEvalModel(1, n_classes=2 if what == "two_class" else 1)
    if what != "cpu":
        model = model.cuda()
    over = {"moment_detr": {"model_id": "moment_detr"}, "ce": {"span_loss_type": "ce"}}.get(what, {})
    with pytest.raises((NotImplementedError, RuntimeError)):
        _run_device(p, str(tmp_path), model, **over)
    assert os.listdir(tmp_path) == []
    if what != "two_class":
        assert model.calls == 0
