"""Time one moment-retrieval evaluation epoch of QVHighlights-val size on one GPU, in one call.

    python tools/eval_epoch_cost.py [--epochs 3] [--json tools/records/eval_epoch_cost_h100.json]

Epoch: 1550 queries, Lv 75, Lt 8-32, eval_bsz 32, nms_thd 0.7, clip_length 2, the device criterion, a TensorBoard stand-in, in two
configurations - "add" (eval_mode add, round_multiple -1: the QVHL scripts) and "round_multiple" (eval_mode None,
round_multiple 1: the pretrain / cotrain scripts).  Two arrangements are timed:
  (a) device: univtg_b200.evaluation.eval_epoch;
  (b) pieces: the reference's loop with today's pieces - per batch postproc.compose_submission (nms_thd -1) and the criterion with
      float(v) on every loss, then the host post-processing of the reference (round_multiple with a torch.tensor per line, list
      NMS), save_jsonl / save_json and univtg_b200.metrics.eval_submission for both submissions.
Each runs with replayed outputs (device-resident, no forward) and with the cfg2-sized model forward (univtg_b200 Model, seeded
weights).  Reported: the median wall time of --epochs epochs after one warm-up epoch (host clock; each epoch ends with its
files written, which follows a device synchronise), and whether (a) and (b) wrote the same before-NMS submission file.  The
GPU's name and power limit are read in the same call.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time
from collections import defaultdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from clip_cost import gpu_info  # noqa: E402
from tests import eval_epoch_oracle as O  # noqa: E402
from univtg_b200 import build_model, evaluation, metrics, postproc, synth  # noqa: E402
from univtg_b200.criterion import SetCriterion  # noqa: E402

N_QUERIES, LV, EVAL_BSZ = 1550, 75, 32
WEIGHTS = {"loss_b": 10, "loss_g": 1, "loss_f": 10, "loss_s_intra": 0.1, "loss_s_inter": 0.1}
CONFIGS = {"add": dict(eval_mode="add", round_multiple=-1), "round_multiple": dict(eval_mode=None, round_multiple=1)}


class QvhlDataset(synth.EvalEpochDataset):
    """EvalEpochDataset at QVHL-val size: every video 75 clips; cfg2 feature widths, drawn from a pool of 64 seeded tensors."""

    def __init__(self, dv, dt):
        super().__init__(5, n_queries=N_QUERIES, lv=(LV, LV), lt=(8, 32), dv=1, dt=1)
        g = torch.Generator().manual_seed(6)
        vid = [torch.randn(LV, dv, generator=g) for _ in range(64)]
        txt = [torch.randn(32, dt, generator=g) for _ in range(64)]
        for i, it in enumerate(self.items):
            mi = it["model_inputs"]
            mi["video_feat"] = vid[i % 64]
            mi["query_feat"] = txt[i % 64][:mi["query_feat"].shape[0]]


class Replay(torch.nn.Module):
    """Device-resident outputs of synth.ReplayEvalModel, one set per batch shape, returned without copies."""

    def __init__(self, d):
        super().__init__()
        self.gen = synth.ReplayEvalModel(5, d=d).cuda()
        self.cache = {}
        self.register_buffer("anchor", torch.zeros(1, device="cuda"))

    def forward(self, src_txt, src_txt_mask, src_vid, src_vid_mask):
        key = tuple(src_vid.shape[:2])
        if key not in self.cache:
            self.cache[key] = self.gen(src_txt, src_txt_mask, src_vid, src_vid_mask)
        out = dict(self.cache[key])
        out["src_vid_mask"] = src_vid_mask
        return out


def pieces_epoch(model, ds, opt, name, crit, tb):
    """(b): the reference's eval_epoch with today's per-batch pieces."""
    loader = torch.utils.data.DataLoader(ds, collate_fn=O.start_end_collate_mr, batch_size=opt.eval_bsz, num_workers=opt.num_workers,
                                         shuffle=False, pin_memory=opt.pin_memory)
    mr_res, meters = [], defaultdict(O.AverageMeter)
    with torch.no_grad():
        for batch in loader:
            mi, tg = O.prepare_batch_inputs_mr(batch[1], opt.device, non_blocking=opt.pin_memory)
            out = model(**mi)
            mr_res += postproc.compose_submission(batch[0], out, tg, mi)
            loss_dict = dict(crit(out, tg))
            loss_dict["loss_overall"] = float(sum(loss_dict[k] * WEIGHTS[k] for k in loss_dict if k in WEIGHTS))
            for k, v in loss_dict.items():
                meters[k].update(float(v) * WEIGHTS[k] if k in WEIGHTS else float(v))
    for k, v in meters.items():
        tb.add_scalar(f"Eval/{k}", v.avg, 1)
    if opt.round_multiple > 0:
        for e in mr_res:
            e["pred_relevant_windows"] = O.round_multiple(e["pred_relevant_windows"], opt.clip_length)
    path = os.path.join(opt.results_dir, name)
    O.save_jsonl(mr_res, path)
    m = metrics.eval_submission(mr_res, ds.data)
    O.save_json(m, path.replace(".jsonl", "_metrics.json"))
    after = []
    for e in mr_res:
        e = dict(e)
        e["pred_relevant_windows"] = O.reference_temporal_nms(e["pred_relevant_windows"][:opt.max_before_nms], opt.nms_thd,
                                                              opt.max_after_nms)
        after.append(e)
    p2 = path.replace(".jsonl", "_nms_thd_{}.jsonl".format(opt.nms_thd))
    O.save_jsonl(after, p2)
    O.save_json(metrics.eval_submission(after, ds.data), p2.replace(".jsonl", "_metrics.json"))


def device_epoch(model, ds, opt, name, crit, tb):
    evaluation.eval_epoch(model, ds, opt, name, epoch_i=0, criterion=crit, tb_writer=tb, collate_fn=O.start_end_collate_mr,
                          prepare_batch=O.prepare_batch_inputs_mr)


def time_epochs(fn, epochs):
    fn()
    times = []
    for _ in range(epochs):
        torch.cuda.synchronize()
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t) * 1e3)
    return {"median_ms": statistics.median(times), "min_max_ms": [min(times), max(times)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_epoch_cost: no CUDA device")
    info = gpu_info()
    cfg = synth.CONFIGS["cfg2"]
    ds = QvhlDataset(cfg["v_feat_dim"], cfg["t_feat_dim"])
    real, _ = build_model(synth.reference_args(cfg, device="cuda:0"))
    real.load_state_dict(synth.make_state_dict(cfg, seed=0), strict=True)
    real = real.to("cuda:0").eval()
    models = {"replay": Replay(cfg["hidden_dim"]), "cfg2_forward": real}
    crit = SetCriterion(dict(WEIGHTS), 0.1, ["spans", "labels", "saliency"], 0.07, "l1", 75)
    res = {"gpu": info, "queries": N_QUERIES, "lv": LV, "eval_bsz": EVAL_BSZ, "nms_thd": 0.7, "clip_length": 2.0, "cases": {}}
    for mname, model in models.items():
        for cname, over in CONFIGS.items():
            row = {}
            with tempfile.TemporaryDirectory() as ta, tempfile.TemporaryDirectory() as tb_:
                for label, fn, d in (("device", device_epoch, ta), ("pieces", pieces_epoch, tb_)):
                    opt = synth.eval_epoch_opt(eval_bsz=EVAL_BSZ, nms_thd=0.7, clip_length=2.0, results_dir=d, pin_memory=True, **over)
                    rec = type("Tb", (), {"add_scalar": lambda self, *a: None})()
                    row[label] = time_epochs(lambda: fn(model, ds, opt, "preds.jsonl", crit, rec), args.epochs)
                if cname == "round_multiple":  # (b) has no eval_mode "add"; with None both write the same file
                    with open(os.path.join(ta, "preds.jsonl")) as fa, open(os.path.join(tb_, "preds.jsonl")) as fb:
                        row["same_submission_file"] = fa.read() == fb.read()
            row["speedup"] = row["pieces"]["median_ms"] / row["device"]["median_ms"]
            res["cases"][f"{mname}/{cname}"] = row
            print(mname, cname, json.dumps(row), flush=True)
    print(json.dumps(res))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
