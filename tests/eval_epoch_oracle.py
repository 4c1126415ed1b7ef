"""TEST INFRASTRUCTURE ONLY - CPU restatement of the reference's moment-retrieval evaluation epoch.

Only tests/ and tools/ may import this module; the product path (univtg_b200/evaluation.py) never does.  It builds on the decode
and NMS restatements of oracle/postproc_oracle.py and the metrics of oracle/metrics_oracle.py.  Follows, in behaviour:
  * main/inference_mr.py:112-136  highlight values by eval_mode: fp16 saliency, or ("add") fp32(fp16 saliency) + prob
  * eval/postprocessing.py:26-51  PostProcessorDETR(process_func_names=["round_multiple"]) as compute_mr_results applies it (:184-192)
  * main/inference_mr.py:43-84,101-222  eval_epoch: loader, loop, loss meters, TensorBoard scalars, files, metrics, NMS
  * main/dataset.py:1037-1052,1071-1100, utils/tensor_utils.py:5-53  start_end_collate_mr / prepare_batch_inputs_mr (stand-ins)
  * utils/basic_utils.py:34-50,133-160  save_json(save_pretty=True) / save_jsonl, AverageMeter
Pinning: tests/golden/reference_eval_epoch.json holds what the live reference eval_epoch wrote and returned on the seeded cases of
tests/golden/make_golden_eval_epoch.py; tests/test_eval_epoch_cpu.py checks this restatement against it byte for byte.
"""
import json
import os
from collections import defaultdict

import torch

from oracle.postproc_oracle import decode_mr, temporal_nms


def highlight_lists(saliency_scores, pred_logits, timestamp_mask, src_vid_mask, eval_mode=None):
    """main/inference_mr.py:112-136: `prob` is pred_logits with scores[~mask] = 0 applied in place (scores is a view of prob); with
    eval_mode "add" the highlight values are saliency.half() + prob.squeeze(-1) (fp32), otherwise saliency.half().  "add_mr"
    rebinds prob after scores was taken and so changes nothing here."""
    prob = pred_logits.detach().to("cpu", torch.float32).clone()
    scores = prob[..., 0]
    scores[~timestamp_mask.detach().to("cpu").bool()] = 0
    sal = saliency_scores.detach().to("cpu", torch.float32)
    hl = sal.half() + prob.squeeze(-1) if eval_mode == "add" else sal.half()
    lens = src_vid_mask.detach().to("cpu").sum(1).tolist()
    return [hl[j, :int(lens[j])].tolist() for j in range(len(lens))]


def round_multiple(rows, clip_length):
    """PostProcessorDETR.__call__ with round_to_multiple_clip_lengths on one query's rows (eval/postprocessing.py:26-51)."""
    ws = torch.tensor(rows)
    windows = torch.round(ws[:, :2] / clip_length) * clip_length
    out = torch.cat([windows, ws[:, 2:3]], dim=1).tolist()
    return [e[:2] + [float(f"{e[2]:.4f}")] for e in out]


def reference_temporal_nms(predictions, nms_thd, max_after_nms=100):
    """utils/temporal_nms.py: temporal_nms, including its pass-through of a single row."""
    if len(predictions) == 1:
        return predictions
    return temporal_nms(predictions, nms_thd, max_after_nms)


# ---- stand-ins for the reference's collate / batch preparation ---------------------------------------------------------------
def pad_sequences_1d(sequences, dtype=torch.float32):
    if isinstance(sequences[0], list):
        sequences = [torch.tensor(s, dtype=dtype) for s in sequences]
    lengths = [len(s) for s in sequences]
    padded = torch.zeros((len(sequences), max(lengths)) + tuple(sequences[0].shape[1:]), dtype=dtype)
    mask = torch.zeros((len(sequences), max(lengths)), dtype=torch.float32)
    for i, s in enumerate(sequences):
        padded[i, :lengths[i]] = s
        mask[i, :lengths[i]] = 1
    return padded, mask


def start_end_collate_mr(batch):
    meta = [e["meta"] for e in batch]
    data = {}
    for k in batch[0]["model_inputs"].keys():
        if k == "span_labels":
            data[k] = [dict(spans=e["model_inputs"]["span_labels"]) for e in batch]
        elif k in ("saliency_pos_labels", "saliency_neg_labels"):
            data[k] = torch.LongTensor([e["model_inputs"][k] for e in batch])
        else:
            data[k] = pad_sequences_1d([e["model_inputs"][k] for e in batch], dtype=torch.float32)
    return meta, data


def prepare_batch_inputs_mr(b, device, non_blocking=False):
    to = lambda t: t.to(device, non_blocking=non_blocking)  # noqa: E731
    model_inputs = dict(src_txt=to(b["query_feat"][0]), src_txt_mask=to(b["query_feat"][1]), src_vid=to(b["video_feat"][0]),
                        src_vid_mask=to(b["video_feat"][1]))
    targets = {"timestamp": to(b["timestamp"][0]), "timestamp_mask": to(b["timestamp"][1]),
               "timestamp_window": to(b["timestamp_window"][0]), "span_labels_nn": to(b["span_labels_nn"][0])}
    if "saliency_scores" in b:
        targets["saliency_scores"] = to(b["saliency_scores"][0])
    if "span_labels" in b:
        targets["span_labels"] = [dict(spans=to(e["spans"])) for e in b["span_labels"]]
    for name in ("saliency_pos_labels", "saliency_neg_labels"):
        if name in b:
            targets[name] = to(b[name])
    return model_inputs, targets


# ---- the epoch --------------------------------------------------------------------------------------------------------------
class AverageMeter:
    """utils/basic_utils.py:133-160."""

    def __init__(self):
        self.val, self.avg, self.sum, self.count, self.max, self.min = 0, 0, 0, 0, -1e10, 1e10

    def update(self, val, n=1):
        self.max = max(val, self.max)
        self.min = min(val, self.min)
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def loss_meters(batch_losses, weight_dict):
    """compute_mr_results' criterion block (main/inference_mr.py:167-173) on per-batch loss dicts ({name: 0-dim fp32 tensor}):
    loss_overall is the sequential fp32 sum of loss * weight, the meters take float(v) * weight in Python floats."""
    meters = defaultdict(AverageMeter)
    for loss_dict in batch_losses:
        loss_dict = dict(loss_dict)
        losses = sum(loss_dict[k] * weight_dict[k] for k in loss_dict.keys() if k in weight_dict)
        loss_dict["loss_overall"] = float(losses)
        for k, v in loss_dict.items():
            meters[k].update(float(v) * weight_dict[k] if k in weight_dict else float(v))
    return meters


def meter_fields(meters):
    return {k: {f: getattr(m, f) for f in ("val", "avg", "sum", "count", "max", "min")} for k, m in meters.items()}


def save_jsonl(data, filename):
    with open(filename, "w") as f:
        f.write("\n".join([json.dumps(e) for e in data]))


def save_json(data, filename):
    with open(filename, "w") as f:
        f.write(json.dumps(data, indent=4, sort_keys=False))


def eval_epoch(model, eval_dataset, opt, save_submission_filename, epoch_i=None, criterion=None, tb_writer=None, *,
               collate_fn=start_end_collate_mr, prepare_batch=prepare_batch_inputs_mr, eval_submission=None):
    """main/inference_mr.py eval_epoch (:200-222) with compute_mr_results (:101-196) and eval_epoch_post_processing (:43-84), on
    the CPU.  `criterion` is called as the reference calls it; eval_submission defaults to oracle.metrics_oracle's."""
    from torch.utils.data import DataLoader

    if eval_submission is None:
        from oracle.metrics_oracle import eval_submission
    model.eval()
    if not (criterion is not None and eval_dataset.load_labels):
        criterion = None
    loader = DataLoader(eval_dataset, collate_fn=collate_fn, batch_size=opt.eval_bsz, num_workers=opt.num_workers, shuffle=False,
                        pin_memory=opt.pin_memory)
    write_tb = tb_writer is not None and epoch_i is not None
    mr_res, batch_losses = [], []
    with torch.no_grad():
        for batch in loader:
            query_meta = batch[0]
            model_inputs, targets = prepare_batch(batch[1], opt.device, non_blocking=opt.pin_memory)
            outputs = model(**model_inputs)
            windows = decode_mr(outputs["pred_logits"], outputs["pred_spans"], targets["timestamp"], targets["timestamp_mask"],
                                [m["duration"] for m in query_meta], sort=not opt.no_sort_results)
            hl = highlight_lists(outputs["saliency_scores"], outputs["pred_logits"], targets["timestamp_mask"],
                                 model_inputs["src_vid_mask"], opt.eval_mode)
            for meta, w, h in zip(query_meta, windows, hl):
                mr_res.append(dict(qid=meta["qid"], query=meta["query"], vid=meta["vid"], pred_relevant_windows=w,
                                   pred_saliency_scores=h))
            if criterion:
                batch_losses.append(criterion(outputs, targets))
            if opt.debug:
                break
    meters = loss_meters(batch_losses, criterion.weight_dict) if criterion else defaultdict(AverageMeter)
    if write_tb and criterion:
        for k, v in meters.items():
            tb_writer.add_scalar("Eval/{}".format(k), v.avg, epoch_i + 1)
    if opt.round_multiple > 0:
        for e in mr_res:
            e["pred_relevant_windows"] = round_multiple(e["pred_relevant_windows"], opt.clip_length)
    if opt.no_sort_results:
        save_submission_filename = save_submission_filename.replace(".jsonl", "_unsorted.jsonl")
    gt_data = eval_dataset.data
    submission_path = os.path.join(opt.results_dir, save_submission_filename)
    save_jsonl(mr_res, submission_path)
    if opt.eval_split_name in ["val", "test"]:
        metrics = eval_submission(mr_res, gt_data, verbose=opt.debug, match_number=not opt.debug)
        save_metrics_path = submission_path.replace(".jsonl", "_metrics.json")
        save_json(metrics, save_metrics_path)
        latest_file_paths = [submission_path, save_metrics_path]
    else:
        metrics = None
        latest_file_paths = [submission_path, ]
    metrics_nms = None
    if opt.nms_thd != -1:
        after = []
        for e in mr_res:
            e = dict(e)
            e["pred_relevant_windows"] = reference_temporal_nms(e["pred_relevant_windows"][:opt.max_before_nms], opt.nms_thd,
                                                                opt.max_after_nms)
            after.append(e)
        submission_nms_path = submission_path.replace(".jsonl", "_nms_thd_{}.jsonl".format(opt.nms_thd))
        save_jsonl(after, submission_nms_path)
        if opt.eval_split_name == "val":
            metrics_nms = eval_submission(after, gt_data, verbose=opt.debug, match_number=not opt.debug)
            save_metrics_nms_path = submission_nms_path.replace(".jsonl", "_metrics.json")
            save_json(metrics_nms, save_metrics_nms_path)
            latest_file_paths += [submission_nms_path, save_metrics_nms_path]
        else:
            latest_file_paths = [submission_nms_path, ]
    return metrics, metrics_nms, meters, latest_file_paths


# ---- the golden cases -------------------------------------------------------------------------------------------------------
def golden_cases():
    from tests.helpers import GOLDEN

    with open(os.path.join(GOLDEN, "reference_eval_epoch.json")) as f:
        return json.load(f)["cases"]


def file_digests(results_dir):
    """{file name: [sha256, size]} of every file in results_dir (the golden's form)."""
    from tests.golden.make_golden_eval_epoch import read_results

    return read_results(results_dir)


class ReplayCriterion(torch.nn.Module):
    """Returns the stored per-batch loss values (fp32, as the criterion produced them) in batch order."""

    def __init__(self, batch_losses, weight_dict, device="cpu"):
        super().__init__()
        self.batches, self.weight_dict, self.device, self.calls = batch_losses, weight_dict, device, 0

    def forward(self, outputs, targets):
        out = {k: torch.tensor(v, dtype=torch.float32, device=self.device) for k, v in self.batches[self.calls].items()}
        self.calls += 1
        return out
