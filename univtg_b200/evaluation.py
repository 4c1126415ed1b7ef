"""The moment-retrieval evaluation epoch of the reference (`eval_epoch`, main/inference_mr.py:43-222), on the device.

    from univtg_b200.evaluation import eval_epoch   # instead of: from main.inference_mr import eval_epoch

Same arguments, same files (byte for byte), same returned (metrics, metrics_nms, eval_loss_meters, latest_file_paths).  Every
batch is enqueued without a host synchronisation: the forward, one univtg_decode_mr_pool launch that writes the batch's sorted,
rounded rows (with round_multiple applied) and its highlight values (by eval_mode) into one epoch-wide row pool, and the
criterion, whose loss values stay on the device.  The durations reach the device through pinned staging.  At the end of the epoch
one univtg_temporal_nms_pool launch runs the NMS of every query, one device-to-host copy brings everything back, and the
reference's files and metrics (univtg_b200.metrics.eval_submission) are produced from it.

Options read from `opt`, as the reference reads them: eval_bsz, num_workers, pin_memory, device, span_loss_type, model_id,
eval_mode (None / "add" / "add_mr" / other), round_multiple, clip_length, no_sort_results, debug, results_dir, eval_split_name,
nms_thd, max_before_nms, max_after_nms.  CUDA only.
"""
import json
import os
from collections import defaultdict

import numpy as np
import torch

from . import _lib
from .metrics import eval_submission

METER_FIELDS = ("val", "avg", "sum", "count", "max", "min")


class AverageMeter:
    """utils/basic_utils.py AverageMeter: the fields the reference's loss meters carry."""

    def __init__(self):
        self.val, self.avg, self.sum, self.count, self.max, self.min = 0, 0, 0, 0, -1e10, 1e10

    def update(self, val, n=1):
        self.max = max(val, self.max)
        self.min = min(val, self.min)
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def _save_jsonl(data, filename):  # utils/basic_utils.py save_jsonl
    with open(filename, "w") as f:
        f.write("\n".join([json.dumps(e) for e in data]))


def _save_json_pretty(data, filename):  # utils/basic_utils.py save_json(save_pretty=True, sort_keys=False)
    with open(filename, "w") as f:
        f.write(json.dumps(data, indent=4, sort_keys=False))


def _model_device(model, opt):
    for t in model.parameters():
        return t.device
    for t in model.buffers():
        return t.device
    return torch.device(opt.device)


def check_options(model, opt):
    """The refusals of the device path, raised before anything launches."""
    if getattr(opt, "model_id", None) == "moment_detr":
        raise NotImplementedError("eval_epoch: moment_detr decoding (span_cxw_to_xx) is outside the univtg path")
    if opt.span_loss_type != "l1":
        raise NotImplementedError("eval_epoch: span_loss_type 'ce' is outside the univtg path")
    dev = _model_device(model, opt)
    if dev.type != "cuda":
        raise RuntimeError("univtg_b200: eval_epoch runs on CUDA only (no CPU path); move the model to a CUDA device")
    return dev


class RowPool:
    """The epoch's device buffers: rows [R, 3] f64 and highlight values [R] f32 (query q owns the Lv rows of its batch from row
    offsets[q]), valid lengths [Q] i32.  Grows by doubling (a device-to-device copy) when a batch does not fit."""

    def __init__(self, dev, rows, queries):
        self.dev = dev
        self.rows = torch.empty(max(rows, 1), 3, dtype=torch.float64, device=dev)
        self.hl = torch.empty(max(rows, 1), dtype=torch.float32, device=dev)
        self.lens = torch.empty(max(queries, 1), dtype=torch.int32, device=dev)

    def reserve(self, rows, queries):
        if rows > self.rows.shape[0]:
            n = max(rows, 2 * self.rows.shape[0])
            r, h = torch.empty(n, 3, dtype=torch.float64, device=self.dev), torch.empty(n, dtype=torch.float32, device=self.dev)
            r[:self.rows.shape[0]].copy_(self.rows)
            h[:self.hl.shape[0]].copy_(self.hl)
            self.rows, self.hl = r, h
        if queries > self.lens.shape[0]:
            ln = torch.empty(max(queries, 2 * self.lens.shape[0]), dtype=torch.int32, device=self.dev)
            ln[:self.lens.shape[0]].copy_(self.lens)
            self.lens = ln


def _f32(t, dev):
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def decode_into_pool(pool, outputs, targets, src_vid_mask, durations, row0, q0, sort, eval_mode, round_multiple, clip_length):
    """One univtg_decode_mr_pool launch for a batch; durations: [B] f32 on the device."""
    logits = outputs["pred_logits"]
    B, Lv = logits.shape[:2]
    dev = pool.dev
    lg = _f32(logits.reshape(B, Lv), dev)
    sp = _f32(outputs["pred_spans"], dev)
    ts = _f32(targets["timestamp"], dev)
    tm = _f32(targets["timestamp_mask"], dev)
    sal = _f32(outputs["saliency_scores"], dev)
    vm = _f32(src_vid_mask, dev)
    lib = _lib.load_library()
    rm = int(round_multiple) if round_multiple > 0 else 0
    _lib.check(lib.univtg_decode_mr_pool(_lib.ptr(lg), _lib.ptr(sp), _lib.ptr(ts), _lib.ptr(tm), _lib.ptr(durations), _lib.ptr(sal),
                                         _lib.ptr(vm), B, Lv, int(bool(sort)), int(eval_mode == "add"), rm, float(clip_length), row0,
                                         q0, _lib.ptr(pool.rows), _lib.ptr(pool.hl), _lib.ptr(pool.lens), _lib.stream_ptr()),
               "univtg_decode_mr_pool")


def nms_pool(rows, offsets_dev, n_queries, max_rows, nms_thd, max_before_nms, max_after_nms, sort):
    """One univtg_temporal_nms_pool launch -> (kept rows [Q, max_after_nms, 3] f64, counts [Q] i32) on the device."""
    dev = rows.device
    out = torch.zeros(max(n_queries, 1), max_after_nms, 3, dtype=torch.float64, device=dev)
    counts = torch.zeros(max(n_queries, 1), dtype=torch.int32, device=dev)
    lib = _lib.load_library()
    _lib.check(lib.univtg_temporal_nms_pool(_lib.ptr(rows), _lib.ptr(offsets_dev), n_queries, max_rows, int(max_before_nms),
                                            float(nms_thd), int(max_after_nms), int(bool(sort)), _lib.ptr(out), _lib.ptr(counts),
                                            _lib.stream_ptr()), "univtg_temporal_nms_pool")
    return out, counts


def pinned_to_device(values, dtype, dev):
    """Host numbers -> device tensor through a pinned staging buffer: the copy does not synchronise the stream."""
    host = torch.tensor(values, dtype=dtype).pin_memory()
    return host.to(dev, non_blocking=True)


class EpochState:
    """What one evaluation epoch accumulates on the device, and its single read-back."""

    def __init__(self, dev, n_queries_hint, opt):
        self.dev, self.opt = dev, opt
        self.pool = None
        self.n_queries_hint = n_queries_hint
        self.rows = 0
        self.meta, self.row_off, self.n_rows = [], [], []
        self.losses, self.loss_keys = [], None

    def add_batch(self, query_meta, model_inputs, targets, outputs):
        """Enqueue the decode of one batch (no host synchronisation)."""
        logits = outputs["pred_logits"]
        if logits.shape[-1] != 1:
            raise NotImplementedError("eval_epoch: two-class pred_logits (moment_detr) are outside the univtg path")
        if logits.device != self.dev:
            raise RuntimeError(f"eval_epoch: model outputs on {logits.device}, expected {self.dev}")
        B, Lv = logits.shape[:2]
        if self.pool is None:
            self.pool = RowPool(self.dev, self.n_queries_hint * Lv, self.n_queries_hint)
        q0 = len(self.meta)
        self.pool.reserve(self.rows + B * Lv, q0 + B)
        dur = pinned_to_device([float(m["duration"]) for m in query_meta], torch.float64, self.dev).to(torch.float32)
        decode_into_pool(self.pool, outputs, targets, model_inputs["src_vid_mask"], dur, self.rows, q0, not self.opt.no_sort_results,
                         self.opt.eval_mode, self.opt.round_multiple, self.opt.clip_length)
        for b in range(B):
            self.row_off.append(self.rows + b * Lv)
            self.n_rows.append(Lv)
        self.meta.extend(query_meta)
        self.rows += B * Lv

    def add_losses(self, loss_dict):
        """Keep one batch's loss values on the device ([K] fp32, in the criterion's key order)."""
        keys = tuple(loss_dict.keys())
        if self.loss_keys is None:
            self.loss_keys = keys
        elif keys != self.loss_keys:
            raise ValueError(f"eval_epoch: the criterion returned keys {keys}, earlier batches {self.loss_keys}")
        vals = [v if torch.is_tensor(v) else torch.full((), float(v), device=self.dev) for v in loss_dict.values()]
        self.losses.append(torch.stack([v.detach().reshape(()).to(device=self.dev, dtype=torch.float32) for v in vals]))

    def finish(self, weight_dict):
        """NMS over the pool, loss_overall, and one device-to-host copy -> host numpy arrays."""
        opt, dev = self.opt, self.dev
        Q = len(self.meta)
        offsets = np.array(self.row_off + [self.rows], dtype=np.int64)
        parts_f64 = [self.pool.rows[:self.rows].reshape(-1)]
        nms = opt.nms_thd != -1
        if nms:
            off_dev = pinned_to_device(offsets, torch.int64, dev)
            kept, counts = nms_pool(self.pool.rows, off_dev, Q, max(self.n_rows), opt.nms_thd, opt.max_before_nms,
                                    opt.max_after_nms, opt.no_sort_results)
            parts_f64.append(kept[:Q].reshape(-1))
        parts_32 = [self.pool.hl[:self.rows]]
        if self.losses:
            L = torch.stack(self.losses)  # [n_batches, K]
            # loss_overall = sum(loss_dict[k] * weight_dict[k] ...): Python's sum starts at 0, then one fp32 add per weighted key
            total = None
            for j, k in enumerate(self.loss_keys):
                if k in weight_dict:
                    term = L[:, j] * weight_dict[k]
                    total = (0 + term) if total is None else total + term
            if total is None:
                total = torch.zeros(L.shape[0], device=dev)
            parts_32.append(torch.cat([L, total[:, None]], 1).reshape(-1))
        parts_i32 = [self.pool.lens[:Q]] + ([counts[:Q]] if nms else [])
        arena = torch.cat([t.contiguous().view(torch.uint8) for t in parts_f64 + parts_32 + parts_i32])
        host = arena.cpu().numpy()
        o = 0

        def take(n, dt):
            nonlocal o
            a = host[o:o + n * np.dtype(dt).itemsize].view(dt)
            o += n * np.dtype(dt).itemsize
            return a

        res = {"rows": take(self.rows * 3, np.float64).reshape(-1, 3)}
        if nms:
            res["kept"] = take(Q * opt.max_after_nms * 3, np.float64).reshape(Q, opt.max_after_nms, 3)
        res["hl"] = take(self.rows, np.float32)
        if self.losses:
            K = len(self.loss_keys)
            res["losses"] = take(len(self.losses) * (K + 1), np.float32).reshape(len(self.losses), K + 1)
        res["lens"] = take(Q, np.int32)
        if nms:
            res["counts"] = take(Q, np.int32)
        res["offsets"] = offsets
        return res


def _submission(meta, host, windows_of):
    out = []
    rows_l = host["rows"]
    for q, m in enumerate(meta):
        o = int(host["offsets"][q])
        out.append(dict(qid=m["qid"], query=m["query"], vid=m["vid"], pred_relevant_windows=windows_of(q, o),
                        pred_saliency_scores=host["hl"][o:o + int(host["lens"][q])].tolist()))
    return out


def eval_epoch(model, eval_dataset, opt, save_submission_filename, epoch_i=None, criterion=None, tb_writer=None, *, collate_fn=None,
               prepare_batch=None):
    """main/inference_mr.py eval_epoch on the device -> (metrics, metrics_nms, eval_loss_meters, latest_file_paths).

    collate_fn / prepare_batch default to main.dataset.start_end_collate_mr / prepare_batch_inputs_mr of the UniVTG checkout on
    sys.path.  Refuses, before anything launches: model_id "moment_detr", span_loss_type other than "l1" and a model that is not on
    a CUDA device; two-class pred_logits are refused before the first decode.

    As in the reference, the padded clips of pred_logits are scored 0 for the submission.  The reference does this in place on
    the model's outputs before its criterion runs; the criterion weights those clips by 0 (loss_labels' weights and mask), so the
    outputs are handed to the criterion unchanged here."""
    from torch.utils.data import DataLoader

    dev = check_options(model, opt)
    if collate_fn is None or prepare_batch is None:
        from main.dataset import prepare_batch_inputs_mr, start_end_collate_mr

        collate_fn = collate_fn or start_end_collate_mr
        prepare_batch = prepare_batch or prepare_batch_inputs_mr
    model.eval()
    if criterion is not None and eval_dataset.load_labels:
        criterion.eval()
    else:
        criterion = None
    loader = DataLoader(eval_dataset, collate_fn=collate_fn, batch_size=opt.eval_bsz, num_workers=opt.num_workers, shuffle=False,
                        pin_memory=opt.pin_memory)
    write_tb = tb_writer is not None and epoch_i is not None
    state = EpochState(dev, len(eval_dataset), opt)
    with torch.no_grad(), torch.cuda.device(dev):
        for batch in loader:
            step(model, criterion, state, batch, prepare_batch, opt)
            if opt.debug:
                break
        weight_dict = criterion.weight_dict if criterion else {}
        host = state.finish(weight_dict)

    meters = defaultdict(AverageMeter)
    if criterion:
        keys = list(state.loss_keys) + ["loss_overall"]
        for row in host["losses"]:
            for k, v in zip(keys, row.tolist()):
                meters[k].update(float(v) * weight_dict[k] if k in weight_dict else float(v))
    if write_tb and criterion:
        for k, v in meters.items():
            tb_writer.add_scalar("Eval/{}".format(k), v.avg, epoch_i + 1)

    rows = host["rows"]
    submission = _submission(state.meta, host, lambda q, o: rows[o:o + state.n_rows[q]].tolist())
    if opt.no_sort_results:
        save_submission_filename = save_submission_filename.replace(".jsonl", "_unsorted.jsonl")
    gt_data = eval_dataset.data
    submission_path = os.path.join(opt.results_dir, save_submission_filename)
    _save_jsonl(submission, submission_path)
    if opt.eval_split_name in ["val", "test"]:
        metrics = eval_submission(submission, gt_data, verbose=opt.debug, match_number=not opt.debug)
        save_metrics_path = submission_path.replace(".jsonl", "_metrics.json")
        _save_json_pretty(metrics, save_metrics_path)
        latest_file_paths = [submission_path, save_metrics_path]
    else:
        metrics = None
        latest_file_paths = [submission_path, ]
    metrics_nms = None
    if opt.nms_thd != -1:
        kept, counts = host["kept"], host["counts"]
        after = []
        for q, e in enumerate(submission):
            e = dict(e)
            e["pred_relevant_windows"] = kept[q, :int(counts[q])].tolist()
            after.append(e)
        submission_nms_path = submission_path.replace(".jsonl", "_nms_thd_{}.jsonl".format(opt.nms_thd))
        _save_jsonl(after, submission_nms_path)
        if opt.eval_split_name == "val":
            metrics_nms = eval_submission(after, gt_data, verbose=opt.debug, match_number=not opt.debug)
            save_metrics_nms_path = submission_nms_path.replace(".jsonl", "_metrics.json")
            _save_json_pretty(metrics_nms, save_metrics_nms_path)
            latest_file_paths += [submission_nms_path, save_metrics_nms_path]
        else:
            latest_file_paths = [submission_nms_path, ]
    return metrics, metrics_nms, meters, latest_file_paths


def step(model, criterion, state, batch, prepare_batch, opt):
    """One batch of the epoch: forward, decode into the pool, criterion - enqueued without a host synchronisation."""
    query_meta = batch[0]
    model_inputs, targets = prepare_batch(batch[1], opt.device, non_blocking=opt.pin_memory)
    outputs = model(**model_inputs)
    state.add_batch(query_meta, model_inputs, targets, outputs)
    if criterion:
        state.add_losses(criterion(outputs, targets))
