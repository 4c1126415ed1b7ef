"""Post-forward decode of the reference's moment-retrieval evaluation, on the device.

What `compute_mr_results` (main/inference_mr.py:101-167) and `post_processing_mr_nms` (:31-40) do per batch in Python -
add the clip timestamps, zero the scores of padded clips, scale / clamp to the video duration, sort by score, round to four
decimals, temporal NMS - as two kernel launches on the batch (univtg_decode_mr, univtg_temporal_nms); one device-to-host
copy of the finished rows replaces the per-sample `.cpu()`, `sorted` and O(n^2) list surgery.  CUDA only.
"""
import torch

from . import _lib


def _f32(t, dev):
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def decode_mr(outputs, targets, durations, sort=True, rounded=True):
    """Rows [st, ed, score] per clip, sorted by score (descending, ties in clip order).

    outputs: the model's output dict; targets: dict with 'timestamp' [B,Lv,2] and 'timestamp_mask' [B,Lv];
    durations: [B] seconds (or None: windows stay in timestamp units, no clamp - the main_gradio.py convention).
    Returns {'windows': [B,Lv,3] f32, 'windows_r4': [B,Lv,3] f64 (float(f"{e:.4f}") of every number) or None, 'order': [B,Lv] i32}.
    """
    logits = outputs["pred_logits"]
    dev = logits.device
    if dev.type != "cuda":
        raise RuntimeError("univtg_b200: decode_mr runs on CUDA tensors only (no CPU path)")
    if logits.shape[-1] != 1:
        raise NotImplementedError("decode_mr: two-class pred_logits (moment_detr) are outside the univtg path")
    B, Lv = logits.shape[:2]
    lib = _lib.load_library()
    with torch.cuda.device(dev):
        lg = _f32(logits.reshape(B, Lv), dev)
        sp = _f32(outputs["pred_spans"], dev)
        ts = _f32(targets["timestamp"], dev)
        tm = _f32(targets["timestamp_mask"], dev)
        dur = None
        if durations is not None:
            dur = torch.as_tensor(durations, dtype=torch.float64).to(torch.float32).to(dev).contiguous()
        windows = torch.empty(B, Lv, 3, dtype=torch.float32, device=dev)
        r4 = torch.empty(B, Lv, 3, dtype=torch.float64, device=dev) if rounded else None
        order = torch.empty(B, Lv, dtype=torch.int32, device=dev)
        _lib.check(lib.univtg_decode_mr(_lib.ptr(lg), _lib.ptr(sp), _lib.ptr(ts), _lib.ptr(tm), _lib.ptr(dur), B, Lv, int(bool(sort)),
                                        _lib.ptr(windows), _lib.ptr(r4), _lib.ptr(order), _lib.stream_ptr()), "univtg_decode_mr")
    return {"windows": windows, "windows_r4": r4, "order": order}


def temporal_nms(windows_r4, nms_thd, max_before_nms=10, max_after_nms=10):
    """Batched utils/temporal_nms.py over sorted rows [B,n,3] f64 -> (kept rows [B,max_after_nms,3] f64, counts [B] i32)."""
    dev = windows_r4.device
    if dev.type != "cuda":
        raise RuntimeError("univtg_b200: temporal_nms runs on CUDA tensors only (no CPU path)")
    w = windows_r4.detach().to(torch.float64).contiguous()
    B, n = w.shape[:2]
    lib = _lib.load_library()
    with torch.cuda.device(dev):
        out = torch.zeros(B, max_after_nms, 3, dtype=torch.float64, device=dev)
        counts = torch.zeros(B, dtype=torch.int32, device=dev)
        _lib.check(lib.univtg_temporal_nms(_lib.ptr(w), B, n, int(max_before_nms), float(nms_thd), int(max_after_nms), _lib.ptr(out),
                                           _lib.ptr(counts), _lib.stream_ptr()), "univtg_temporal_nms")
    return out, counts


def compose_submission(query_meta, outputs, targets, model_inputs, nms_thd=-1, max_before_nms=10, max_after_nms=10, sort=True, *,
                       eval_mode=None, round_multiple=0, clip_length=1.0):
    """The list of dicts `compute_mr_results` appends to `mr_res` (main/inference_mr.py:158-165), for one batch; with
    nms_thd != -1 `pred_relevant_windows` is what post_processing_mr_nms would leave (:31-40).

    eval_mode "add" gives pred_saliency_scores = fp32(fp16(saliency)) + prob (:124-125; None, "add_mr" and other values: the fp16
    saliency), and round_multiple > 0 applies PostProcessorDETR's round_multiple with clip_length (:184-192) before the NMS, as
    eval_epoch does.  For a whole evaluation epoch use univtg_b200.evaluation.eval_epoch, which also writes the files."""
    if eval_mode is not None or round_multiple > 0:
        return _compose_pool(query_meta, outputs, targets, model_inputs, nms_thd, max_before_nms, max_after_nms, sort, eval_mode,
                             round_multiple, clip_length)
    durations = [m["duration"] for m in query_meta]
    dec = decode_mr(outputs, targets, durations, sort=sort, rounded=True)
    rows = dec["windows_r4"]
    if nms_thd != -1:
        kept, counts = temporal_nms(rows, nms_thd, max_before_nms, max_after_nms)
        kept, counts = kept.cpu(), counts.cpu().tolist()
        windows = [kept[b, :counts[b]].tolist() for b in range(len(query_meta))]
    else:
        windows = rows.cpu().tolist()
    sal = outputs["saliency_scores"].detach().half().cpu()
    lens = model_inputs["src_vid_mask"].detach().sum(1).cpu().tolist()
    res = []
    for b, meta in enumerate(query_meta):
        res.append(dict(qid=meta["qid"], query=meta["query"], vid=meta["vid"], pred_relevant_windows=windows[b],
                        pred_saliency_scores=sal[b, :int(lens[b])].tolist()))
    return res


def _compose_pool(query_meta, outputs, targets, model_inputs, nms_thd, max_before_nms, max_after_nms, sort, eval_mode, round_multiple,
                  clip_length):
    from types import SimpleNamespace

    from .evaluation import EpochState

    dev = outputs["pred_logits"].device
    if dev.type != "cuda":
        raise RuntimeError("univtg_b200: compose_submission runs on CUDA tensors only (no CPU path)")
    opt = SimpleNamespace(no_sort_results=not sort, eval_mode=eval_mode, round_multiple=round_multiple, clip_length=clip_length,
                          nms_thd=nms_thd, max_before_nms=max_before_nms, max_after_nms=max_after_nms)
    with torch.cuda.device(dev):
        state = EpochState(dev, len(query_meta), opt)
        state.add_batch(query_meta, model_inputs, targets, outputs)
        host = state.finish({})
    res = []
    for b, meta in enumerate(query_meta):
        o = int(host["offsets"][b])
        if nms_thd != -1:
            windows = host["kept"][b, :int(host["counts"][b])].tolist()
        else:
            windows = host["rows"][o:o + state.n_rows[b]].tolist()
        res.append(dict(qid=meta["qid"], query=meta["query"], vid=meta["vid"], pred_relevant_windows=windows,
                        pred_saliency_scores=host["hl"][o:o + int(host["lens"][b])].tolist()))
    return res
