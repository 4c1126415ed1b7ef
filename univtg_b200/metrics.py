"""Moment-retrieval and highlight metrics of the reference's `eval_submission` (eval/eval.py:292-374), computed on the device.

    from univtg_b200.metrics import eval_submission   # instead of: from eval.eval import eval_submission

Same arguments, same returned OrderedDict (`json.dumps` of both is the same string).  The per-query values - AP over the IoU
thresholds for every length range, the R1 / R5 IoUs, the highlight AP of every (min score, annotator) curve and HIT@1 - come from
two kernel launches (univtg_eval_mr, univtg_eval_hl) and equal the reference's bit for bit.  The means over queries and the
`.2f` formatting are the reference's own numpy calls on arrays of the same shapes, so they are identical by construction.

The host packs the lists into flat arrays with one host-to-device copy and reads the small per-query arrays back with one
device-to-host copy.  Only the first 10 windows of a query are read (AP: 10, R5: 5, R1: 1), in submission order, so clip-order
submissions (--no_sort_results) are evaluated as the reference evaluates them.

Inputs the reference cannot evaluate (it crashes or produces NaN) raise ValueError before anything launches: an empty
submission, duplicate qids, a query without predicted windows, a ground-truth entry without relevant_windows, more than 64 gt
windows, int(duration / 2) outside 1..4096, empty or out-of-range relevant_clip_ids, an empty or (within the first
int(duration / 2) clips) non-finite predicted saliency list.  A qid mismatch under match_number=True raises AssertionError, as
the reference does.  Nothing is printed.  CUDA only.

evaluate_hl (bottom of this module) does the same for the TVSum / YouTube highlight evaluation of main/dataset.py.
"""
import json
import os
from collections import OrderedDict
from itertools import chain

import numpy as np
import torch

from . import _lib

MAX_PRED = 10
MAX_GT = 64
MAX_CLIPS = 4096
MR_THDS = [float(f"{e:.2f}") for e in np.linspace(0.5, 0.95, 10)]
R_THDS = [float(f"{e:.2f}") for e in np.linspace(0.3, 0.95, 14)]
RANGES = ("short", "middle", "long", "full")  # (0, 10], (10, 30], (30, inf), everything
HL_NAMES = ("Fair", "Good", "VeryGood")  # min score 2, 3, 4
# brief key -> (range, metric, sub-key)
MR_BRIEF = {
    "MR-full-mAP-key": ("full", "MR-mAP", "average"), "MR-full-mAP@0.5-key": ("full", "MR-mAP", "0.5"),
    "MR-full-mAP@0.75-key": ("full", "MR-mAP", "0.75"), "MR-short-mAP": ("short", "MR-mAP", "average"),
    "MR-middle-mAP": ("middle", "MR-mAP", "average"), "MR-long-mAP": ("long", "MR-mAP", "average"),
    "MR-short-mIoU": ("short", "MR-mIoU", None), "MR-middle-mIoU": ("middle", "MR-mIoU", None),
    "MR-long-mIoU": ("long", "MR-mIoU", None), "MR-full-mIoU-key": ("full", "MR-mIoU", None),
    "MR-full-R1@0.3-key": ("full", "MR-R1", "0.3"), "MR-full-R1@0.5-key": ("full", "MR-R1", "0.5"),
    "MR-full-R1@0.7-key": ("full", "MR-R1", "0.7"), "MR-full-R5@0.3-key": ("full", "MR-R5", "0.3"),
    "MR-full-R5@0.5-key": ("full", "MR-R5", "0.5"), "MR-full-R5@0.7-key": ("full", "MR-R5", "0.7"),
}


def _unique_qids(items, what):
    qids = [d["qid"] for d in items]
    if len(set(qids)) != len(qids):
        raise ValueError(f"eval_submission: duplicate qids in {what}")
    return qids


def _scatter(flat, counts, width, tail):
    """Rows of `flat` (grouped by query, counts[q] each) -> zero-padded [Q, width, *tail]."""
    out = np.zeros((len(counts), width) + tail)
    if len(flat):
        q = np.repeat(np.arange(len(counts)), counts)
        pos = np.arange(len(flat)) - np.repeat(np.cumsum(counts) - counts, counts)
        out[q, pos] = flat
    return out


def _rows(lists, cols, what):
    flat = [w[:cols] for lst in lists for w in lst]
    try:
        arr = np.array(flat, dtype=np.float64).reshape(len(flat), cols)
    except (ValueError, TypeError):
        raise ValueError(f"eval_submission: every {what} must hold {cols} numbers") from None
    return arr


def pack_mr(submission, gts):
    """-> (pred [Q,10,3], n_pred [Q], gt [Q,G,2], n_gt [Q]) in submission order."""
    preds = [d["pred_relevant_windows"][:MAX_PRED] for d in submission]
    n_pred = np.array([len(p) for p in preds], dtype=np.int32)
    if (n_pred == 0).any():
        raise ValueError(f"eval_submission: query {submission[int(np.argmin(n_pred))]['qid']!r} has no predicted window")
    wins = [g.get("relevant_windows") or [] for g in gts]
    n_gt = np.array([len(w) for w in wins], dtype=np.int32)
    if (n_gt == 0).any():
        raise ValueError(f"eval_submission: ground truth of qid {gts[int(np.argmin(n_gt))]['qid']!r} has no relevant_windows")
    if (n_gt > MAX_GT).any():
        raise ValueError(f"eval_submission: more than {MAX_GT} ground-truth windows in one query")
    pred = _scatter(_rows(preds, 3, "predicted window [st, ed, score]"), n_pred, MAX_PRED, (3,))
    gt = _scatter(_rows(wins, 2, "ground-truth window [st, ed]"), n_gt, int(n_gt.max()), (2,))
    return pred, n_pred, gt, n_gt


def pack_hl(submission, gts):
    """-> (sal [Q,S], n_sal [Q], labels [Q,C] u16 with bit 3*l + a = (score of annotator a >= 2 + l), n_clips [Q])."""
    sal_lists = [d["pred_saliency_scores"] for d in submission]
    n_sal = np.array([len(s) for s in sal_lists], dtype=np.int32)
    if (n_sal == 0).any():
        raise ValueError("eval_submission: empty pred_saliency_scores")
    sal = _scatter(np.fromiter(chain.from_iterable(sal_lists), np.float64, int(n_sal.sum())), n_sal, int(n_sal.max()), ())
    n_clips = np.array([int(g["duration"] / 2) for g in gts], dtype=np.int64)
    if (n_clips < 1).any() or (n_clips > MAX_CLIPS).any():
        raise ValueError(f"eval_submission: int(duration / 2) must be in 1..{MAX_CLIPS}")
    C = int(n_clips.max())
    seen = np.minimum(n_sal, n_clips)  # the part of the prediction scikit-learn sees
    if not np.isfinite(sal[np.arange(sal.shape[1])[None, :] < seen[:, None]]).all():
        raise ValueError("eval_submission: non-finite pred_saliency_scores")
    ids = [g["relevant_clip_ids"] for g in gts]
    n_ids = np.array([len(i) for i in ids], dtype=np.int64)
    if (n_ids == 0).any() or (n_ids > MAX_CLIPS).any():
        raise ValueError(f"eval_submission: relevant_clip_ids must hold 1..{MAX_CLIPS} clips")
    if any(len(g["saliency_scores"]) != n for g, n in zip(gts, n_ids.tolist())):
        raise ValueError("eval_submission: saliency_scores and relevant_clip_ids differ in length")
    flat_ids = np.fromiter(chain.from_iterable(ids), np.int64, int(n_ids.sum()))
    qi = np.repeat(np.arange(len(gts)), n_ids)
    if (flat_ids < 0).any() or (flat_ids >= n_clips[qi]).any():
        raise ValueError("eval_submission: a relevant_clip_ids entry is outside [0, int(duration / 2))")
    full = np.zeros((len(gts), C, 3))
    full[qi, flat_ids] = _rows([g["saliency_scores"] for g in gts], 3, "saliency_scores row")
    labels = np.zeros((len(gts), C), dtype=np.uint16)
    for lv in range(3):
        for a in range(3):
            labels |= (full[:, :, a] >= 2 + lv).astype(np.uint16) << (3 * lv + a)
    return sal, n_sal, labels, n_clips.astype(np.int32)


def _stage(arrays):
    """Lay contiguous numpy arrays out in one byte buffer (8-byte aligned) -> (buffer, offsets)."""
    offs, total = [], 0
    for a in arrays:
        offs.append(total)
        total += (a.nbytes + 7) // 8 * 8
    buf = np.zeros(max(total, 8), dtype=np.uint8)
    for a, o in zip(arrays, offs):
        buf[o:o + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    return buf, offs


def per_query(mr_in, hl_in):
    """Launch the kernels on packed inputs (either may be None) -> dict of per-query numpy arrays:
    ap [4,Q,10], iou_r1 [4,Q], iou_r5 [4,Q], kept [4,Q] bool; hl_ap [3,Q,3], hit [3,Q,3]."""
    if not torch.cuda.is_available():
        raise RuntimeError("univtg_b200: eval_submission runs on CUDA only (no CPU path)")
    lib = _lib.load_library()
    ins = (list(mr_in) if mr_in else []) + (list(hl_in) if hl_in else [])
    Q = len(ins[1])
    hbuf, hoff = _stage(ins)
    shapes = []  # output (name, dtype, shape)
    if mr_in:
        shapes += [("ap", np.float64, (4, Q, 10)), ("iou_r1", np.float64, (4, Q)), ("iou_r5", np.float64, (4, Q)),
                   ("kept", np.uint8, (4, Q))]
    if hl_in:
        shapes += [("hl_ap", np.float64, (3, Q, 3)), ("hit", np.float64, (3, Q, 3))]
    ooff, total = [], 0
    for _, dt, shp in shapes:
        ooff.append(total)
        total += (int(np.prod(shp)) * np.dtype(dt).itemsize + 7) // 8 * 8
    dev = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        dbuf = torch.from_numpy(hbuf).to(dev)
        dout = torch.empty(total, dtype=torch.uint8, device=dev)
        ib, ob = dbuf.data_ptr(), dout.data_ptr()
        inp = [_lib.c_void_p(ib + o) for o in hoff]
        out = {name: _lib.c_void_p(ob + o) for (name, _, _), o in zip(shapes, ooff)}
        stream = _lib.stream_ptr()
        if mr_in:
            pred, n_pred, gt, n_gt = mr_in
            _lib.check(lib.univtg_eval_mr(inp[0], inp[1], inp[2], inp[3], Q, gt.shape[1], out["ap"], out["iou_r1"], out["iou_r5"],
                                          out["kept"], stream), "univtg_eval_mr")
        if hl_in:
            k = 4 if mr_in else 0
            sal, labels = hl_in[0], hl_in[2]
            scratch = torch.empty(Q * 9 * labels.shape[1], dtype=torch.float64, device=dev)
            _lib.check(lib.univtg_eval_hl(inp[k], inp[k + 1], inp[k + 2], inp[k + 3], Q, sal.shape[1], labels.shape[1],
                                          _lib.ptr(scratch), out["hl_ap"], out["hit"], stream), "univtg_eval_hl")
        host = dout.cpu().numpy()
    res = {}
    for (name, dt, shp), o in zip(shapes, ooff):
        res[name] = host[o:o + int(np.prod(shp)) * np.dtype(dt).itemsize].view(dt).reshape(shp)
    if "kept" in res:
        res["kept"] = res["kept"].astype(bool)
    return res


def _fmt(v):
    return float(f"{v:.2f}")


def _mr_metrics(pq):
    out = {}
    for r, name in enumerate(RANGES):
        src = r if pq["kept"][r].any() else 3  # no query in the range: the reference evaluates the full set
        keep = pq["kept"][src]
        ap_thds = pq["ap"][src][keep].mean(0)
        mr_ap = dict(zip([str(t) for t in MR_THDS], ap_thds))
        mr_ap["average"] = np.mean(ap_thds)
        i1, i5 = pq["iou_r1"][src][keep], pq["iou_r5"][src][keep]
        out[name] = {"MR-mIoU": _fmt(np.mean(i1) * 100), "MR-mAP": {k: _fmt(100 * v) for k, v in mr_ap.items()},
                     "MR-R1": {str(t): _fmt(np.mean(i1 >= t) * 100) for t in R_THDS},
                     "MR-R5": {str(t): _fmt(np.mean(i5 >= t) * 100) for t in R_THDS}}
    return out


def _hl_metrics(pq):
    return {f"HL-min-{name}": {"HL-mAP": _fmt(100 * np.mean(pq["hl_ap"][lv])), "HL-Hit1": _fmt(100 * np.mean(np.max(pq["hit"][lv], 1)))}
            for lv, name in enumerate(HL_NAMES)}


def eval_submission(submission, ground_truth, verbose=True, match_number=True):
    """eval/eval.py eval_submission on the device.  `verbose` is accepted for compatibility; nothing is printed."""
    sub_q = _unique_qids(submission, "submission")
    gt_q = _unique_qids(ground_truth, "ground_truth")
    if match_number:
        if set(sub_q) != set(gt_q):
            raise AssertionError("qids in ground_truth and submission must match. "
                                 "use `match_number=False` if you wish to disable this check")
    else:
        shared = set(sub_q) & set(gt_q)
        submission = [d for d in submission if d["qid"] in shared]
        ground_truth = [d for d in ground_truth if d["qid"] in shared]
    if not submission:
        raise ValueError("eval_submission: empty submission" + ("" if match_number else " (no qid shared with the ground truth)"))
    gt_by = {d["qid"]: d for d in ground_truth}
    gts = [gt_by[d["qid"]] for d in submission]
    do_mr = "pred_relevant_windows" in submission[0]
    do_hl = ("pred_saliency_scores" in submission[0] and "saliency_scores" in ground_truth[0]
             and isinstance(ground_truth[0]["saliency_scores"], list))
    mr_in = pack_mr(submission, gts) if do_mr else None
    hl_in = pack_hl(submission, gts) if do_hl else None
    metrics, brief = {}, OrderedDict()
    if do_mr or do_hl:
        pq = per_query(mr_in, hl_in)
    if do_mr:
        mr = _mr_metrics(pq)
        metrics.update(mr)
        for k in sorted(MR_BRIEF):
            rng, m, sub = MR_BRIEF[k]
            brief[k] = mr[rng][m] if sub is None else mr[rng][m][sub]
    if do_hl:
        hl = _hl_metrics(pq)
        metrics.update(hl)
        for k, v in hl.items():
            brief[f"{k}-mAP"] = v["HL-mAP"]
            brief[f"{k}-Hit1"] = v["HL-Hit1"]
        brief["HL-min-VeryGood-mAP-key"] = brief.pop("HL-min-VeryGood-mAP")
        brief["HL-min-VeryGood-Hit1-key"] = brief.pop("HL-min-VeryGood-Hit1")
    final = OrderedDict()
    final["brief"] = brief
    final.update(sorted(metrics.items()))
    return final


# ---- TVSum / YouTube highlight detection: main/dataset.py DatasetHL.evaluate --------------------------------------------
TVSUM_ANNOTATORS = 20
MAX_ANNOTATORS = 32
HL_SCORE_DTYPES = (torch.float32, torch.float16, torch.bfloat16)  # convert to fp32 without changing order or ties


def _hl_rows(blob):
    rows = []
    for score in blob:
        row = score[0]
        if not torch.is_tensor(row):
            raise TypeError("evaluate_hl: blob entries must be tensors (the reference argsorts score[0] with torch)")
        if row.dim() != 1:
            raise ValueError(f"evaluate_hl: score[0] must be one score row, got shape {list(row.shape)}")
        if row.dtype not in HL_SCORE_DTYPES:
            raise ValueError(f"evaluate_hl: scores must be float32, float16 or bfloat16, got {row.dtype}")
        if row.numel() > MAX_CLIPS:
            raise ValueError(f"evaluate_hl: more than {MAX_CLIPS} scores in one row")
        rows.append(row.detach())
    return rows


def pack_hl_labels(dataset, n_videos, lengths, k=5):
    """-> (labels [V,C,A] f32, n_label [V] i32, n_cut [V] i32, median flag) for the first n_videos videos of `dataset` in its
    current state.  TVSum: the first 20 columns of `anno`, thresholded on the device at their lower median, n_cut =
    len(list[:k]); YouTube: [1 if s > 0 else 0 for s in match] in one column, the whole list."""
    name = dataset.dset_name
    if name not in ("tvsum", "youtube"):
        raise NotImplementedError(f"evaluate_hl: dset_name {name!r}")
    cols, rows_n = [], []
    for idx in range(n_videos):
        lab = dataset.label[dataset.get_video_id(idx)]
        if name == "tvsum":
            a = np.asarray(lab["anno"], dtype=np.float32)
            if a.ndim != 2 or a.shape[1] < TVSUM_ANNOTATORS:
                raise IndexError(f"evaluate_hl: anno of video {idx} has shape {list(a.shape)}, the reference reads 20 columns")
            a = a[:, :TVSUM_ANNOTATORS]
        else:
            a = np.array([1 if s > 0 else 0 for s in lab["match"]], dtype=np.float32).reshape(-1, 1)
        if lengths[idx] > len(a):
            raise IndexError(f"evaluate_hl: score row {idx} has {lengths[idx]} entries, its video {len(a)} labels")
        if len(a) > MAX_CLIPS:
            raise ValueError(f"evaluate_hl: more than {MAX_CLIPS} labelled clips in one video")
        if not np.isfinite(a).all():
            raise ValueError(f"evaluate_hl: non-finite labels in video {idx}")
        cols.append(a)
        rows_n.append(len(a))
    A = cols[0].shape[1]
    C = max(1, max(rows_n))
    labels = np.zeros((n_videos, C, A), dtype=np.float32)
    for v, a in enumerate(cols):
        labels[v, :len(a)] = a
    if name == "tvsum":
        n_cut = [len(range(n)[:k]) for n in lengths]
    else:
        n_cut = list(lengths)
    return labels, np.array(rows_n, dtype=np.int32), np.array(n_cut, dtype=np.int32), int(name == "tvsum")


def hl_topk_ap(rows, labels, n_label, n_cut, median):
    """univtg_eval_hl_topk on finite score rows (1-D tensors on any device) and packed labels -> ap [V, A] float64 numpy."""
    if not torch.cuda.is_available():
        raise RuntimeError("univtg_b200: evaluate_hl runs on CUDA only (no CPU path)")
    lib = _lib.load_library()
    V, C, A = labels.shape
    n_score = np.array([r.numel() for r in rows], dtype=np.int32)
    dev = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        S = max(1, int(n_score.max()))
        scores = torch.zeros(V, S, dtype=torch.float32, device=dev)
        for v, r in enumerate(rows):
            scores[v, :r.numel()] = r.to(device=dev, dtype=torch.float32)
        hbuf, hoff = _stage([n_score, n_cut, labels, n_label])
        dbuf = torch.from_numpy(hbuf).to(dev)
        ap = torch.empty(V, A, dtype=torch.float64, device=dev)
        ib = dbuf.data_ptr()
        _lib.check(lib.univtg_eval_hl_topk(_lib.ptr(scores), _lib.c_void_p(ib + hoff[0]), _lib.c_void_p(ib + hoff[1]),
                                           _lib.c_void_p(ib + hoff[2]), _lib.c_void_p(ib + hoff[3]), V, S, C, A, median,
                                           _lib.ptr(ap), _lib.stream_ptr()), "univtg_eval_hl_topk")
        return ap.cpu().numpy()


def _write_hl_jsonl(dataset, blob, save_dir):
    """The reference's per-video prediction file, <save_dir>/<dset_name>/<domain>.jsonl."""
    with open(os.path.join(save_dir, dataset.dset_name, dataset.domain + ".jsonl"), "w") as f:
        for idx, score in enumerate(blob):
            video_id = dataset.get_video_id(idx)
            lab = dataset.label[video_id]
            entry = {"vid": video_id, "pred": score[0].tolist(), "gt": dataset.get_saliency(idx).tolist(),
                     "duration": int(lab["frames"]) / int(lab["fps"]), "domain": lab["domain"], "fps": lab["fps"]}
            if dataset.dset_name == "tvsum":
                entry.update({"title": lab["title"]})
            if dataset.dset_name == "youtube":
                entry.update({"clip": lab["clip"]})
            f.write(json.dumps(entry) + "\n")


def evaluate_hl(dataset, blob, k=5, save_dir=None):
    """main/dataset.py DatasetHL.evaluate on the device: `evaluate_hl(train_val_dataset, scores)` for
    `train_val_dataset.evaluate(scores)`.  Returns the same {'mAP': round(mean AP, 5)}.

    dataset: anything with dset_name ('tvsum' / 'youtube'), domain, label (video id -> dict with 'anno' [clips, >= 20] or
    'match' [clips]) and get_video_id(idx) in its 'val' state; get_saliency(idx) is read only for save_dir.
    blob: the list eval_epoch collects, one tensor per eval batch, on the CPU or CUDA.  As in the reference, row 0 of entry idx
    is scored against video idx - with eval_bsz 1 that is every video; with the default eval_bsz 100 it is not the video that
    row belongs to, and only len(blob) videos are evaluated.  This is kept as the reference has it so results stay comparable.

    The ranking is the reference's torch.argsort(descending=True) on the CPU (ties included), TVSum labels are > the lower median
    of each annotator's column, the APs are computed per (video, annotator) by univtg_eval_hl_topk bit for bit, and the means
    are the reference's own Python sums (over videos, then over annotators) and round().

    Raises, before any launch: IndexError for a score row longer than its video's labels (or anno with fewer than 20 columns),
    ZeroDivisionError for an empty blob, TypeError for non-tensor entries, ValueError for non-finite scores or labels, score
    dtypes other than float32 / float16 / bfloat16 and more than 4,096 clips.  With save_dir the reference's jsonl file is
    written first, as the reference does.  CUDA only."""
    if dataset.dset_name not in ("tvsum", "youtube"):
        raise NotImplementedError(f"evaluate_hl: dset_name {dataset.dset_name!r}")
    if save_dir is not None:
        _write_hl_jsonl(dataset, blob, save_dir)
    rows = _hl_rows(blob)
    if not rows:
        raise ZeroDivisionError("evaluate_hl: empty blob")
    by_device = {}
    for r in rows:
        by_device.setdefault(r.device, []).append(r.float())
    if not all(bool(torch.isfinite(torch.cat(rs)).all()) for rs in by_device.values()):
        raise ValueError("evaluate_hl: non-finite scores")
    labels, n_label, n_cut, median = pack_hl_labels(dataset, len(rows), [r.numel() for r in rows], k)
    ap = hl_topk_ap(rows, labels, n_label, n_cut, median)
    if median:
        collected = []
        for i in range(TVSUM_ANNOTATORS):
            video_ap = ap[:, i].tolist()
            collected.append(sum(video_ap) / len(video_ap))
    else:
        collected = ap[:, 0].tolist()
    mean_ap = sum(collected) / len(collected)
    return dict(mAP=round(mean_ap, 5))
