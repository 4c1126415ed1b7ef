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
"""
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
