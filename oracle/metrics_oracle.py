"""TEST INFRASTRUCTURE ONLY - plain-Python / numpy restatement of the reference's moment-retrieval and highlight metrics.

Only tests/ and tools/ may import this module; the product path (univtg_b200/metrics.py -> univtg_eval_mr / univtg_eval_hl)
never does.  It imports neither scikit-learn nor the reference.

Follows, in behaviour (not in code):
  * eval/eval.py:20-70    compute_mr_ap: first 10 windows per query, per-query AP over the IoU thresholds, mean over queries
  * eval/eval.py:73-132   compute_mr_r1 / compute_mr_r5: the paired "IoU" (intersection / convex hull) of the chosen pair
  * eval/eval.py:139-195  get_data_by_range and the four length ranges (with the empty-range fallback to the full set)
  * eval/eval.py:198-289  highlight HIT@1 and mAP at min scores 2 / 3 / 4
  * eval/eval.py:292-374  eval_submission: the key layout of the returned OrderedDict
  * eval/utils.py:17-211  temporal IoUs, interpolated_precision_recall, compute_average_precision_detection, get_ap
  * sklearn.metrics.precision_recall_curve as pinned by the reference (scikit-learn 1.1.2)

Ground-truth order inside compute_average_precision_detection: the reference visits the gt windows in
`tiou_arr.argsort()[::-1]` order.  numpy's default argsort is not stable everywhere (AVX-512 builds), so which of two distinct
gt windows with equal IoU gets locked is machine dependent there.  This restatement takes the rule a stable argsort gives:
NaN IoUs first (argsort puts NaN last), then decreasing IoU, ties to the higher gt index.

scikit-learn versions: 1.1.2 cuts the curve at the first threshold that reaches full recall; later versions (1.9.0 here) keep
the remaining points.  Those points all have recall 1 and precision no higher than the kept full-recall point (tps is
constant, fps grows).  After get_ap's reversal they form the head of the curve, so the running maximum reaches the kept point
with the same value; np.diff(recall) is 0 inside that head, so none of them is selected either.  get_ap is therefore the same
under both versions; the cut is what this module restates.

The per-query values are what the device kernels must reproduce bit for bit; the means over queries use numpy exactly as the
reference does.  The reference's multiprocessing (imap_unordered) can reorder the rows of its AP array, and so the last bits
of its means; here the rows are in submission order.
"""
from collections import OrderedDict

import numpy as np

MR_THDS = [float(f"{e:.2f}") for e in np.linspace(0.5, 0.95, 10)]
R_THDS = [float(f"{e:.2f}") for e in np.linspace(0.3, 0.95, 14)]
RANGES = (("short", 0, 10), ("middle", 10, 30), ("long", 30, float("inf")), ("full", 0, float("inf")))
HL_LEVELS = ((2, "Fair"), (3, "Good"), (4, "VeryGood"))
MAX_PRED = 10


# ---------------------------------------------------------------- temporal IoUs (eval/utils.py:17-63)
def iou_cross(a, b):
    """[N,2] x [M,2] -> [N,M]; intersection over (len a + len b - intersection); 0/0 gives NaN, as numpy does."""
    a = np.asarray(a, dtype=float).reshape(-1, 2)
    b = np.asarray(b, dtype=float).reshape(-1, 2)
    inter = np.clip(np.minimum(a[:, None, 1], b[None, :, 1]) - np.maximum(a[:, None, 0], b[None, :, 0]), 0, None)
    with np.errstate(invalid="ignore", divide="ignore"):
        return inter / ((a[:, 1] - a[:, 0])[:, None] + (b[:, 1] - b[:, 0])[None, :] - inter)


def iou_paired(p, g):
    """One pair: intersection over the convex hull (the reference's "union"), 0 when the hull is empty."""
    inter = max(0.0, min(p[1], g[1]) - max(p[0], g[0]))
    hull = max(p[1], g[1]) - min(p[0], g[0])
    return inter / hull if hull != 0 else 0.0


# ---------------------------------------------------------------- numpy's summation order
def pairwise_sum(x):
    """np.sum of a contiguous float64 vector as numpy computes it (pairwise_sum in numpy's loops_utils): below 8 elements a
    plain loop from -0.0; up to 128 eight interleaved accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the
    remainder in order; above 128 the sum of the halves split at n/2 rounded down to a multiple of 8.  The device kernels
    sum in this order; tests/test_metrics_cpu.py checks it against np.sum."""
    x = [float(v) for v in x]
    n = len(x)
    if n < 8:
        r = -0.0
        for v in x:
            r += v
        return r
    if n <= 128:
        acc = x[:8]
        i = 8
        while i < n - n % 8:
            for j in range(8):
                acc[j] += x[i + j]
            i += 8
        r = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]))
        for v in x[i:]:
            r += v
        return r
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(x[:n2]) + pairwise_sum(x[n2:])


# ---------------------------------------------------------------- moment retrieval, per query
def interpolated_ap(precision, recall):
    """VOC-2011 interpolated AP over one cumulative precision / recall curve (eval/utils.py:66-82)."""
    p = np.concatenate([[0.0], precision, [0.0]])
    r = np.concatenate([[0.0], recall, [1.0]])
    for i in range(len(p) - 2, -1, -1):
        p[i] = max(p[i], p[i + 1])
    sel = np.nonzero(r[1:] != r[:-1])[0] + 1
    return np.sum((r[sel] - r[sel - 1]) * p[sel])


def gt_visit_order(tiou):
    """Order in which the greedy matcher visits the gt windows: NaN first, then decreasing IoU, ties to the higher index."""
    return np.argsort(tiou, kind="stable")[::-1]


def ap_detection(gt_windows, pred_rows, thds=MR_THDS):
    """compute_average_precision_detection for one query: gt [[st, ed], ...], predictions [[st, ed, score], ...] -> [len(thds)]."""
    ap = np.zeros(len(thds))
    if len(pred_rows) == 0:
        return ap
    preds = sorted(pred_rows, key=lambda r: -r[2])  # stable: equal scores keep submission order
    n = len(preds)
    hit = np.zeros((len(thds), n))
    locked = np.zeros((len(thds), len(gt_windows)), dtype=bool)
    for k, row in enumerate(preds):
        tiou = iou_cross([row[:2]], gt_windows)[0]
        order = gt_visit_order(tiou)
        for t, thd in enumerate(thds):
            for j in order:
                if tiou[j] < thd:
                    break
                if not locked[t, j]:
                    locked[t, j] = True
                    hit[t, k] = 1
                    break
    tp = np.cumsum(hit, axis=1)
    fp = np.cumsum(1 - hit, axis=1)
    recall = tp / float(len(gt_windows))
    precision = tp / (tp + fp)
    for t in range(len(thds)):
        ap[t] = interpolated_ap(precision[t], recall[t])
    return ap


def r1_iou(pred_rows, gt_windows):
    """compute_mr_r1 for one query: the first window against the gt window of highest IoU (np.argmax: first max, NaN wins)."""
    p = pred_rows[0][:2]
    j = int(np.argmax(iou_cross([p], gt_windows)[0]))
    return iou_paired([float(p[0]), float(p[1])], [float(x) for x in gt_windows[j]])


def r5_iou(pred_rows, gt_windows):
    """compute_mr_r5 for one query: NaN -> 0, the first maximum in row-major order over the first 5 windows x gt windows."""
    ious = iou_cross([r[:2] for r in pred_rows[:5]], gt_windows)
    ious[np.isnan(ious)] = 0
    pi, gi = np.where(ious == np.max(ious))
    p, g = pred_rows[:5][pi[0]], gt_windows[gi[0]]
    return iou_paired([float(p[0]), float(p[1])], [float(g[0]), float(g[1])])


def windows_in_range(windows, lo, hi):
    return [w for w in windows if lo < w[1] - w[0] <= hi]


# ---------------------------------------------------------------- highlight detection, per query
def precision_recall_curve(y_true, y_score):
    """scikit-learn 1.1.2's precision_recall_curve for labels in {0, 1} (positive label 1, no sample weights)."""
    y_true = np.asarray(y_true, dtype=float)
    y_score = np.asarray(y_score, dtype=float)
    order = np.argsort(y_score, kind="mergesort")[::-1]
    s, t = y_score[order], y_true[order]
    ends = np.concatenate([np.nonzero(np.diff(s))[0], [t.size - 1]])
    tps = np.cumsum(t, dtype=np.float64)[ends]
    fps = 1 + ends - tps
    with np.errstate(invalid="ignore", divide="ignore"):
        precision = tps / (tps + fps)
    precision[np.isnan(precision)] = 0
    recall = tps / tps[-1]
    last = tps.searchsorted(tps[-1])
    keep = slice(last, None, -1)
    return np.concatenate([precision[keep], [1.0]]), np.concatenate([recall[keep], [0.0]]), s[ends][keep]


def get_ap(y_true, y_predict):
    """eval/utils.py get_ap with its defaults (interpolate=True, point_11=False)."""
    labels = set(np.asarray(y_true).tolist())
    if len(labels) == 1:
        return 0 if y_true[0] == 0 else 1
    precision, recall, _ = precision_recall_curve(y_true, y_predict)
    recall = recall.astype(np.float32)
    for i in range(1, len(precision)):
        precision[i] = max(precision[i - 1], precision[i])
    return np.mean(precision[np.where(np.diff(recall))])


def ap_from_tuple(y_true, y_predict):
    """compute_ap_from_tuple: the prediction cut or zero-padded to the number of clips, then get_ap."""
    y_predict = np.asarray(y_predict, dtype=float)
    n = len(y_true)
    if len(y_predict) >= n:
        y = y_predict[:n]
    else:
        y = np.zeros(n)
        y[:len(y_predict)] = y_predict
    return get_ap(y_true, y)


def gt_scores(gt):
    """mk_gt_scores: [int(duration / 2), 3] scores, zero outside relevant_clip_ids."""
    full = np.zeros((int(gt["duration"] / 2), 3))
    full[np.array(gt["relevant_clip_ids"])] = np.array(gt["saliency_scores"])
    return full


# ---------------------------------------------------------------- per-query arrays in the device layout
def per_query(submission, ground_truth, mr=True, hl=True):
    """Per-query values in submission order, laid out like the device outputs:
    ap [4,Q,10], iou_r1 [4,Q], iou_r5 [4,Q], kept [4,Q] bool (ranges short, middle, long, full; rows where kept is False are 0),
    hl_ap [3,Q,3], hit [3,Q,3] (min score 2 / 3 / 4 x annotator)."""
    gt_by = {d["qid"]: d for d in ground_truth}
    Q = len(submission)
    out = {}
    if mr:
        ap, r1, r5 = np.zeros((4, Q, len(MR_THDS))), np.zeros((4, Q)), np.zeros((4, Q))
        kept = np.zeros((4, Q), dtype=bool)
        for q, d in enumerate(submission):
            rows = d["pred_relevant_windows"][:MAX_PRED]
            for r, (_, lo, hi) in enumerate(RANGES):
                g = gt_by[d["qid"]]["relevant_windows"]
                if r < 3:
                    g = windows_in_range(g, lo, hi)
                if not g:
                    continue
                kept[r, q] = True
                ap[r, q] = ap_detection(g, rows)
                r1[r, q] = r1_iou(rows, g)
                r5[r, q] = r5_iou(rows, g)
        out.update(ap=ap, iou_r1=r1, iou_r5=r5, kept=kept)
    if hl:
        hap, hit = np.zeros((3, Q, 3)), np.zeros((3, Q, 3))
        for q, d in enumerate(submission):
            full = gt_scores(gt_by[d["qid"]])
            top = int(np.argmax(d["pred_saliency_scores"]))
            for lv, (m, _) in enumerate(HL_LEVELS):
                binary = (full >= m).astype(float)
                if top < len(binary):
                    hit[lv, q] = binary[top]
                for a in range(3):
                    hap[lv, q, a] = ap_from_tuple(binary[:, a], d["pred_saliency_scores"])
        out.update(hl_ap=hap, hit=hit)
    return out


# ---------------------------------------------------------------- eval_submission
def _fmt(v):
    return float(f"{v:.2f}")


def mr_metrics(pq):
    """The per-range metric dicts from per-query arrays (empty range -> the full set's rows)."""
    res = {}
    for r, (name, _, _) in enumerate(RANGES):
        rows = pq["kept"][r] if pq["kept"][r].any() else pq["kept"][3]
        src = r if pq["kept"][r].any() else 3
        ap_thds = pq["ap"][src][rows].mean(0)
        mr_ap = dict(zip([str(e) for e in MR_THDS], ap_thds))
        mr_ap["average"] = np.mean(ap_thds)
        mr_ap = {k: _fmt(100 * v) for k, v in mr_ap.items()}
        i1, i5 = pq["iou_r1"][src][rows], pq["iou_r5"][src][rows]
        res[name] = {"MR-mIoU": _fmt(np.mean(i1) * 100), "MR-mAP": mr_ap,
                     "MR-R1": {str(t): _fmt(np.mean(i1 >= t) * 100) for t in R_THDS},
                     "MR-R5": {str(t): _fmt(np.mean(i5 >= t) * 100) for t in R_THDS}}
    return res


def hl_metrics(pq):
    res = {}
    for lv, (_, name) in enumerate(HL_LEVELS):
        res[f"HL-min-{name}"] = {"HL-mAP": _fmt(100 * np.mean(pq["hl_ap"][lv])),
                                 "HL-Hit1": _fmt(100 * np.mean(np.max(pq["hit"][lv], 1)))}
    return res


MR_BRIEF = (("MR-full-mAP-key", "full", "MR-mAP", "average"), ("MR-full-mAP@0.5-key", "full", "MR-mAP", "0.5"),
            ("MR-full-mAP@0.75-key", "full", "MR-mAP", "0.75"), ("MR-short-mAP", "short", "MR-mAP", "average"),
            ("MR-middle-mAP", "middle", "MR-mAP", "average"), ("MR-long-mAP", "long", "MR-mAP", "average"),
            ("MR-short-mIoU", "short", "MR-mIoU", None), ("MR-middle-mIoU", "middle", "MR-mIoU", None),
            ("MR-long-mIoU", "long", "MR-mIoU", None), ("MR-full-mIoU-key", "full", "MR-mIoU", None),
            ("MR-full-R1@0.3-key", "full", "MR-R1", "0.3"), ("MR-full-R1@0.5-key", "full", "MR-R1", "0.5"),
            ("MR-full-R1@0.7-key", "full", "MR-R1", "0.7"), ("MR-full-R5@0.3-key", "full", "MR-R5", "0.3"),
            ("MR-full-R5@0.5-key", "full", "MR-R5", "0.5"), ("MR-full-R5@0.7-key", "full", "MR-R5", "0.7"))


def eval_submission(submission, ground_truth, verbose=True, match_number=True):
    """eval/eval.py eval_submission, serially.  Raises AssertionError on a qid mismatch under match_number, like the reference."""
    pred_qids = {d["qid"] for d in submission}
    gt_qids = {d["qid"] for d in ground_truth}
    if match_number:
        if pred_qids != gt_qids:
            raise AssertionError("qids in ground_truth and submission must match")
    else:
        shared = pred_qids & gt_qids
        submission = [d for d in submission if d["qid"] in shared]
        ground_truth = [d for d in ground_truth if d["qid"] in shared]
    do_mr = "pred_relevant_windows" in submission[0]
    do_hl = ("pred_saliency_scores" in submission[0] and "saliency_scores" in ground_truth[0]
             and isinstance(ground_truth[0]["saliency_scores"], list))
    pq = per_query(submission, ground_truth, mr=do_mr, hl=do_hl)
    metrics, brief = {}, OrderedDict()
    if do_mr:
        mr = mr_metrics(pq)
        metrics.update(mr)
        brief.update(sorted((k, mr[rng][m] if sub is None else mr[rng][m][sub]) for k, rng, m, sub in MR_BRIEF))
    if do_hl:
        hl = hl_metrics(pq)
        metrics.update(hl)
        for k, v in hl.items():
            for sub_k, x in v.items():
                brief[f"{k}-{sub_k.split('-')[1]}"] = x
        brief["HL-min-VeryGood-mAP-key"] = brief.pop("HL-min-VeryGood-mAP")
        brief["HL-min-VeryGood-Hit1-key"] = brief.pop("HL-min-VeryGood-Hit1")
    final = OrderedDict()
    final["brief"] = brief
    final.update(sorted(metrics.items()))
    return final
