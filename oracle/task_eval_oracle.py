"""TEST INFRASTRUCTURE ONLY - plain-Python restatement of the reference's TVSum / YouTube highlight evaluation and QFVS semantic
matching.

Only tests/ and tools/ may import this module; the product path (univtg_b200/metrics.py evaluate_hl -> univtg_eval_hl_topk,
univtg_b200/qfvs.py calculate_semantic_matching -> univtg_qfvs_match) never does.  It imports neither networkx nor
scikit-learn nor the reference.

Follows, in behaviour (not in code):
  * main/dataset.py:853-921  DatasetHL.evaluate: torch.argsort(score[0], descending=True) on the CPU, TVSum labels
    `anno[:, i] > median` (torch's lower median of the float32 column) cut to the first k, YouTube labels `match > 0` over the
    whole list, the AP recursion in Python floats, the means over videos and then annotators, round(mean, 5)
  * eval/qfvs.py:32-74       semantic_iou, the maximum-weight matching of the complete bipartite graph, P / R / F1

The matching optimum is computed exactly: a Hungarian method over fractions.Fraction weights |a & b| / |a | b|.  Its value is
the exact optimum of the rational weights; `s` sums the float64 weights of that assignment, which is what the reference's
networkx matching adds up (in its own order).
"""
from fractions import Fraction

import torch

TVSUM_ANNOTATORS = 20


def _ap(label):
    """The reference's recursion over one ranked 0 / 1 list (Python floats)."""
    if (num_gt := sum(label)) == 0:
        return 0
    hits = ap = rec = 0
    prc = 1
    for j, gt in enumerate(label):
        hits += gt
        _rec = hits / num_gt
        _prc = hits / (j + 1)
        ap += (_rec - rec) * (prc + _prc) / 2
        rec, prc = _rec, _prc
    return ap


def per_video_ap(dset_name, labels, blob, k=5):
    """[[AP of each annotator] per video]: labels[idx] is video idx's `anno` (TVSum) or `match` (YouTube), blob the score list."""
    out = []
    for idx, score in enumerate(blob):
        inds = torch.argsort(score[0].cpu(), descending=True)
        if dset_name == "tvsum":
            row = []
            for i in range(TVSUM_ANNOTATORS):
                label = torch.Tensor(labels[idx])[:, i]
                label = torch.where(label > label.median(), 1.0, .0)
                row.append(_ap(label[inds].tolist()[:k]))
            out.append(row)
        elif dset_name == "youtube":
            out.append([_ap(torch.Tensor([1 if s > 0 else 0 for s in labels[idx]])[inds].tolist())])
        else:
            raise NotImplementedError(dset_name)
    return out


def evaluate_hl(dset_name, labels, blob, k=5):
    """{'mAP': ...} of DatasetHL.evaluate."""
    aps = per_video_ap(dset_name, labels, blob, k)
    if dset_name == "tvsum":
        collected = []
        for i in range(TVSUM_ANNOTATORS):
            video_ap = [row[i] for row in aps]
            collected.append(sum(video_ap) / len(video_ap))
    else:
        collected = [row[0] for row in aps]
    mean_ap = sum(collected) / len(collected)
    return dict(mAP=round(mean_ap, 5))


def _bits(row):
    return {c for c, x in enumerate(row) if x}


def semantic_iou(a, b):
    """Exact |a & b| / |a | b| of two tag rows (0 when both are empty)."""
    a, b = _bits(a), _bits(b)
    u = len(a | b)
    return Fraction(len(a & b), u) if u else Fraction(0)


def max_weight_assignment(w):
    """Hungarian method (shortest augmenting paths, exact arithmetic) maximising sum w[i][col[i]] over a rectangular matrix of
    Fractions -> (optimum, col).  Every row of the smaller side is matched; with weights >= 0 that is a maximum-weight
    matching."""
    n, m = len(w), len(w[0])
    if n > m:
        opt, col = max_weight_assignment([list(r) for r in zip(*w)])
        row = [None] * n
        for j, i in enumerate(col):
            row[i] = j
        return opt, row
    inf = None  # no finite bound needed: None stands for +infinity
    u = [Fraction(0)] * (n + 1)
    v = [Fraction(0)] * (m + 1)
    p = [0] * (m + 1)  # p[j]: 1-based row on column j, 0 = free; column 0 is the virtual one
    way = [0] * (m + 1)
    for i in range(1, n + 1):
        p[0] = i
        j0 = 0
        minv = [inf] * (m + 1)
        used = [False] * (m + 1)
        while True:
            used[j0] = True
            i0, delta, j1 = p[j0], inf, 0
            for j in range(1, m + 1):
                if not used[j]:
                    cur = -w[i0 - 1][j - 1] - u[i0] - v[j]
                    if minv[j] is inf or cur < minv[j]:
                        minv[j], way[j] = cur, j0
                    if delta is inf or minv[j] < delta:
                        delta, j1 = minv[j], j
            for j in range(m + 1):
                if used[j]:
                    u[p[j]] += delta
                    v[j] -= delta
                else:
                    minv[j] -= delta
            j0 = j1
            if p[j0] == 0:
                break
        while j0:
            j1 = way[j0]
            p[j0] = p[j1]
            j0 = j1
    col = [None] * n
    for j in range(1, m + 1):
        if p[j]:
            col[p[j] - 1] = j - 1
    return sum(w[i][col[i]] for i in range(n)), col


def semantic_matching(machine_summary, gt_summary, shots_tag):
    """-> (exact optimum as a Fraction, s = float64 sum of the matched weights, p, r, f1) of calculate_semantic_matching."""
    import numpy as np

    a, b = np.asarray(shots_tag)[machine_summary], np.asarray(shots_tag)[gt_summary]
    w = [[semantic_iou(x, y) for y in b] for x in a]
    opt, col = max_weight_assignment(w)
    s = np.float64(0)
    for i, j in enumerate(col):
        if j is not None:
            s += np.float64(float(w[i][j]))
    p = s / a.shape[0]
    r = s / b.shape[0]
    with np.errstate(invalid="ignore"):
        f1 = 2 * p * r / (p + r)
    return opt, s, p, r, f1
