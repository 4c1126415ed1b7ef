"""Operator-level fp64 parity of the criterion kernels (csrc/loss.cu: loss_cos, loss_finish, qfvs_loss, loss_bwd_small / vid / txt),
driven through univtg_loss_forward / univtg_loss_backward and univtg_qfvs_loss_forward / univtg_qfvs_loss_backward.

Method: each batch of tests/loss_ref.py (mr_case / qfvs_case: ragged masks with gaps, dyadic spans and saliency scores so that
ties are exact in fp32, planted edges) runs the forward once and the backward six times: with each one-hot w5, which isolates one
loss's gradient, and with the training weights (10, 1, 10, 0.1, 0.1).  Every output buffer is NaN-filled first.  The reference is
fp64 autograd through a restatement of the reference's SetCriterion from the fp32 inputs the kernels got (tests/loss_ref.py,
pinned to the reference by tests/test_loss_ops_cpu.py).  NaN must appear exactly where the reference has NaN (no foreground clip:
loss_b, loss_g and, through 0 * inf, the span gradient; no valid clip: loss_f and the logit gradient).

Bounds (tests/bounds.py): |got - ref| <= c(K) 2^-24 S + E elementwise, c(K) = 4 (ceil(log2 K) + 1), E first-order propagated:
  cosine              S = sum_j |u_j v_j| / (|u||v|) + 2 |cos|, K = d
  z = (cos + m) / tau dz = (dcos + 4 2^-24 (|cos| + |m|)) / tau, m = 0 or log 2^-149
  logsumexp (K terms) dlse = max dz + 2^-24 sum_k p_k |z_k - max z| + c(K) 2^-24 (1 + |lse| + |max z|)
  softmax entries     dp = p (dz + dlse + 2^-24 |z - lse| + 8 2^-24)   (expf: 2 ulp)
  g_sim / g_cos_in    sums of those entries (plus 2 at the positive): d = sum dp + 4 2^-24 sum |terms|, over tau B
  loss_s_*            S = sum |2 z_pos| + |lse_row| + |lse_col| over B, K = B; E = the same sum of the d's
  d_vid / d_txt       sums coef * vec: S = sum |coef||vec|, K = B + 3 (vid) or Lv + B + 2 (txt); E = sum dcoef |vec|, where
                      dcoef carries the weight, dg and the norms' relative error c(d) 2^-24
  spans               dyadic, so s1, e1, inter, union, enclose are exact: a few roundings of smooth-L1' w / n_fg and of
                      d GIoU / d(s, e) = (di u - i du) / u^2 + (du e - u de) / e^2 with S = (u + 2 i) / u^2 + (2 e + u) / e^2, K = 8
  BCE                 S = |w (p - y) / max(p (1 - p), 1e-12) / n|, K = 8; loss_f S = sum w (2 |log| + 1) / n (logf 1 ulp, and
                      the rounding of 1 - p), K = N
  QFVS                as above with the softmax over the kept positions; sum(t) adds c(count) 2^-24 sum |t| / sum t
The block-wide sums of loss_finish / qfvs_loss add at most ceil(N / 1024) + 5 + 32 terms in sequence, which c(N) covers for every N
used here.  Entries whose reference is exactly zero (masked BCE, background span gradients, the no-saliency branches, non-positive
clips' inter terms) have S = 0 and must be exactly zero.  The module prints the worst |got - ref| / bound per family and the
coverage of shapes and edges (pytest -s).
"""
import ctypes

import pytest
import torch

from tests import loss_ref as R
from tests.bounds import check, report_fixture
from univtg_b200 import _lib

pytestmark = pytest.mark.gpu

_SEEN = {"mr_shape": set(), "mr_edge": set(), "qfvs_n": set(), "qfvs_keep": set(), "qfvs_case": set()}
_report = report_fixture(_SEEN)
ONE_HOT = [tuple(float(i == k) for i in range(5)) for k in range(5)]
WEIGHTS = ONE_HOT + [R.TRAIN_W]
WNAME = list(R.LOSS_NAMES) + ["train"]


def lib():
    return _lib.load_library()


def P(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def cu(t):
    return None if t is None else t.cuda().contiguous()


def check_nan(fam, name, got, ref, S, K, extra=None):
    """check() on the entries where the reference is finite; NaN exactly where the reference is NaN."""
    got = got.double().cpu()
    isn = torch.isnan(ref)
    assert torch.equal(torch.isnan(got), isn), f"{fam}/{name}: NaN at {int(torch.isnan(got).sum())} entries, reference {int(isn.sum())}"
    f = ~isn
    if not f.any():
        return
    S = torch.nan_to_num(S.double(), nan=0.0) if torch.is_tensor(S) else torch.full_like(ref, float(S))
    e = None if extra is None else (torch.nan_to_num(extra.double(), nan=0.0) if torch.is_tensor(extra) else torch.full_like(ref, float(extra)))
    check(fam, name, got[f], ref[f], S[f], K, extra=None if e is None else e[f])


def check_losses(tag, got, ref, lb):
    for k, n in enumerate(R.LOSS_NAMES):
        S, K, E = lb[n]
        check_nan("loss scalars", f"{tag}/{n}", got[k:k + 1], ref[n].double().reshape(1), torch.tensor([float(S)]), K,
                  torch.tensor([float(E)]))


# ================================================== moment retrieval ==================================================
# (id, B, Lv, d, edges, eos_coef)
MR_CASES = [
    ("b1_l1", 1, 1, 64, ("pos", "sal_ties"), 0.1),
    ("b2", 2, 75, 64, ("giou", "bce", "pos", "sal_ties"), 0.1),
    ("b4_d320_eos05", 4, 75, 320, ("giou", "bce", "pos", "sal_ties"), 0.5),
    ("b32_d1024", 32, 75, 1024, ("giou", "bce", "pos", "sal_ties"), 0.1),
    ("b33_d192", 33, 40, 192, ("giou", "bce", "pos", "sal_ties"), 0.1),
    ("b64_l150", 64, 150, 256, ("giou", "bce", "pos"), 0.1),
    ("b256", 256, 75, 64, ("giou", "bce", "pos", "sal_ties"), 0.1),
    ("l1100", 3, 1100, 128, ("giou", "bce", "pos", "sal_ties"), 0.5),
    ("d3072", 8, 75, 3072, ("giou", "pos", "sal_ties"), 0.1),
    ("sal_zero", 4, 75, 64, ("sal_zero", "bce"), 0.1),
    ("no_pos", 4, 75, 64, ("no_pos", "giou"), 0.1),
    ("spanless", 4, 75, 64, ("spanless", "bce", "pos"), 0.1),
    ("no_fg", 33, 40, 64, ("no_fg", "pos"), 0.1),
    ("no_valid", 4, 75, 64, ("no_valid", "pos"), 0.1),
]


def run_mr(c):
    B, Lv = c["timestamp_mask"].shape
    d = c["vid_mem_proj"].shape[-1]
    g = {k: cu(v) for k, v in c.items() if torch.is_tensor(v)}
    scratch = torch.full((lib().univtg_loss_scratch_bytes(B, Lv),), 0xFF, dtype=torch.uint8, device="cuda")
    losses = nan(5)
    _lib.check(lib().univtg_loss_forward(P(g["pred_logits"]), P(g["pred_spans"]), P(g["vid_mem_proj"]), P(g["txt_mem_proj"]),
                                         P(g.get("timestamp")), P(g["timestamp_mask"]), P(g["timestamp_window"]),
                                         P(g.get("span_labels_nn")), P(g["saliency_scores"]), P(g.get("pos")), B, Lv, d,
                                         c["eos_coef"], R.TAU, P(losses), P(scratch), None), "univtg_loss_forward")
    outs = []
    for w in WEIGHTS:
        w5 = torch.tensor(w, dtype=torch.float32, device="cuda")
        o = {"pred_logits": nan(B, Lv), "pred_spans": nan(B, Lv, 2), "vid_mem_proj": nan(B, Lv, d), "txt_mem_proj": nan(B, d)}
        _lib.check(lib().univtg_loss_backward(P(w5), P(g["vid_mem_proj"]), P(g["txt_mem_proj"]), P(g.get("pos")), B, Lv, d,
                                              P(scratch), P(o["pred_logits"]), P(o["pred_spans"]), P(o["vid_mem_proj"]),
                                              P(o["txt_mem_proj"]), None), "univtg_loss_backward")
        outs.append(o)
    torch.cuda.synchronize()
    return losses.cpu(), outs


FAM = {"pred_logits": "BCE d_logits", "pred_spans": "spans d_spans", "vid_mem_proj": "d_vid_mem_proj", "txt_mem_proj": "d_txt_mem_proj"}


@pytest.mark.parametrize("cid,B,Lv,d,edges,eos", MR_CASES, ids=[c[0] for c in MR_CASES])
def test_mr_criterion(cid, B, Lv, d, edges, eos):
    c = R.mr_case(B, Lv, d, 700 + B + Lv + d, edges, eos)
    losses, outs = run_mr(c)
    ref_l, ref_g = R.mr_reference(c, WEIGHTS)
    lb, _ = R.mr_bounds(c, R.TRAIN_W)
    check_losses(cid, losses, ref_l, lb)
    for w, wn, o, rg in zip(WEIGHTS, WNAME, outs, ref_g):
        _, ob = R.mr_bounds(c, w)
        for k, fam in FAM.items():
            S, K, E = ob[k]
            check_nan(fam, f"{cid}/{wn}", o[k], rg[k], S, K, E)
    if c["pos"] is None or float(c["saliency_scores"].sum()) == 0.0:
        for o in outs:  # the no-saliency branch writes exact zeros over the NaN fill
            assert (o["vid_mem_proj"] == 0).all() and (o["txt_mem_proj"] == 0).all()
    if "no_fg" in edges:
        assert torch.isnan(losses[:2]).all() and torch.isfinite(losses[2:]).all()
        for o in outs:
            assert torch.isfinite(o["pred_logits"]).all() and torch.isfinite(o["vid_mem_proj"]).all()
    if "no_valid" in edges:
        assert torch.isnan(losses[2]) and torch.isfinite(losses[[0, 1, 3, 4]]).all()
    _SEEN["mr_shape"].add(f"{B}x{Lv}x{d}")
    _SEEN["mr_edge"].update(edges)
    _SEEN["mr_edge"].add(f"eos{eos}")


def test_mr_edges_are_planted():
    """The planted cases are in the batches the criterion test runs (ties exact in fp32, positives where they should be)."""
    c = R.mr_case(33, 40, 192, 700 + 33 + 40 + 192, ("giou", "bce", "pos", "sal_ties"), 0.1)
    src = c["timestamp"] + c["pred_spans"]
    gt = c["span_labels_nn"]
    fg = c["timestamp_window"] != 0
    assert ((src[..., 0] == gt[..., 0]) & fg).any() and ((src[..., 1] == gt[..., 1]) & fg).any()
    inter = torch.minimum(src[..., 1], gt[..., 1]) - torch.maximum(src[..., 0], gt[..., 0])
    assert ((inter == 0) & fg).any() and ((inter < 0) & fg).any()
    assert (((src - gt).abs() == 1.0) & fg[..., None]).any()
    p = c["pred_logits"]
    for v in (0.0, 1.0, 2.0 ** -24, 1.0 - 2.0 ** -24):
        for y in (0, 1):
            for valid in (0, 1):
                assert ((p == v) & (fg == bool(y)) & ((c["timestamp_mask"] != 0) == bool(valid))).any(), (v, y, valid)
    pos = c["pos"]
    assert pos[0] == 0 and pos[1] == 39 and c["timestamp_mask"][2, int(pos[2])] == 0 and len(set(pos.tolist())) < 33
    sal = c["saliency_scores"]
    bi = torch.arange(33)
    tie = (sal == sal[bi, pos][:, None]) & (torch.arange(40)[None, :] != pos[:, None]) & (c["timestamp_mask"] != 0)
    assert tie.any()
    tm = c["timestamp_mask"]
    assert any(((tm[b, 1:] - tm[b, :-1]) > 0).any() for b in range(33))  # a gap inside a sample, not only tail padding


# ================================================== QFVS ==================================================
# (id, B, Lv, d, keep pattern, options)
QF_CASES = [
    ("n1", 1, 1, 64, "all", {}),
    ("n1023_alt", 3, 341, 64, "alt", dict(vmask_kept_zero=True)),
    ("n1024_all", 4, 256, 192, "all", dict(rising=True)),
    ("n1025_chunk", 5, 205, 64, "chunk", {}),
    ("n3079_random", 1, 3079, 64, "random", dict(rising=True, vmask_kept_zero=True, targets="frac")),
    ("n3079_all_frac", 1, 3079, 128, "all", dict(targets="frac")),
    ("n3079_chunk", 1, 3079, 64, "chunk", dict(targets="ones")),
    ("n1025_none", 5, 205, 64, "none", {}),
    ("n1024_nopos", 4, 256, 64, "random", dict(has_pos=0)),
    ("n1023_zero_t", 3, 341, 64, "random", dict(targets="zero")),
]


def run_qfvs(c):
    B, Lv, d = c["vid_mem_proj"].shape
    g = {k: cu(v) for k, v in c.items() if torch.is_tensor(v)}
    mask = g["mask_gt"].to(torch.uint8)
    scratch = torch.full((lib().univtg_loss_scratch_bytes(B, Lv),), 0xFF, dtype=torch.uint8, device="cuda")
    losses = nan(5)
    _lib.check(lib().univtg_qfvs_loss_forward(P(g["pred_logits"]), P(g["vid_mem_proj"]), P(g["txt_mem_proj"]), P(g["src_vid_mask"]),
                                              P(mask), P(g["saliency_scores"]), c["has_pos"], B, Lv, d, R.TAU, P(losses), P(scratch),
                                              None), "univtg_qfvs_loss_forward")
    outs = []
    for w in WEIGHTS:
        w5 = torch.tensor(w, dtype=torch.float32, device="cuda")
        o = {"pred_logits": nan(B * Lv), "vid_mem_proj": nan(B, Lv, d), "txt_mem_proj": nan(B, d)}
        _lib.check(lib().univtg_qfvs_loss_backward(P(w5), P(g["vid_mem_proj"]), P(g["txt_mem_proj"]), B, Lv, d, P(scratch),
                                                   P(o["pred_logits"]), P(o["vid_mem_proj"]), P(o["txt_mem_proj"]), None),
                   "univtg_qfvs_loss_backward")
        outs.append(o)
    torch.cuda.synchronize()
    return losses.cpu(), outs


@pytest.mark.parametrize("cid,B,Lv,d,keep,opt", QF_CASES, ids=[c[0] for c in QF_CASES])
def test_qfvs_criterion(cid, B, Lv, d, keep, opt):
    c = R.qfvs_case(B, Lv, d, 900 + B * Lv + d, keep=keep, **opt)
    losses, outs = run_qfvs(c)
    ref_l, ref_g = R.qfvs_reference(c, WEIGHTS)
    lb, _ = R.qfvs_bounds(c, R.TRAIN_W)
    for k in (0, 1, 3):
        assert losses[k] == 0.0, (cid, k)
    for k, n in ((2, "loss_f"), (4, "loss_s_intra")):
        S, K, E = lb[n]
        check_nan("loss scalars", f"qfvs {cid}/{n}", losses[k:k + 1], ref_l[n].double().reshape(1), torch.tensor([float(S)]), K,
                  torch.tensor([float(E)]))
    for w, wn, o, rg in zip(WEIGHTS, WNAME, outs, ref_g):
        _, ob = R.qfvs_bounds(c, w)
        for k, fam in (("pred_logits", "qfvs d_logits"), ("vid_mem_proj", "qfvs d_vid_mem_proj"), ("txt_mem_proj", "qfvs d_txt_mem_proj")):
            S, K, E = ob[k]
            check_nan(fam, f"{cid}/{wn}", o[k], rg[k].reshape(o[k].shape), S, K, E)
    _SEEN["qfvs_n"].add(B * Lv)
    _SEEN["qfvs_keep"].add(keep)
    _SEEN["qfvs_case"].update(f"{k}={v}" for k, v in opt.items())


def test_coverage_is_complete():
    """Runs last in the module: every shape and edge the parametrized cases promise has run."""
    want_mr = {f"{B}x{Lv}x{d}" for _, B, Lv, d, _, _ in MR_CASES}
    want_edges = {"giou", "bce", "pos", "sal_ties", "sal_zero", "no_pos", "spanless", "no_fg", "no_valid", "eos0.1", "eos0.5"}
    if len(_SEEN["mr_shape"]) and len(_SEEN["qfvs_n"]):
        assert _SEEN["mr_shape"] == want_mr and want_edges <= _SEEN["mr_edge"]
        assert {1, 1023, 1024, 1025, 3079} == _SEEN["qfvs_n"]
        assert {"all", "none", "alt", "chunk", "random"} == _SEEN["qfvs_keep"]
    else:
        pytest.skip("run the whole module")
