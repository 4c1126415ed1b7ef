"""fp64 reference of the criterion kernels (csrc/loss.cu) and the edge batches that drive them.

mr_reference restates SetCriterion of the reference (model/univtg.py:195-282, utils/span_utils.py:46-122) with the reference's own
functions -- F.smooth_l1_loss, the diagonal of generalized_temporal_iou with torch.maximum / minimum / clamp (so that ties split
the gradient as torch does), F.binary_cross_entropy with weight=, sim_matrix, F.cosine_similarity, F.log_softmax -- in fp64 from
exactly the fp32 values a kernel receives.  src_spans = timestamp + pred_spans is formed in fp32 first, as the reference does,
so the same comparisons decide the same branches; tau is float32(0.07) and the mask term log(2^-149), the fp32 value of the
reference's 1e-45.  torch's BCE backward clamps p (1 - p) at float32(1e-12) in every dtype, as the kernels do.  qfvs_reference does the same for model/univtg_qfvs.py:215-261, 358-377.

tests/test_loss_ops_cpu.py pins both to tests/golden/reference_loss_edges.npz (the unmodified reference, fp32, on CPU);
tests/test_loss_ops_gpu.py compares the kernels with them under the bounds of mr_bounds / qfvs_bounds (derivation in its docstring).
"""
import math

import torch
import torch.nn.functional as F

from tests.bounds import U, cfac

TAU = float(torch.tensor(0.07, dtype=torch.float32))
MASK_LOG = math.log(2.0 ** -149)
BCE_EPS32 = float(torch.tensor(1e-12, dtype=torch.float32))
TRAIN_W = (10.0, 1.0, 10.0, 0.1, 0.1)  # loss_b, loss_g, loss_f, loss_s_inter, loss_s_intra
LOSS_NAMES = ("loss_b", "loss_g", "loss_f", "loss_s_inter", "loss_s_intra")


# ================================================== edge batches ==================================================
def _dy(g, lo, hi, shape, q=512):
    """Dyadic values k / q in [lo, hi): sums and differences of them are exact in fp32."""
    return torch.randint(int(lo * q), int(hi * q), shape, generator=g).float() / q


def mr_case(B, Lv, d, seed, edges=(), eos=0.1):
    """A moment-retrieval batch as the loss kernels take it (fp32 / int64 CPU tensors).  Ragged timestamp_mask with gaps inside
    samples, dyadic spans and saliency scores (multiples of 2^-9 and 1/4, so ties are exact), cosines spread over [-1, 1].
    edges plants cases: giou (GIoU ties / touching / disjoint / nested spans, smooth-L1 at |d| = 0 and 1), bce (p in
    {0, 1, 2^-24, 1 - 2^-24} x y in {0, 1} x valid / masked), pos (positives at l = 0, Lv - 1, a masked clip, duplicates),
    sal_ties (clips scored exactly as the positive), and the degenerate sal_zero, no_pos, spanless, no_fg, no_valid."""
    g = torch.Generator().manual_seed(seed)
    n = B * Lv
    tmask = torch.zeros(B, Lv)
    for b in range(B):
        tmask[b, :int(torch.randint(max(1, Lv // 2), Lv + 1, (1,), generator=g))] = 1.0
        if Lv >= 8 and b % 3 == 1:  # a gap inside the sample
            j = int(torch.randint(1, Lv // 2, (1,), generator=g))
            tmask[b, j:j + 2] = 0.0
    window = torch.zeros(B, Lv)
    for b in range(B):
        valid = torch.nonzero(tmask[b]).flatten()
        s = int(valid[int(torch.randint(0, len(valid), (1,), generator=g))])
        window[b, s:s + max(1, Lv // 8)] = 1.0
    window *= tmask
    c = (torch.arange(Lv) % 256).float() / 32.0
    ts = torch.stack([c, c], -1).expand(B, Lv, 2).contiguous()
    ps = torch.stack([-_dy(g, 0, 2, (B, Lv)), _dy(g, 0, 2, (B, Lv))], -1)
    gt = torch.stack([c - _dy(g, 0, 2, (B, Lv)), c + _dy(g, 0, 2, (B, Lv))], -1)
    pl = torch.sigmoid(2.0 * torch.randn(B, Lv, generator=g))
    xt = torch.randn(B, d, generator=g)
    xv = torch.randn(B, Lv, d, generator=g) + (3.0 * torch.randn(B, Lv, 1, generator=g) / math.sqrt(d)) * xt[:, None, :] * 0.5
    sal = torch.randint(0, 8, (B, Lv), generator=g).float() / 4.0 * tmask
    pos = torch.empty(B, dtype=torch.int64)
    for b in range(B):
        valid = torch.nonzero(tmask[b]).flatten()
        pos[b] = valid[int(torch.randint(0, len(valid), (1,), generator=g))]
    flat = lambda t: t.view(n, *t.shape[2:])  # noqa: E731
    if "giou" in edges:  # (pred start offset a, end offset b) -> gt from the resulting src span (s1, e1)
        plants = [("tie_s", lambda s1, e1: (s1, e1 + 0.25)), ("tie_e", lambda s1, e1: (s1 - 0.25, e1)),
                  ("same", lambda s1, e1: (s1, e1)), ("touch_r", lambda s1, e1: (e1, e1 + 0.5)),
                  ("touch_l", lambda s1, e1: (s1 - 0.5, s1)), ("disjoint", lambda s1, e1: (e1 + 0.25, e1 + 1.0)),
                  ("inside", lambda s1, e1: (s1 + 0.25, e1 - 0.5)), ("around", lambda s1, e1: (s1 - 0.5, e1 + 0.75)),
                  ("sl1_one", lambda s1, e1: (s1 - 1.0, e1 + 1.0)), ("tie_s_inside", lambda s1, e1: (s1, e1 - 0.5))]
        for k, (_, f) in enumerate(plants[:n]):
            i = (k * 7) % n
            flat(tmask)[i] = 1.0
            flat(window)[i] = 1.0
            flat(ps)[i] = torch.tensor([-1.0, 1.0])
            s1, e1 = float(flat(ts)[i, 0]) - 1.0, float(flat(ts)[i, 1]) + 1.0
            flat(gt)[i] = torch.tensor(f(s1, e1))
    if "bce" in edges:
        vals = [0.0, 1.0, 2.0 ** -24, 1.0 - 2.0 ** -24]
        for k in range(min(16, n)):
            i = n - 1 - 3 * k if n > 48 else (n - 1 - k)
            flat(pl)[i] = vals[k % 4]
            flat(window)[i] = float((k // 4) % 2)
            flat(tmask)[i] = float(k // 8 == 0)
            if flat(window)[i] != 0:  # a foreground clip with a well-formed span
                flat(gt)[i] = flat(ts)[i] + torch.tensor([-0.5, 0.5])
    if "pos" in edges:
        pos[0] = 0
        tmask[0, 0] = 1.0
        if B > 1:
            pos[1] = Lv - 1
            tmask[1, Lv - 1] = 1.0
        if B > 2:
            pos[2] = Lv // 2
            tmask[2, Lv // 2] = 0.0  # positive at a masked clip
            window[2, Lv // 2] = 0.0
        for b in range(3, min(B, 6)):
            pos[b] = min(3, Lv - 1)  # duplicates across samples
            tmask[b, pos[b]] = 1.0
        if B > 7:
            pos[7] = 0  # duplicate of sample 0's positive
            tmask[7, 0] = 1.0
    if "sal_ties" in edges:
        for b in range(B):
            p = int(pos[b])
            sal[b, p] = 1.0
            for j in (p + 1, p - 2, p + 5):
                if 0 <= j < Lv:
                    sal[b, j] = 1.0
    if "sal_zero" in edges:
        sal.zero_()
    if "no_fg" in edges:
        window.zero_()
    if "no_valid" in edges:
        tmask.zero_()
    return {"pred_logits": pl, "pred_spans": ps, "vid_mem_proj": xv, "txt_mem_proj": xt,
            "timestamp": None if "spanless" in edges else ts, "timestamp_mask": tmask, "timestamp_window": window,
            "span_labels_nn": None if "spanless" in edges else gt, "saliency_scores": sal,
            "pos": None if "no_pos" in edges else pos, "eos_coef": float(eos)}


def qfvs_case(B, Lv, d, seed, keep="random", vmask_kept_zero=False, has_pos=1, targets="binary", rising=False):
    """A QFVS criterion input: mask_gt by pattern (all / none / alternating / one per 1024-wide chunk / random), targets
    (binary, all one, fractional or all zero), src_vid_mask 0 at some kept positions, z rising along each thread's chunks."""
    g = torch.Generator().manual_seed(seed)
    n = B * Lv
    if keep == "all":
        m = torch.ones(n, dtype=torch.bool)
    elif keep == "none":
        m = torch.zeros(n, dtype=torch.bool)
    elif keep == "alt":
        m = torch.arange(n) % 2 == 0
    elif keep == "chunk":
        m = torch.zeros(n, dtype=torch.bool)
        m[(torch.arange(0, n, 1024) + 517).clamp(max=n - 1)] = True
    else:
        m = torch.rand(n, generator=g) < 0.6
    xt = torch.randn(B, d, generator=g)
    xv = torch.randn(B, Lv, d, generator=g) + (3.0 * torch.randn(B, Lv, 1, generator=g) / math.sqrt(d)) * xt[:, None, :] * 0.5
    if rising:  # cos grows with the chunk index: every thread's running max moves and its sum is rescaled
        ramp = (torch.arange(n).float() // 1024 + 1.0).view(B, Lv, 1) * 0.6
        xv = torch.randn(B, Lv, d, generator=g) * 0.3 + ramp * xt[:, None, :]
    if targets == "zero":
        sal = torch.zeros(n)
    elif targets == "ones":
        sal = torch.ones(n)
    elif targets == "frac":
        sal = torch.randint(0, 5, (n,), generator=g).float() / 4.0
    else:
        sal = (torch.rand(n, generator=g) < 0.3).float()
    vmask = torch.ones(n)
    if vmask_kept_zero:  # at kept negatives: a masked positive's softmax entry underflows to 0 and the reference takes log(0)
        kept = torch.nonzero(m).flatten()
        neg = kept[sal[:len(kept)] == 0]
        vmask[neg[::3]] = 0.0
    pl = torch.sigmoid(2.0 * torch.randn(n, generator=g))
    return {"pred_logits": pl, "vid_mem_proj": xv, "txt_mem_proj": xt, "src_vid_mask": vmask, "mask_gt": m, "saliency_scores": sal,
            "has_pos": int(has_pos)}


# ================================================== references ==================================================
def _sim_matrix(a, b, eps=1e-8):
    a_n, b_n = a.norm(dim=1)[:, None], b.norm(dim=1)[:, None]
    return torch.mm(a / torch.max(a_n, eps * torch.ones_like(a_n)), (b / torch.max(b_n, eps * torch.ones_like(b_n))).t())


def _giou_diag(s, t):
    inter = (torch.minimum(s[:, 1], t[:, 1]) - torch.maximum(s[:, 0], t[:, 0])).clamp(min=0)
    union = (s[:, 1] - s[:, 0]) + (t[:, 1] - t[:, 0]) - inter
    enclose = (torch.maximum(s[:, 1], t[:, 1]) - torch.minimum(s[:, 0], t[:, 0])).clamp(min=0)
    return inter / union - (enclose - union) / enclose


def mr_losses(c, leaves):
    """The five losses (fp64 tensors) of an mr_case from fp64 leaves pred_logits, src_spans, vid_mem_proj, txt_mem_proj."""
    f64 = lambda t: t.double()  # noqa: E731
    tmask, window, sal = f64(c["timestamp_mask"]), f64(c["timestamp_window"]), f64(c["saliency_scores"])
    B, Lv = tmask.shape
    zero = torch.zeros((), dtype=torch.float64)
    out = {}
    if c["timestamp"] is not None:
        src, gt = leaves["src_spans"], f64(c["span_labels_nn"])
        fg = window.bool()
        out["loss_b"] = (F.smooth_l1_loss(src, gt, reduction="none") * window.unsqueeze(2)).sum() / fg.sum()
        out["loss_g"] = (1 - _giou_diag(src[fg], gt[fg])).mean()
    else:
        out["loss_b"] = out["loss_g"] = zero
    fg = window.bool()
    w = torch.zeros(B, Lv, dtype=torch.float64)
    w[tmask.bool()] = float(torch.tensor(c["eos_coef"], dtype=torch.float32))
    w[fg] = 1.0
    out["loss_f"] = (F.binary_cross_entropy(leaves["pred_logits"], fg.double(), weight=w, reduction="none") * tmask.bool()).sum() / tmask.bool().sum()
    if c["pos"] is None or float(sal.sum()) == 0.0:
        out["loss_s_inter"] = out["loss_s_intra"] = zero
        return out
    xv, xt = leaves["vid_mem_proj"], leaves["txt_mem_proj"]
    bi, pi = torch.arange(B), c["pos"]
    sim = _sim_matrix(xv[bi, pi], xt)
    out["loss_s_inter"] = -torch.diag(F.log_softmax(sim / TAU, dim=1)).sum() / B - torch.diag(F.log_softmax(sim.t() / TAU, dim=1)).sum() / B
    neg = sal < sal[bi, pi].unsqueeze(-1)
    neg[bi, pi] = True
    keep = neg * tmask.bool()
    sim_in = F.cosine_similarity(xv, xt.unsqueeze(1), dim=-1) + torch.log(keep.double() + 2.0 ** -149)
    li = F.log_softmax(sim_in / TAU, dim=1)[bi, pi]
    lj = F.log_softmax(sim_in.t() / TAU, dim=1)[pi, bi]
    out["loss_s_intra"] = -li.sum() / B - lj.sum() / B
    return out


def mr_leaves(c):
    """fp64 leaves; src_spans is timestamp + pred_spans rounded in fp32 (d src / d pred_spans = 1)."""
    ps = c["pred_spans"]
    src = (c["timestamp"] + ps) if c["timestamp"] is not None else ps
    return {"pred_logits": c["pred_logits"].double().requires_grad_(True), "src_spans": src.double().requires_grad_(True),
            "vid_mem_proj": c["vid_mem_proj"].double().requires_grad_(True),
            "txt_mem_proj": c["txt_mem_proj"].double().requires_grad_(True)}


def mr_reference(c, weights):
    """Losses and, for each weight vector w5, the gradients of sum_k w_k loss_k w.r.t. (pred_logits, pred_spans, vid_mem_proj,
    txt_mem_proj), fp64.  A NaN loss poisons the gradients exactly as autograd does (0 * inf)."""
    res = []
    losses = None
    for w in weights:
        lv = mr_leaves(c)
        L = mr_losses(c, lv)
        losses = L
        tot = sum(w[k] * L[n] for k, n in enumerate(LOSS_NAMES))
        names = ("pred_logits", "src_spans", "vid_mem_proj", "txt_mem_proj")
        grads = torch.autograd.grad(tot, [lv[k] for k in names], allow_unused=True)
        g = {k: (gr if gr is not None else torch.zeros_like(lv[k])) for k, gr in zip(names, grads)}
        g["pred_spans"] = g.pop("src_spans")
        res.append(g)
    return {k: v.detach() for k, v in losses.items()}, res


def qfvs_losses(c, pl, xv, xt):
    """SetCriterion.forward of model/univtg_qfvs.py (fp64) on one flattened criterion input."""
    keep = c["mask_gt"]
    count = int(keep.sum())
    t = c["saliency_scores"][:count].double()
    zero = torch.zeros((), dtype=torch.float64)
    if float(t.sum()) == 0.0:
        return {"loss_f": zero, "loss_s_intra": zero}
    out = {"loss_f": F.binary_cross_entropy(pl[keep], t, reduction="none").sum() / t.sum()}
    if not c["has_pos"]:
        out["loss_s_intra"] = zero
        return out
    B, Lv = xv.shape[:2]
    s = F.cosine_similarity(xv, xt.unsqueeze(1), dim=-1) + torch.log(c["src_vid_mask"].double().view(B, Lv) + 2.0 ** -149)
    soft = F.softmax(s.reshape(-1)[keep] / TAU, dim=0)
    lg = torch.log(soft[t > 0])
    out["loss_s_intra"] = -lg.sum() / len(lg)
    return out


def qfvs_reference(c, weights):
    res, losses = [], None
    for w in weights:
        pl = c["pred_logits"].double().requires_grad_(True)
        xv = c["vid_mem_proj"].double().requires_grad_(True)
        xt = c["txt_mem_proj"].double().requires_grad_(True)
        L = qfvs_losses(c, pl, xv, xt)
        losses = L
        tot = w[2] * L["loss_f"] + w[4] * L["loss_s_intra"]
        if tot.requires_grad:
            grads = torch.autograd.grad(tot, [pl, xv, xt], allow_unused=True)
        else:
            grads = (None, None, None)
        g = [gr if gr is not None else torch.zeros_like(x) for gr, x in zip(grads, (pl, xv, xt))]
        res.append({"pred_logits": g[0], "vid_mem_proj": g[1], "txt_mem_proj": g[2]})
    return {k: v.detach() for k, v in losses.items()}, res


# ================================================== bounds ==================================================
def _cos_parts(xv, xt):
    """cos(xv[..., :], xt) with its rounding scale S = sum |x_j y_j| / (|x||y|) + 2 |cos| and the norms."""
    vn = xv.norm(dim=-1).clamp_min(1e-8)
    tn = xt.norm(dim=-1).clamp_min(1e-8)
    cos = (xv * xt).sum(-1) / (vn * tn)
    S = (xv * xt).abs().sum(-1) / (vn * tn) + 2 * cos.abs()
    return cos, S, vn, tn


def _lse(z, dz, dim, K):
    """logsumexp and its bound: max dz + u sum_k p_k |z_k - max| (the rounded exp arguments) + c(K) u (1 + |lse| + |max|)."""
    lse = torch.logsumexp(z, dim)
    mx = z.amax(dim)
    p = torch.exp(z - lse.unsqueeze(dim))
    b = dz.amax(dim) + U * (p * (z - mx.unsqueeze(dim)).abs()).sum(dim) + cfac(K) * U * (1 + lse.abs() + mx.abs())
    return lse, b


def _soft(z, dz, lse, dlse):
    """p = exp(z - lse) and dp <= p (dz + dlse + u |z - lse| + 8u) (expf: 2 ulp)."""
    p = torch.exp(z - lse)
    return p, p * (dz + dlse + U * (z - lse).abs() + 8 * U)


def _vec_bounds(xv, xt, vn, tn, cos, dcos, gi, dgi, pos=None, gx=None, dgx=None, sim=None, dsim=None):
    """Bounds of d_vid_mem_proj / d_txt_mem_proj = sums coef * vec: c(K) u sum |coef||vec| + sum dcoef |vec|.
    gi [B, Lv]: weighted d loss / d cos_in; gx [B, B]: weighted d loss / d sim (rows b: positive clip of b, columns: text k)."""
    B, Lv, d = xv.shape
    rn = cfac(d) * U + 4 * U  # relative error of a norm and of one product / quotient by it
    avx, axt = xv.abs(), xt.abs()
    s1 = gi / (vn * tn[:, None])
    ds1 = dgi / (vn * tn[:, None]) + s1.abs() * 2 * rn
    s2 = gi * cos / vn ** 2
    ds2 = (dgi * cos.abs() + gi.abs() * dcos) / vn ** 2 + s2.abs() * 2 * rn
    S_v = s1.abs()[..., None] * axt[:, None, :] + s2.abs()[..., None] * avx
    E_v = ds1[..., None] * axt[:, None, :]
    pc = gi * cos
    S_c = (gi * cos).abs().sum(1)
    D_c = (dgi * cos.abs() + gi.abs() * dcos).sum(1)
    sc = gi / (vn * tn[:, None])
    dsc = dgi / (vn * tn[:, None]) + sc.abs() * 2 * rn
    S_t = torch.einsum("bl,bld->bd", sc.abs(), avx)
    E_t = torch.einsum("bl,bld->bd", dsc, avx)
    K_v, K_t = 3, Lv + 2
    if gx is not None:
        bi = torch.arange(B)
        un = vn[bi, pos]  # [B] norm of each sample's positive clip
        xp = xv[bi, pos]  # [B, d]
        c1 = gx / (un[:, None] * tn[None, :])
        dc1 = dgx / (un[:, None] * tn[None, :]) + c1.abs() * 2 * rn
        s2b = (gx * sim).sum(1) / un ** 2
        Ss2b = (gx * sim).abs().sum(1) / un ** 2
        ds2b = (dgx * sim.abs() + gx.abs() * dsim).sum(1) / un ** 2 + Ss2b * (cfac(B) * U + 2 * rn)
        S_pos = c1.abs() @ axt + Ss2b[:, None] * xp.abs()
        E_pos = dc1 @ axt + ds2b[:, None] * xp.abs()
        S_v[bi, pos] += S_pos
        E_v[bi, pos] += E_pos
        # the positive row's s2 = s2a + s2b is one fp32 value: its rounding and error multiply xv
        E_v[bi, pos] += (U * (s2[bi, pos] + s2b).abs())[:, None] * xp.abs()
        # text side: columns b of gx, rows k = positive clip of sample k
        sck = gx.t() / (un[None, :] * tn[:, None])  # [b, k]
        dsck = dgx.t() / (un[None, :] * tn[:, None]) + sck.abs() * 2 * rn
        S_t = S_t + sck.abs() @ xp.abs()
        E_t = E_t + dsck @ xp.abs()
        S_c = S_c + (gx * sim).abs().sum(0)
        D_c = D_c + (dgx * sim.abs() + gx.abs() * dsim).sum(0)
        K_v = B + 3
        K_t = Lv + B + 2
    E_v = E_v + ds2[..., None] * avx
    c2 = (pc.sum(1) if gx is None else pc.sum(1) + (gx * sim).sum(0)) / tn ** 2
    dc2 = D_c / tn ** 2 + S_c / tn ** 2 * (cfac(K_t) * U + 2 * rn)
    S_t = S_t + c2.abs()[:, None] * axt
    E_t = E_t + dc2[:, None] * axt
    return (S_v, K_v, E_v), (S_t, K_t, E_t)


def mr_bounds(c, w):
    """Per-output (S, K, extra) of the kernel results for weight vector w, and (S, K, extra) of each loss scalar."""
    f64 = lambda t: t.double()  # noqa: E731
    tmask, window, sal = f64(c["timestamp_mask"]), f64(c["timestamp_window"]), f64(c["saliency_scores"])
    B, Lv = tmask.shape
    fg = window != 0
    valid = tmask != 0
    n_fg, n_valid = float(fg.sum()), float(valid.sum())
    xv, xt = f64(c["vid_mem_proj"]), f64(c["txt_mem_proj"])
    d = xv.shape[-1]
    n = B * Lv
    lb = {}
    # ---- spans: few roundings of each elementwise formula (spans are dyadic: s1, e1, inter, union, enclose are exact) ----
    S_sp = torch.zeros(B, Lv, 2, dtype=torch.float64)
    if c["timestamp"] is not None:
        src = (c["timestamp"] + c["pred_spans"]).double()
        gt = f64(c["span_labels_nn"])
        dd = (src - gt)
        gb = torch.where(dd.abs() < 1, dd, dd.sign()) * window[..., None] / max(n_fg, 1.0)
        s1, e1, s2, e2 = src[..., 0], src[..., 1], gt[..., 0], gt[..., 1]
        inter = (torch.minimum(e1, e2) - torch.maximum(s1, s2)).clamp(min=0)
        uni = (e1 - s1) + (e2 - s2) - inter
        enc = (torch.maximum(e1, e2) - torch.minimum(s1, s2)).clamp(min=0)
        # |d giou / d (s1, e1)| in absolute values: |di| <= 1, |du| <= 2, |de| <= 1
        Sg = ((uni + 2 * inter) / uni ** 2 + (2 * enc + uni) / enc ** 2) * fg / max(n_fg, 1.0)
        S_sp = abs(w[0]) * gb.abs() + abs(w[1]) * torch.nan_to_num(Sg)[..., None].expand(B, Lv, 2)
        sl1 = torch.where(dd.abs() < 1, 0.5 * dd * dd, dd.abs() - 0.5) * window[..., None]
        lb["loss_b"] = (sl1.abs().sum() / n_fg if n_fg else 0.0, 2 * n, 0.0)
        gi_ = torch.where(fg, inter / uni - (enc - uni) / enc, torch.zeros_like(uni))
        Sgl = (inter / uni + (enc + uni) / enc) * fg
        lb["loss_g"] = ((torch.nan_to_num(Sgl).sum() + (1 - gi_).abs().sum()) / n_fg if n_fg else 0.0, n, 0.0)
    else:
        lb["loss_b"] = lb["loss_g"] = (0.0, 1, 0.0)
    spans = (S_sp, 8, None)
    # ---- BCE ----
    p = f64(c["pred_logits"])
    y = fg.double()
    wt = torch.where(fg, torch.ones_like(p), torch.where(valid, torch.full_like(p, float(torch.tensor(c["eos_coef"], dtype=torch.float32))), torch.zeros_like(p)))
    gf = wt * (p - y) / torch.clamp_min(p * (1 - p), BCE_EPS32) / max(n_valid, 1.0) * valid
    logits = (abs(w[2]) * gf.abs(), 8, None)
    lp, l1p = torch.log(p).clamp(min=-100), torch.log(1 - p).clamp(min=-100)
    Sf = (valid * wt * (y * (2 * lp.abs() + 1) + (1 - y) * (2 * l1p.abs() + 1))).sum() / max(n_valid, 1.0)
    lb["loss_f"] = (float(Sf), n, 0.0)
    # ---- saliency ----
    if c["pos"] is None or float(sal.sum()) == 0.0:
        z0 = torch.zeros_like(xv), torch.zeros_like(xt)
        lb["loss_s_inter"] = lb["loss_s_intra"] = (0.0, 1, 0.0)
        return lb, {"pred_logits": logits, "pred_spans": spans, "vid_mem_proj": (z0[0], 1, None), "txt_mem_proj": (z0[1], 1, None)}
    pos = c["pos"]
    bi = torch.arange(B)
    cos, Scos, vn, tn = _cos_parts(xv, xt[:, None, :])
    tn = tn.reshape(-1)
    dcos = cfac(d) * U * Scos
    sim, Ssim, _, _ = _cos_parts(xv[bi, pos][:, None, :], xt[None, :, :])
    dsim = cfac(d) * U * Ssim
    # inter
    zi = sim / TAU
    dzi = (dsim + 4 * U * sim.abs()) / TAU
    irow, dirow = _lse(zi, dzi, 1, B)
    icol, dicol = _lse(zi, dzi, 0, B)
    Pr, dPr = _soft(zi, dzi, irow[:, None], dirow[:, None])
    Pc, dPc = _soft(zi, dzi, icol[None, :], dicol[None, :])
    eye = torch.eye(B, dtype=torch.float64)
    g_sim = (Pr + Pc - 2 * eye) / (TAU * B)
    dg_sim = (dPr + dPc + 4 * U * (2 * eye + Pr + Pc)) / (TAU * B)
    dz_d = torch.diagonal(dzi)
    lb["loss_s_inter"] = (float((2 * torch.diagonal(zi).abs() + irow.abs() + icol.abs()).sum() / B), B,
                          float((2 * dz_d + dirow + dicol).sum() / B))
    # intra
    keep = ((sal < sal[bi, pos][:, None]) | (torch.arange(Lv)[None, :] == pos[:, None])) & valid
    m = torch.where(keep, torch.zeros_like(cos), torch.full_like(cos, MASK_LOG))
    z = (cos + m) / TAU
    dz = (dcos + 4 * U * (cos.abs() + m.abs())) / TAU
    rlse, drlse = _lse(z, dz, 1, Lv)
    zc = z[:, pos]  # [b', k]: column pos_k
    clse, dclse = _lse(zc, dz[:, pos], 0, B)
    Pr2, dPr2 = _soft(z, dz, rlse[:, None], drlse[:, None])
    Q = torch.zeros(B, Lv, dtype=torch.float64)
    dQ = torch.zeros(B, Lv, dtype=torch.float64)
    ndup = torch.zeros(Lv, dtype=torch.float64)
    for k in range(B):
        pk = int(pos[k])
        e, de = _soft(z[:, pk], dz[:, pk], clse[k], dclse[k])
        Q[:, pk] += e
        dQ[:, pk] += de
        ndup[pk] += 1
    dQ += (ndup[None, :] + 4) * U * Q
    ispos = torch.zeros(B, Lv, dtype=torch.float64)
    ispos[bi, pos] = 1.0
    g_cos = (Pr2 + Q - 2 * ispos) / (TAU * B)
    dg_cos = (dPr2 + dQ + 4 * U * (Pr2 + Q + 2 * ispos)) / (TAU * B)
    zp = z[bi, pos]
    lb["loss_s_intra"] = (float((2 * zp.abs() + rlse.abs() + clse.abs()).sum() / B), B,
                          float((2 * dz[bi, pos] + drlse + dclse).sum() / B))
    gi, dgi = w[4] * g_cos, abs(w[4]) * dg_cos + U * (w[4] * g_cos).abs()
    gx, dgx = w[3] * g_sim, abs(w[3]) * dg_sim + U * (w[3] * g_sim).abs()
    vb, tb = _vec_bounds(xv, xt, vn, tn, cos, dcos, gi, dgi, pos, gx, dgx, sim, dsim)
    return lb, {"pred_logits": logits, "pred_spans": spans, "vid_mem_proj": vb, "txt_mem_proj": tb}


def qfvs_bounds(c, w):
    xv, xt = c["vid_mem_proj"].double(), c["txt_mem_proj"].double()
    B, Lv, d = xv.shape
    keep = c["mask_gt"]
    count = int(keep.sum())
    t = torch.zeros(B * Lv, dtype=torch.float64)
    t[keep] = c["saliency_scores"][:count].double()
    sum_t = float(t.sum())
    p = c["pred_logits"].double()
    lb = {}
    if sum_t == 0.0:
        lb["loss_f"] = lb["loss_s_intra"] = (0.0, 1, 0.0)
        zero = (torch.zeros_like(p), 1, None)
        return lb, {"pred_logits": zero, "vid_mem_proj": (torch.zeros_like(xv), 1, None), "txt_mem_proj": (torch.zeros_like(xt), 1, None)}
    dsum = cfac(max(count, 1)) * U * float(t.abs().sum())
    gf = (p - t) / torch.clamp_min(p * (1 - p), BCE_EPS32) / sum_t * keep
    logits = (abs(w[2]) * gf.abs(), 8, abs(w[2]) * gf.abs() * dsum / sum_t)
    lp, l1p = torch.log(p).clamp(min=-100), torch.log(1 - p).clamp(min=-100)
    bce = -(t * lp + (1 - t) * l1p) * keep
    Sf = (keep * (t.abs() * (2 * lp.abs() + 1) + (1 - t).abs() * (2 * l1p.abs() + 1))).sum() / sum_t
    lb["loss_f"] = (float(Sf), count, float(bce.sum().abs() / sum_t * dsum / sum_t))
    cos, Scos, vn, tn = _cos_parts(xv, xt[:, None, :])
    tn = tn.reshape(-1)
    dcos = cfac(d) * U * Scos
    if not c["has_pos"]:
        lb["loss_s_intra"] = (0.0, 1, 0.0)
        gi = torch.zeros(B, Lv, dtype=torch.float64)
        dgi = gi.clone()
    else:
        vm = c["src_vid_mask"].double().view(B, Lv)
        m = torch.where(vm != 0, torch.zeros_like(cos), torch.full_like(cos, MASK_LOG))
        z = ((cos + m) / TAU).reshape(-1)
        dz = ((dcos + 4 * U * (cos.abs() + m.abs())) / TAU).reshape(-1)
        lse, dlse = _lse(z[keep], dz[keep], 0, count)
        P, dP = _soft(z, dz, lse, dlse)
        pos = (t > 0) & keep
        npos = float(pos.sum())
        gc = (P - pos.double() / npos) / TAU * keep
        dgc = (dP + 4 * U * (P + pos.double() / npos)) / TAU * keep
        lb["loss_s_intra"] = (float(lse.abs() + (z.abs() * pos).sum() / npos), count, float(dlse + (dz * pos).sum() / npos))
        gi = (w[4] * gc).view(B, Lv)
        dgi = (abs(w[4]) * dgc + U * (w[4] * gc).abs()).view(B, Lv)
    vb, tb = _vec_bounds(xv, xt, vn, tn, cos, dcos, gi, dgi)
    return lb, {"pred_logits": logits, "vid_mem_proj": vb, "txt_mem_proj": tb}
