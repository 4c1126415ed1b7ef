"""Query-focused video summarisation (QFVS): the reference's `univtg_qfvs` model plugin (model/univtg_qfvs.py), which
main/train_qfvs.py and main/inference_qfvs.py load through the usual `model_id` lookup.

    from univtg_b200.qfvs import build_model
    model, criterion = build_model(args)
    loss_dict = criterion(outputs, targets, mask_GT)

The model is the MR/HL `Model` (the reference's QFVS model has the same parameters, state_dict keys and forward); only the
criterion differs.  Its losses run in the CUDA library (univtg_qfvs_loss_forward / univtg_qfvs_loss_backward) without a host
synchronisation, where the reference's masked_select, count slice and zero-sum branches synchronise four times per call.

calculate_semantic_matching (bottom of this module) is the drop-in for eval/qfvs.py's evaluation of one oracle summary.
"""
import numpy as np
import torch

from . import _lib
from .criterion import SetCriterion
from .losses import LossDict


class _QFVSLossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred_logits, vid_mem_proj, txt_mem_proj, vmask, mask_gt, sal, has_pos, temperature):
        lib = _lib.load_library()
        dev = pred_logits.device
        B, Lv, d = vid_mem_proj.shape
        with torch.cuda.device(dev):
            pl = pred_logits.detach().to(torch.float32).contiguous()
            xv = vid_mem_proj.detach().to(torch.float32).contiguous()
            xt = txt_mem_proj.detach().to(torch.float32).contiguous()
            scratch = torch.empty(lib.univtg_loss_scratch_bytes(B, Lv), dtype=torch.uint8, device=dev)
            losses = torch.zeros(5, device=dev)
            _lib.check(lib.univtg_qfvs_loss_forward(_lib.ptr(pl), _lib.ptr(xv), _lib.ptr(xt), _lib.ptr(vmask), _lib.ptr(mask_gt),
                                                    _lib.ptr(sal), int(has_pos), B, Lv, d, float(temperature), _lib.ptr(losses),
                                                    _lib.ptr(scratch), _lib.stream_ptr()), "univtg_qfvs_loss_forward")
        ctx.saved = (xv, xt, scratch, B, Lv, d)
        return losses

    @staticmethod
    def backward(ctx, g_losses):
        lib = _lib.load_library()
        xv, xt, scratch, B, Lv, d = ctx.saved
        dev = xv.device
        with torch.cuda.device(dev):
            w = g_losses.detach().to(torch.float32).contiguous()
            d_logits = torch.empty(B, Lv, 1, device=dev)
            d_xv = torch.empty(B, Lv, d, device=dev)
            d_xt = torch.empty(B, 1, d, device=dev)
            _lib.check(lib.univtg_qfvs_loss_backward(_lib.ptr(w), _lib.ptr(xv), _lib.ptr(xt), B, Lv, d, _lib.ptr(scratch),
                                                     _lib.ptr(d_logits), _lib.ptr(d_xv), _lib.ptr(d_xt), _lib.stream_ptr()),
                       "univtg_qfvs_loss_backward")
        return d_logits, d_xv, d_xt, None, None, None, None, None


class QFVSCriterion(SetCriterion):
    """SetCriterion of model/univtg_qfvs.py (:156-377) behind the same interface."""

    def forward(self, outputs, targets, mask_GT=None):
        """Returns the reference's loss dict for one forward over S segments of Lf frames (model/univtg_qfvs.py:358-377).

        outputs: the model's dict (pred_logits [S, Lf, 1], vid_mem_proj, txt_mem_proj, src_vid_mask).
        targets: saliency_scores [1, >= S*Lf] (row 0 pairs, in order, with the kept positions), optionally saliency_pos_labels.
        mask_GT: S*Lf bools (the reference passes [1, S*Lf]); flat position i of [S, Lf] is kept iff mask_GT is set there.

        Every entry is a tensor: where the reference returns the Python float 0. (loss_s_inter always; loss_f and loss_s_intra
        when the kept targets sum to 0; loss_s_intra without saliency_pos_labels) this returns a 0 tensor whose gradient is 0.
        The losses are differentiable w.r.t. pred_logits, vid_mem_proj and txt_mem_proj; loss_s_intra is computed from the
        latter two as the model computes saliency_scores, so it is the same function of them.

        Unlike the reference, outputs["pred_logits"], outputs["saliency_scores"] and targets["saliency_scores"] are left as
        they are instead of being replaced with their masked selections; neither QFVS loop reads them afterwards.

        Raises ValueError, before anything runs on the device, for a missing or mis-sized mask_GT, a target row shorter than
        S*Lf, and a loss list with 'spans' (dset_type mr / vlp: QFVS targets carry no timestamps)."""
        if "spans" in self.losses:
            raise ValueError("the QFVS criterion has no 'spans' loss (QFVS targets carry no timestamp): use dset_type 'vs' or 'hl'")
        if mask_GT is None:
            raise ValueError("the QFVS criterion needs mask_GT (the kept frames of the [S, Lf] segment grid)")
        pl = outputs["pred_logits"]
        xv, xt = outputs["vid_mem_proj"], outputs["txt_mem_proj"]
        B, Lv = pl.shape[:2]
        n = B * Lv
        if pl.numel() != n or tuple(xv.shape[:2]) != (B, Lv) or xt.numel() != B * xv.shape[2]:
            raise ValueError(f"outputs must be pred_logits [S, Lf, 1], vid_mem_proj [S, Lf, d], txt_mem_proj [S, 1, d]; got "
                             f"{list(pl.shape)}, {list(xv.shape)}, {list(xt.shape)}")
        if mask_GT.numel() != n:
            raise ValueError(f"mask_GT has {mask_GT.numel()} elements, the outputs {n} = {B} x {Lv} positions")
        vmask = outputs["src_vid_mask"]
        if vmask.numel() != n:
            raise ValueError(f"outputs['src_vid_mask'] has {vmask.numel()} elements, expected {n}")
        ts = targets["saliency_scores"]
        if ts.dim() != 2 or ts.shape[0] < 1 or ts.shape[1] < n:
            raise ValueError(f"targets['saliency_scores'] must be [1, >= {n}] (row 0 pairs with the kept positions), got "
                             f"{list(ts.shape)}")
        dev = pl.device
        if dev.type != "cuda":
            raise RuntimeError("univtg_b200: the criterion runs on CUDA tensors only (no CPU path)")
        mask = mask_GT.detach().reshape(-1).to(device=dev, dtype=torch.bool).contiguous()
        sal = ts.detach()[0, :n].to(device=dev, dtype=torch.float32).contiguous()
        vm = vmask.detach().to(device=dev, dtype=torch.float32).contiguous()
        has_pos = "saliency" in self.losses and "saliency_pos_labels" in targets
        losses = _QFVSLossFunction.apply(pl, xv, xt, vm, mask, sal, has_pos, self.temperature)
        out = LossDict()
        out.vector = losses  # [loss_b, loss_g, loss_f, loss_s_inter, loss_s_intra] (SetCriterion.weighted_total)
        if "labels" in self.losses:
            out["loss_f"] = losses[2]
        if "saliency" in self.losses:
            out["loss_s_inter"] = losses[3]
            out["loss_s_intra"] = losses[4]
        return out


def build_model(args):
    """Same contract as reference model/univtg_qfvs.py build_model: (Model(args), QFVSCriterion); reads the same `args` fields."""
    from .plugin import build_model as _build

    model, crit = _build(args)
    qcrit = QFVSCriterion(weight_dict=crit.weight_dict, losses=crit.losses, eos_coef=crit.eos_coef, temperature=args.temperature,
                          span_loss_type=crit.span_loss_type, max_v_l=crit.max_v_l, saliency_margin=crit.saliency_margin)
    return model, qcrit.to(crit.empty_weight.device)


# ---- semantic evaluation: eval/qfvs.py calculate_semantic_matching ----------------------------------------------------------
MAX_SIDE = 1024  # shots per summary
MAX_TAGS = 64    # tag columns (Tags.mat has 48)


def tag_masks(rows):
    """Shot-tag rows [n, <= 64] of 0 / 1 -> n uint64 masks (bit c = tag column c)."""
    t = np.asarray(rows)
    if t.ndim != 2:
        raise ValueError(f"semantic matching: the selected tag rows must form a matrix, got shape {list(t.shape)}")
    if t.shape[1] > MAX_TAGS:
        raise ValueError(f"semantic matching: more than {MAX_TAGS} tag columns")
    if not np.isin(t, (0, 1)).all():
        raise ValueError("semantic matching: tags must be 0 or 1")
    bits = np.packbits(t.astype(bool), axis=1, bitorder="little")
    out = np.zeros((len(t), 8), dtype=np.uint8)
    out[:, :bits.shape[1]] = bits
    return out.view("<u8").reshape(-1)


def match_sums(pairs):
    """univtg_qfvs_match on [(machine masks, gt masks), ...] (each 1..1024 uint64 masks) -> total matched weight per pair."""
    sides = [len(x) for p in pairs for x in p]
    if min(sides) < 1 or max(sides) > MAX_SIDE:
        raise ValueError(f"semantic matching: each summary must hold 1..{MAX_SIDE} shots")
    if not torch.cuda.is_available():
        raise RuntimeError("univtg_b200: calculate_semantic_matching runs on CUDA only (no CPU path)")
    lib = _lib.load_library()
    a = np.concatenate([p[0] for p in pairs]).astype(np.uint64)
    b = np.concatenate([p[1] for p in pairs]).astype(np.uint64)
    a_off = np.concatenate([[0], np.cumsum([len(p[0]) for p in pairs])]).astype(np.int32)
    b_off = np.concatenate([[0], np.cumsum([len(p[1]) for p in pairs])]).astype(np.int32)
    host = np.concatenate([x.view(np.uint8) for x in (a, b, a_off, b_off)])
    dev = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(dev):
        buf = torch.from_numpy(host).to(dev)
        s = torch.empty(len(pairs), dtype=torch.float64, device=dev)
        base = buf.data_ptr()
        oa, ob = 0, a.nbytes
        oao = ob + b.nbytes
        obo = oao + a_off.nbytes
        _lib.check(lib.univtg_qfvs_match(_lib.c_void_p(base + oa), _lib.c_void_p(base + oao), _lib.c_void_p(base + ob),
                                         _lib.c_void_p(base + obo), len(pairs), max(sides), _lib.ptr(s), _lib.stream_ptr()),
                   "univtg_qfvs_match")
        return s.cpu().numpy()


def calculate_semantic_matching(machine_summary, gt_summary, video_shots_tag, video_id):
    """eval/qfvs.py calculate_semantic_matching on the device; same arguments, same (precision, recall, f1) of np.float64.

    machine_summary / gt_summary: shot indices into video_shots_tag[video_id] (a [shots, tags] 0 / 1 matrix, as
    load_videos_tag returns), indexed with numpy's rules; machine_summary may be the CUDA `top_index` of score.topk as it is.
    The weight of a (machine, gt) pair is the semantic IoU of their tag sets; the total weight s of a maximum-weight matching
    comes from univtg_qfvs_match, then p = s / len(machine), r = s / len(gt), f1 = 2*p*r/(p+r) in numpy scalars as the reference
    computes them.  The reference adds the matched weights in networkx's set order, which depends on the string hash seed, so
    s agrees with it to the last bits only.  All weights 0 gives (0.0, 0.0, nan), as in the reference.

    Raises, before any launch: IndexError for an index outside the tag rows, ValueError for an empty summary (the reference's
    scikit-learn error), non-binary tags, more than 64 tag columns or more than 1,024 shots in a summary.  CUDA only."""
    tags = np.asarray(video_shots_tag[video_id])
    if torch.is_tensor(machine_summary):
        machine_summary = machine_summary.cpu().numpy()
    a_rows, b_rows = tags[machine_summary], tags[gt_summary]
    for rows, what in ((a_rows, "machine"), (b_rows, "ground-truth")):
        if rows.ndim == 2 and rows.shape[0] == 0:
            raise ValueError(f"Found array with 0 sample(s) (shape={rows.shape}) while a minimum of 1 is required: empty {what} summary")
    a, b = tag_masks(a_rows), tag_masks(b_rows)
    s = np.float64(match_sums([(a, b)])[0])
    precision = s / a_rows.shape[0]
    recall = s / b_rows.shape[0]
    f1 = 2 * precision * recall / (precision + recall)
    return precision, recall, f1
