"""Criterion glue: SetCriterion.forward through univtg_loss_forward / univtg_loss_backward (CUDA), autograd-compatible."""
import torch

from . import _lib

LOSS_NAMES = ("loss_b", "loss_g", "loss_f", "loss_s_inter", "loss_s_intra")


class LossDict(dict):
    """The reference's loss dict; additionally carries the five losses as one tensor in `.vector`."""

    vector = None


class _LossFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred_logits, pred_spans, vid_mem_proj, txt_mem_proj, crit, tg):
        lib = _lib.load_library()
        dev = pred_logits.device
        B, Lv = pred_logits.shape[:2]
        d = vid_mem_proj.shape[-1]
        with torch.cuda.device(dev):
            pl = pred_logits.detach().to(torch.float32).contiguous()
            ps = pred_spans.detach().to(torch.float32).contiguous()
            xv = vid_mem_proj.detach().to(torch.float32).contiguous()
            xt = txt_mem_proj.detach().to(torch.float32).contiguous()
            scratch = torch.empty(lib.univtg_loss_scratch_bytes(B, Lv), dtype=torch.uint8, device=dev)
            losses = torch.zeros(5, device=dev)
            _lib.check(lib.univtg_loss_forward(_lib.ptr(pl), _lib.ptr(ps), _lib.ptr(xv), _lib.ptr(xt), _lib.ptr(tg.get("timestamp")),
                                               _lib.ptr(tg["timestamp_mask"]), _lib.ptr(tg["timestamp_window"]),
                                               _lib.ptr(tg.get("span_labels_nn")), _lib.ptr(tg["saliency_scores"]), _lib.ptr(tg["pos"]),
                                               B, Lv, d, float(crit.eos_coef), float(crit.temperature), _lib.ptr(losses),
                                               _lib.ptr(scratch), _lib.stream_ptr()), "univtg_loss_forward")
        ctx.saved = (xv, xt, tg["pos"], scratch, B, Lv, d)
        return losses

    @staticmethod
    def backward(ctx, g_losses):
        lib = _lib.load_library()
        xv, xt, pos, scratch, B, Lv, d = ctx.saved
        dev = xv.device
        with torch.cuda.device(dev):
            w = g_losses.detach().to(torch.float32).contiguous()
            d_logits = torch.empty(B, Lv, 1, device=dev)
            d_spans = torch.empty(B, Lv, 2, device=dev)
            d_xv = torch.empty(B, Lv, d, device=dev)
            d_xt = torch.empty(B, 1, d, device=dev)
            _lib.check(lib.univtg_loss_backward(_lib.ptr(w), _lib.ptr(xv), _lib.ptr(xt), _lib.ptr(pos), B, Lv, d, _lib.ptr(scratch),
                                                _lib.ptr(d_logits), _lib.ptr(d_spans), _lib.ptr(d_xv), _lib.ptr(d_xt),
                                                _lib.stream_ptr()), "univtg_loss_backward")
        return d_logits, d_spans, d_xv, d_xt, None, None


def _f32(t, dev):
    return t.detach().to(device=dev, dtype=torch.float32).contiguous()


def _check_target_shapes(crit, outputs, targets):
    """The loss kernels index the dense targets as [B, Lv] (and [B, Lv, 2]) and saliency_pos_labels by sample: a target of
    another shape would be read out of bounds, so it is refused here (shape metadata only, no device access)."""
    B, Lv = outputs["pred_logits"].shape[:2]
    dense = {"timestamp_mask": (B, Lv), "timestamp_window": (B, Lv)}
    if "spans" in crit.losses:
        dense.update(timestamp=(B, Lv, 2), span_labels_nn=(B, Lv, 2))
    if "saliency" in crit.losses and "saliency_pos_labels" in targets and "saliency_scores" in targets:
        dense["saliency_scores"] = (B, Lv)
        pos = targets["saliency_pos_labels"]
        if pos.dim() != 2 or pos.shape[0] != B or pos.shape[1] < 1:
            raise ValueError(f"saliency_pos_labels must be [B, k >= 1] with B = {B} rows, got {list(pos.shape)}")
    for k, shp in dense.items():
        if tuple(targets[k].shape) != shp:
            raise ValueError(f"target {k} must be {list(shp)} (B, Lv of pred_logits), got {list(targets[k].shape)}")


def criterion_forward(crit, outputs, targets):
    """Returns the reference's loss dict (model/univtg.py:338-351).  Supported loss lists: the ones build_model produces for
    dset_type in {mr, vlp} without 'tal' (spans, labels, saliency) and {hl, vs} (labels, saliency)."""
    if "saliency_cls" in crit.losses:
        raise NotImplementedError("loss 'saliency_cls' ('tal' train_path) is outside the accelerated path")
    _check_target_shapes(crit, outputs, targets)
    dev = outputs["pred_logits"].device
    if dev.type != "cuda":
        raise RuntimeError("univtg_b200: the criterion runs on CUDA tensors only (no CPU path)")
    B, Lv = outputs["pred_logits"].shape[:2]
    tg = {k: _f32(targets[k], dev) for k in ("timestamp_mask", "timestamp_window")}
    if "spans" in crit.losses:  # the hl / vs targets carry neither timestamp nor span_labels_nn (main/dataset.py:1118-1126)
        tg["timestamp"] = _f32(targets["timestamp"], dev)
        tg["span_labels_nn"] = _f32(targets["span_labels_nn"], dev)
    if "saliency" in crit.losses and "saliency_pos_labels" in targets and "saliency_scores" in targets:
        tg["saliency_scores"] = _f32(targets["saliency_scores"], dev)
        tg["pos"] = targets["saliency_pos_labels"][:, 0].detach().to(device=dev, dtype=torch.int64).contiguous()
    else:
        tg["saliency_scores"] = torch.zeros(B, Lv, device=dev)
        tg["pos"] = None
    losses = _LossFunction.apply(outputs["pred_logits"], outputs["pred_spans"], outputs["vid_mem_proj"], outputs["txt_mem_proj"],
                                 crit, tg)
    out = LossDict()
    out.vector = losses  # [loss_b, loss_g, loss_f, loss_s_inter, loss_s_intra] as ONE tensor (SetCriterion.weighted_total)
    if "spans" in crit.losses:
        out["loss_b"] = losses[0]
        out["loss_g"] = losses[1]
    if "labels" in crit.losses:
        out["loss_f"] = losses[2]
    if "saliency" in crit.losses:
        out["loss_s_inter"] = losses[3]
        out["loss_s_intra"] = losses[4]
    return out
