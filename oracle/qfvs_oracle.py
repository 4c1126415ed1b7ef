"""CPU oracle of the QFVS criterion -- TEST INFRASTRUCTURE ONLY (the product package never imports oracle/).

A restatement, in explicit torch tensor algebra (fp64 or fp32, whatever the inputs are), of SetCriterion.forward of the
reference's model/univtg_qfvs.py (paths relative to the UniVTG repository root):
  forward        :358-377  keep flat position i of pred_logits / saliency_scores iff mask_GT[0, i]; targets row 0 sliced to the
                           kept count
  loss_labels    :215-228  0 when the sliced targets sum to 0; else BCE(kept pred_logits, t) summed / sum(t) (the `weights`
                           tensor it builds is never used)
  loss_saliency  :246-261  0 without "saliency_pos_labels" or when sum(t) == 0; else -mean over t > 0 of
                           log softmax(kept saliency_scores / 0.07), the temperature hard-set at :184; loss_s_inter is always 0
tests/test_qfvs_cpu.py pins it to tests/golden/reference_qfvs.npz (written by tests/golden/make_golden_qfvs.py from the reference).
"""
import torch
import torch.nn.functional as F

from oracle.univtg_oracle import cosine


def saliency_scores(vid_mem_proj, txt_mem_proj, src_vid_mask):
    """The model's saliency_scores (model/univtg_qfvs.py:146-153): cos(vid, txt) + log(mask + 1e-45), the constant being the
    smallest fp32 denormal 2**-149 in the reference."""
    tiny = torch.tensor(2.0 ** -149, dtype=vid_mem_proj.dtype, device=vid_mem_proj.device)
    return cosine(vid_mem_proj, txt_mem_proj.reshape(txt_mem_proj.shape[0], 1, -1)) + torch.log(src_vid_mask.to(vid_mem_proj.dtype) + tiny)


def criterion(outputs, targets, mask_GT, losses=("labels", "saliency"), temperature=0.07):
    """Loss dict of one criterion call; every entry a tensor (the reference's Python 0. becomes a 0 tensor)."""
    if "spans" in losses:
        raise KeyError("timestamp")  # loss_spans reads targets['timestamp'], which QFVS targets do not carry
    keep = mask_GT.reshape(-1).bool()
    count = int(keep.sum())
    p = outputs["pred_logits"].reshape(-1)[keep]
    dtype = p.dtype
    t = targets["saliency_scores"][0, :count].to(dtype)
    zero = torch.zeros((), dtype=dtype, device=p.device)
    empty = float(t.sum()) == 0.0
    res = {}
    if "labels" in losses:
        res["loss_f"] = zero if empty else F.binary_cross_entropy(p, t, reduction="sum") / t.sum()
    if "saliency" in losses:
        res["loss_s_inter"] = zero
        if "saliency_pos_labels" not in targets or empty:
            res["loss_s_intra"] = zero
        else:
            z = outputs["saliency_scores"].reshape(-1)[keep] / temperature
            res["loss_s_intra"] = -torch.log_softmax(z, dim=0)[t > 0].mean()
    return res


def gather(dicts, qfvs_loss_gather):
    """The loss dict a train step back-propagates (main/train_qfvs.py:185-195): the key-wise sum of the three criterion calls when
    qfvs_loss_gather > 0, else the oracle query's alone (the last of the three)."""
    if qfvs_loss_gather > 0:
        return {k: dicts[0][k] + dicts[1][k] + dicts[2][k] for k in dicts[0]}
    return dicts[2]
