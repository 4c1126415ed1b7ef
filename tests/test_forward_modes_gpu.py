"""The inference forward and the training forward are one computation: with DropPath and input dropout off, train mode must
launch the same kernels as eval mode and return bit-identical outputs."""
import pytest
import torch

from univtg_b200 import _lib, build_model, synth

pytestmark = pytest.mark.gpu

OUT_KEYS = ("pred_logits", "pred_spans", "saliency_scores", "vid_mem_proj", "txt_mem_proj")


def _counted(lib, fn):
    torch.cuda.synchronize()
    n0 = lib.univtg_launch_count()
    out = fn()
    torch.cuda.synchronize()
    return out, lib.univtg_launch_count() - n0


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("l_vid", [21, 150])  # L = Lv + Lt: one key tile, and L > 128 (several key tiles)
@pytest.mark.parametrize("nheads", [2, 8])  # dh = 128: wgmma attention; dh = 32: SIMT attention
def test_train_forward_matches_eval_forward(nheads, l_vid, fmt):
    cfg = dict(synth.CONFIGS["tiny"], nheads=nheads, l_vid=l_vid)
    model, _ = build_model(synth.reference_args(cfg, device="cuda:0", droppath=0.0, input_dropout=0.0, operand_format=fmt))
    model.load_state_dict(synth.make_state_dict(cfg, seed=31), strict=True)
    model.to("cuda:0")
    inp = {k: v.cuda() for k, v in synth.make_inputs(cfg, seed=32, ragged=True).items()}
    B, Lv, _ = inp["src_vid"].shape
    lib = _lib.load_library()

    model.eval()
    with torch.no_grad():
        model(**inp)  # packs the weights and builds the plan outside the counted call
        ev, n_eval = _counted(lib, lambda: model(**inp))
    model.train()
    model(**inp)
    tr, n_train = _counted(lib, lambda: model(**inp))

    assert n_eval == n_train == model.num_forward_launches(B, Lv, inp["src_txt"].shape[1])
    for k in OUT_KEYS:
        assert torch.equal(ev[k], tr[k].detach()), k
