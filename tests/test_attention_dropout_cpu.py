"""Pin the attention-dropout semantics the CUDA path is tested against to the original UniVTG code: its train-mode outputs with
args.dropout = p (and no other randomness) are stored in tests/golden/reference_attn_dropout.npz, written by
tests/golden/make_golden_attn_dropout.py.  torch's F.dropout draws depend only on the shape (not the values) and p = 0 dropout
draws nothing, so re-drawing F.dropout(ones([B*H, L, L]), p) per encoder layer after the same torch.manual_seed reproduces the
reference's masks; handed to the oracle as attn_masks they must reproduce its outputs."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import univtg_oracle as O
from tests import attn_dropout_oracle as AO
from tests.helpers import GOLDEN
from univtg_b200 import synth

_FIX = None


def fixture():
    global _FIX
    if _FIX is None:
        z = dict(np.load(os.path.join(GOLDEN, "reference_attn_dropout.npz")))
        _FIX = ({k: torch.from_numpy(v) for k, v in z.items() if k != "meta"}, json.loads(z["meta"].tobytes().decode()))
    return _FIX


def _case(cfg_name, batch):
    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=21)
    inp = synth.make_inputs(cfg, seed=22, ragged=True, batch=batch)
    return cfg, sd, inp, synth.make_targets(inp, seed=23)


@pytest.mark.parametrize("cfg_name,batch,p,seed", [tuple(c) for c in json.loads(
    np.load(os.path.join(GOLDEN, "reference_attn_dropout.npz"))["meta"].tobytes().decode())["cases"]])
def test_attention_dropout_masks_match_reference_train_mode(cfg_name, batch, p, seed):
    arrays, meta = fixture()
    cfg, sd, inp, tgt = _case(cfg_name, batch)
    B = inp["src_vid"].shape[0]
    L = inp["src_vid"].shape[1] + inp["src_txt"].shape[1]
    H = cfg["nheads"]
    torch.manual_seed(seed)
    masks = [torch.nn.functional.dropout(torch.ones(B * H, L, L), p, True).reshape(B, H, L, L) for _ in range(cfg["enc_layers"])]
    out = AO.forward(sd, cfg, **inp, attn_masks=masks)
    name = f"{cfg_name}_p{p}"
    for k in ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj"):
        torch.testing.assert_close(out[k], arrays[f"{name}/{k}"].double(), rtol=2e-5, atol=2e-5)
    loss = O.criterion(out, tgt)
    for k, v in meta[f"{name}/losses"].items():
        assert abs(float(loss[k]) - float(v)) < 5e-6 * max(1.0, abs(float(v))), k
    # the masks matter: the eval-mode outputs differ
    ev = O.forward(sd, cfg, **inp)
    assert not torch.allclose(ev["pred_spans"], out["pred_spans"], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("opq", [None, O.round_fp16])
def test_oracle_without_masks_is_the_oracle(opq):
    """attn_masks=None gives exactly oracle.univtg_oracle.forward (with and without fp16 operand emulation)."""
    cfg, sd, inp, _ = _case("tiny", 4)
    a = AO.forward(sd, cfg, **inp, opq=opq)
    b = O.forward(sd, cfg, **inp, opq=opq)
    for k in ("pred_logits", "pred_spans", "saliency_scores", "vid_mem_proj", "txt_mem_proj"):
        assert torch.equal(a[k], b[k]), k


def test_all_ones_masks_change_nothing():
    """A mask of ones (every probability kept, scale 1) is the eval forward bit for bit, also under fp16 operand emulation."""
    cfg, sd, inp, _ = _case("tiny", 4)
    B, L, H = inp["src_vid"].shape[0], inp["src_vid"].shape[1] + inp["src_txt"].shape[1], cfg["nheads"]
    ones = [torch.ones(B, H, L, L) for _ in range(cfg["enc_layers"])]
    a = AO.forward(sd, cfg, **inp, opq=O.round_fp16, attn_masks=ones)
    b = O.forward(sd, cfg, **inp, opq=O.round_fp16)
    for k in ("pred_logits", "pred_spans", "saliency_scores"):
        assert torch.equal(a[k], b[k]), k
