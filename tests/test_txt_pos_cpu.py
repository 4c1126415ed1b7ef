"""Pin the learned-text-position semantics (args.use_txt_pos) the CUDA path is tested against to the original UniVTG code: its
eval outputs, train-mode outputs, losses and gradients with use_txt_pos = True are stored in tests/golden/reference_txt_pos.npz,
written by tests/golden/make_golden_txt_pos.py.  torch's F.dropout draws depend only on the shape, so re-drawing
F.dropout(ones) in the reference's order (video projector layers, text projector layers, then the text positions [B, Lt, d])
after the same torch.manual_seed reproduces the reference's masks; handed to tests/txt_pos_oracle.py they must reproduce its
numbers."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import univtg_oracle as O
from tests import txt_pos_oracle as TO
from tests.helpers import GOLDEN
from univtg_b200 import build_model, synth

OUT = ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj", "saliency_scores")
WD = {"loss_b": 10.0, "loss_g": 1.0, "loss_f": 10.0, "loss_s_intra": 0.1, "loss_s_inter": 0.1}
_FIX = None


def fixture():
    global _FIX
    if _FIX is None:
        z = dict(np.load(os.path.join(GOLDEN, "reference_txt_pos.npz")))
        _FIX = ({k: torch.from_numpy(v) for k, v in z.items() if k != "meta"}, json.loads(z["meta"].tobytes().decode()))
    return _FIX


CASES = [tuple(c) for c in json.loads(np.load(os.path.join(GOLDEN, "reference_txt_pos.npz"))["meta"].tobytes().decode())["cases"]]


def _case(cfg_name, batch):
    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=21)
    inp = synth.make_inputs(cfg, seed=22, ragged=True, batch=batch)
    return cfg, sd, inp, synth.make_targets(inp, seed=23)


def _reference_order_masks(cfg, inp, p, seed):
    """F.dropout(ones) in the reference's draw order: input_vid_proj layers, input_txt_proj layers, txt_position_embed."""
    B, Lv, Dv = inp["src_vid"].shape
    Lt, Dt = inp["src_txt"].shape[1:]
    d, n = cfg["hidden_dim"], cfg["n_input_proj"]
    dims_v = [Dv] + [d] * 3
    dims_t = [Dt] + [d] * 3
    torch.manual_seed(seed)
    drop = lambda shp: torch.nn.functional.dropout(torch.ones(shp), p, True)  # noqa: E731
    masks = [drop((B, Lv, dims_v[i])) for i in range(n)] + [drop((B, Lt, dims_t[i])) for i in range(n)]
    return masks, drop((B, Lt, d))


@pytest.mark.parametrize("cfg_name,batch,seed", CASES)
def test_eval_matches_reference(cfg_name, batch, seed):
    arrays, _ = fixture()
    cfg, sd, inp, _ = _case(cfg_name, batch)
    out = TO.forward(sd, cfg, **inp, use_txt_pos=True)
    for k in OUT:
        torch.testing.assert_close(out[k], arrays[f"{cfg_name}/eval/{k}"].double(), rtol=2e-5, atol=2e-5, msg=lambda m: f"{k}: {m}")
    # the positions matter
    assert not torch.allclose(O.forward(sd, cfg, **inp)["pred_spans"], out["pred_spans"], rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("cfg_name,batch,seed", CASES)
def test_train_mode_outputs_losses_and_gradients_match_reference(cfg_name, batch, seed):
    arrays, meta = fixture()
    cfg, sd, inp, tgt = _case(cfg_name, batch)
    masks, tmul = _reference_order_masks(cfg, inp, 0.5, seed)
    leaves = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    out = TO.forward(leaves, cfg, **inp, drop_masks=masks, use_txt_pos=True, txt_pos_mul=tmul)
    for k in OUT:
        torch.testing.assert_close(out[k].detach(), arrays[f"{cfg_name}/train/{k}"].double(), rtol=2e-5, atol=2e-5,
                                   msg=lambda m: f"{k}: {m}")
    loss = O.criterion(out, tgt)
    for k, v in meta[f"{cfg_name}/losses"].items():
        assert abs(float(loss[k].detach()) - float(v)) < 5e-6 * max(1.0, abs(float(v))), k
    O.weighted_total(loss, WD).backward()
    for k in ("txt_position_embed.position_embeddings.weight", "txt_position_embed.LayerNorm.weight",
              "txt_position_embed.LayerNorm.bias", "token_type_embeddings.weight"):
        ref = arrays[f"{cfg_name}/grad/{k}"].double()
        got = leaves[k].grad
        rel = float((got - ref).norm() / ref.norm())
        assert rel < 2e-5, (k, rel)
    # rows of the position table beyond Lt receive exactly zero
    Lt = inp["src_txt"].shape[1]
    assert float(leaves["txt_position_embed.position_embeddings.weight"].grad[Lt:].abs().max()) == 0.0


@pytest.mark.parametrize("opq", [None, O.round_fp16])
def test_oracle_without_text_positions_is_the_oracle(opq):
    """use_txt_pos=False gives exactly oracle.univtg_oracle.forward (with and without fp16 operand emulation)."""
    cfg, sd, inp, _ = _case("tiny", 4)
    a = TO.forward(sd, cfg, **inp, opq=opq)
    b = O.forward(sd, cfg, **inp, opq=opq)
    for k in OUT:
        assert torch.equal(a[k], b[k]), k


def test_build_model_with_text_positions_on_cpu_refuses_to_run_without_cuda():
    cfg = synth.CONFIGS["tiny"]
    model, _ = build_model(synth.reference_args(cfg, device="cpu", use_txt_pos=True))
    model.load_state_dict(synth.make_state_dict(cfg, seed=3), strict=True)
    ps = model._abi_params()
    tp = model.txt_position_embed
    assert ps[-3:] == [tp.position_embeddings.weight, tp.LayerNorm.weight, tp.LayerNorm.bias]
    assert len(model._packed_params()) == len(ps) - 3
    inp = synth.make_inputs(cfg, seed=1, ragged=True, batch=2)
    with pytest.raises(RuntimeError, match="CUDA"):
        model.eval()
        model(**inp)
    with pytest.raises(RuntimeError, match="CUDA"):
        model.train()
        model(**inp)


def test_more_text_tokens_than_max_q_l_is_a_value_error():
    cfg = synth.CONFIGS["tiny"]
    model, _ = build_model(synth.reference_args(cfg, device="cpu", use_txt_pos=True, max_q_l=8))
    inp = synth.make_inputs(cfg, seed=1, ragged=True, batch=2, l_txt=9)
    with pytest.raises(ValueError, match=r"9 text tokens exceed max_q_l = 8"):
        model(**inp)
    # without the feature the table is never read: no limit
    model, _ = build_model(synth.reference_args(cfg, device="cpu", use_txt_pos=False, max_q_l=8))
    with pytest.raises(RuntimeError, match="CUDA"):
        model(**inp)
