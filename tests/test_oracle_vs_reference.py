"""Pin the oracle, the decode restatement and the plugin boundary against the original UniVTG code: its outputs for these
inputs are stored in tests/golden/reference_pins.npz (written by tests/golden/make_golden_pins.py from an unmodified checkout)."""
import json
import os

import numpy as np
import pytest
import torch

from tests.helpers import GOLDEN
from univtg_b200 import synth

_PINS = None


def pins():
    """(arrays, meta): reference outputs by name, and the structured values (losses, key lists, decoded rows)."""
    global _PINS
    if _PINS is None:
        z = dict(np.load(os.path.join(GOLDEN, "reference_pins.npz")))
        _PINS = ({k: torch.from_numpy(v) for k, v in z.items() if k != "meta"}, json.loads(z["meta"].tobytes().decode()))
    return _PINS


def _ref_outputs(prefix):
    arrays, _ = pins()
    return {k.split("/", 1)[1]: v for k, v in arrays.items() if k.startswith(prefix + "/")}


@pytest.mark.parametrize("cfg_name,ragged,batch", [("tiny", True, None), ("tiny", False, 5), ("cfg1", True, 3)])
def test_forward_and_losses(cfg_name, ragged, batch):
    from oracle import univtg_oracle as O

    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=123)
    inp = synth.make_inputs(cfg, seed=7, ragged=ragged, batch=batch)
    tgt = synth.make_targets(inp, seed=8)
    ref = _ref_outputs(f"fwd_{cfg_name}_{ragged}_{batch}")
    ref_loss = pins()[1][f"fwd_{cfg_name}_{ragged}_{batch}/losses"]
    out = O.forward(sd, cfg, **inp)
    for k in ("pred_logits", "pred_spans", "saliency_scores", "vid_mem_proj", "txt_mem_proj"):
        torch.testing.assert_close(out[k], ref[k].double(), rtol=2e-5, atol=2e-5)
    loss = O.criterion(out, tgt)
    for k, v in ref_loss.items():
        assert abs(float(loss[k]) - float(v)) < 5e-6 * max(1.0, abs(float(v))), k


def test_bool_masks_of_the_highlight_path_give_the_same_outputs():
    """The HL collate hands the model bool masks (main/dataset.py:1104) where the MR collate hands float32 ones
    (utils/tensor_utils.py:36-53): the reference and the restatement must not care."""
    from oracle import univtg_oracle as O

    cfg = synth.CONFIGS["tiny"]
    sd = synth.make_state_dict(cfg, seed=11)
    inp = synth.make_inputs(cfg, seed=3, ragged=True, batch=4)
    as_bool = dict(inp, src_vid_mask=inp["src_vid_mask"].bool(), src_txt_mask=inp["src_txt_mask"].bool())
    ref_f, ref_b = _ref_outputs("bool_float"), _ref_outputs("bool_bool")
    out = O.forward(sd, cfg, **as_bool)
    for k in ("pred_logits", "pred_spans", "saliency_scores", "vid_mem_proj", "txt_mem_proj"):
        torch.testing.assert_close(ref_b[k], ref_f[k], rtol=0, atol=0)
        torch.testing.assert_close(out[k], ref_f[k].double(), rtol=2e-5, atol=2e-5)


def test_droppath_scales_match_reference_train_mode():
    """Train mode with droppath: the reference draws floor(keep + U) per sample, per residual branch, in layer order;
    feeding the same draws to the oracle as scales reproduces its output."""
    from oracle import univtg_oracle as O

    cfg = synth.CONFIGS["tiny"]
    sd = synth.make_state_dict(cfg, seed=5)
    inp = synth.make_inputs(cfg, seed=9, ragged=True, batch=6)
    B = inp["src_vid"].shape[0]
    ref = _ref_outputs("droppath")  # the reference's train-mode output after torch.manual_seed(77)
    torch.manual_seed(77)
    keep = 0.7
    scales = torch.stack([torch.floor(keep + torch.rand((B, 1, 1))).flatten() / keep for _ in range(2 * cfg["enc_layers"])])
    out = O.forward(sd, cfg, **inp, dp_scale=scales)
    torch.testing.assert_close(out["pred_spans"], ref["pred_spans"].double(), rtol=2e-5, atol=2e-5)
    torch.testing.assert_close(out["pred_logits"], ref["pred_logits"].double(), rtol=2e-5, atol=2e-5)


def test_state_dict_keys_and_shapes_match_reference():
    for name in ("tiny", "cfg1"):
        cfg = synth.CONFIGS[name]
        ref = {k: tuple(v) for k, v in pins()[1][f"state_dict/{name}"]}
        assert list(ref.items()) == list(synth.state_dict_shapes(cfg).items())
        assert set(synth.make_state_dict(cfg)) == set(ref)


def test_input_dropout_masks_match_reference_train_mode():
    """Train mode with input dropout (nn.Dropout(0.5) inside every LinearLayer, model/univtg.py:394,401): the reference draws
    one Bernoulli mask per projector layer, video projector first (model/univtg.py:107-108).  Re-drawing the same masks with
    the same torch calls and handing them to the oracle (drop_masks=) reproduces the reference's train-mode output - this pins
    the mask semantics (multiplier 0 or 1/(1-p), applied after the LayerNorm, before the Linear) the CUDA path is tested against."""
    from oracle import univtg_oracle as O

    cfg = synth.CONFIGS["tiny"]
    sd = synth.make_state_dict(cfg, seed=5)
    inp = synth.make_inputs(cfg, seed=9, ragged=True, batch=6)
    tgt = synth.make_targets(inp, seed=10)
    B, Lv, Lt, d = inp["src_vid"].shape[0], inp["src_vid"].shape[1], inp["src_txt"].shape[1], cfg["hidden_dim"]
    ref = _ref_outputs("input_dropout")  # the reference's train-mode output after torch.manual_seed(31)
    ref_loss = pins()[1]["input_dropout/losses"]
    torch.manual_seed(31)
    shapes = [(B, Lv, cfg["v_feat_dim"]), (B, Lv, d), (B, Lt, cfg["t_feat_dim"]), (B, Lt, d)]
    masks = [torch.nn.functional.dropout(torch.ones(s), 0.5, True) for s in shapes]
    out = O.forward(sd, cfg, **inp, drop_masks=masks)
    for k in ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj"):
        torch.testing.assert_close(out[k], ref[k].detach().double(), rtol=2e-5, atol=2e-5)
    loss = O.criterion(out, tgt)
    for k, v in ref_loss.items():
        assert abs(float(loss[k]) - float(v)) < 5e-6 * max(1.0, abs(float(v))), k


def test_hl_loss_list_matches_reference():
    """dset_type 'hl' / 'vs': losses = ['labels', 'saliency'] and the targets carry no timestamp / span_labels_nn
    (model/univtg.py:438-439, main/dataset.py:1118-1126)."""
    from oracle import univtg_oracle as O

    cfg = synth.CONFIGS["tiny"]
    from univtg_b200 import build_model

    sd = synth.make_state_dict(cfg, seed=5)
    assert pins()[1]["hl/crit_losses"] == ["labels", "saliency"]
    assert build_model(synth.reference_args(cfg, device="cpu", dset_type="hl"))[1].losses == ["labels", "saliency"]
    inp = synth.make_inputs(cfg, seed=9, ragged=True, batch=6)
    full = synth.make_targets(inp, seed=10)
    tgt = {"saliency_scores": full["saliency_scores"], "saliency_pos_labels": full["saliency_pos_labels"],
           "timestamp_mask": full["timestamp_mask"], "timestamp_window": 1 * (full["saliency_scores"] > 0)}
    ref_loss = pins()[1]["hl/losses"]
    assert sorted(ref_loss) == ["loss_f", "loss_s_inter", "loss_s_intra"]
    loss = O.criterion(O.forward(sd, cfg, **inp), tgt, losses=("labels", "saliency"))
    assert sorted(loss) == sorted(ref_loss)
    for k, v in ref_loss.items():
        assert abs(float(loss[k]) - float(v)) < 5e-6 * max(1.0, abs(float(v))), k


def decode_case():
    """Fixed model outputs replayed through the evaluation loop: (outputs, timestamps, video mask, durations, B, Lt)."""
    g = torch.Generator().manual_seed(1234)
    B, Lv, Lt = 5, 23, 7
    lens = [23, 9, 17, 1, 12]
    vmask = torch.zeros(B, Lv)
    for b, n in enumerate(lens):
        vmask[b, :n] = 1
    pred_logits = torch.rand(B, Lv, 1, generator=g)
    pred_logits[0, 3] = pred_logits[0, 5]  # ties: sorted() is stable
    pred_logits[2, 0, 0] = 0.12345  # rounding-sensitive values
    pred_spans = torch.rand(B, Lv, 2, generator=g) * torch.tensor([-1.0, 1.0])
    sal = torch.randn(B, Lv, generator=g)
    ts = ((torch.arange(Lv, dtype=torch.float32) + 0.5) / Lv)[None, :, None].expand(B, Lv, 2).contiguous()
    durs = [150.0, 33.3, 126.0, 2.0, 150.0]
    outputs = {"pred_logits": pred_logits, "pred_spans": pred_spans, "saliency_scores": sal}
    return outputs, ts, vmask, durs, B, Lt


@pytest.mark.parametrize("sort", [True, False])
def test_decode_restatement_matches_compute_mr_results(sort):
    """Pins oracle/postproc_oracle.decode_mr + saliency_lists to the reference's own evaluation loop: what compute_mr_results
    (main/inference_mr.py:86-193) returned when a stub model / loader replayed these outputs."""
    from oracle import postproc_oracle as PO

    outputs, ts, vmask, durs, B, _ = decode_case()
    res = pins()[1][f"decode/{sort}"]
    rows = PO.decode_mr(outputs["pred_logits"], outputs["pred_spans"], ts, vmask, durs, sort=sort)
    sal_lists = PO.saliency_lists(outputs["saliency_scores"], vmask)
    assert len(res) == B
    for b in range(B):
        assert [list(r) for r in rows[b]] == res[b]["pred_relevant_windows"], b
        assert list(sal_lists[b]) == res[b]["pred_saliency_scores"], b


def test_plugin_matches_what_reference_setup_model_builds():
    """Boundary (SURVEY 8b): main.config.setup_model does importlib.import_module('model.' + opt.model_id).build_model(opt)
    (main/config.py:341-342) and builds AdamW over every trainable parameter, the WarmupStepLR scheduler and the criterion.
    The plugin built from the same args exposes the same parameter names / order / shapes, so the optimizer and scheduler the
    reference builds around it are the ones it built for --model_id univtg."""
    from univtg_b200 import build_model

    ref = pins()[1]["setup_model"]
    cfg = synth.CONFIGS["tiny"]
    torch.manual_seed(0)
    model, crit = build_model(synth.reference_args(cfg, device="cpu", model_id="univtg_b200"))
    names = [[n, list(p.shape)] for n, p in model.named_parameters() if p.requires_grad]
    assert names == ref["named_parameters"]
    assert [s for _, s in names] == ref["optimizer_shapes"]
    assert ref["optimizer"] == "AdamW" and ref["scheduler"] == "WarmupStepLR"
    assert {k: float(v) for k, v in crit.weight_dict.items()} == ref["weight_dict"] and list(crit.losses) == ref["losses"]
