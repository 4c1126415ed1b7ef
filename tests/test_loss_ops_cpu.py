"""The criterion's references and host checks without a GPU.

* The fp64 reference of tests/loss_ref.py and the oracle's criterion (oracle/univtg_oracle.py) both reproduce the unmodified
  reference SetCriterion on its edge batches (tests/golden/reference_loss_edges.npz, written by
  tests/golden/make_golden_loss_edges.py): losses and output gradients, NaN exactly where the reference's are.  At p = 0 and
  p = 1 the gradient of loss_f is torch's finite w (p - y) / float32(1e-12), not the NaN of differentiating clamped logs.
* univtg_loss_forward / univtg_loss_backward and the QFVS pair refuse, before touching any pointer, the shapes and alignments
  their kernels cannot handle, and name the argument.  The pointers passed here are fake: a refusal launches nothing.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from tests import loss_ref as R
from univtg_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden():
    z = dict(np.load(os.path.join(ROOT, "tests", "golden", "reference_loss_edges.npz")))
    meta = json.loads(bytes(z.pop("meta")).decode())
    return z, meta


def _case(z, meta, name):
    m = meta["cases"][name]
    c = {"timestamp": None, "span_labels_nn": None, "pos": None, "eos_coef": m["eos_coef"]}
    for k in ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj", "timestamp", "timestamp_mask", "timestamp_window",
              "span_labels_nn", "saliency_scores", "pos"):
        if f"{name}/in/{k}" in z:
            c[k] = torch.from_numpy(z[f"{name}/in/{k}"])
    return c


def _close(got, ref, what, rtol=1e-4, atol=1e-5):
    """NaN for NaN; elsewhere |got - ref| <= rtol |ref| + atol max |ref|.  ref is the reference in fp32, whose masked cosines
    cos + log(1e-45) carry 2^-24 * 103.3 / 0.07, about 1e-4, of rounding into the softmax weights."""
    got, ref = got.double(), ref.double()
    assert torch.equal(torch.isnan(got), torch.isnan(ref)), f"{what}: NaN pattern differs"
    f = ~torch.isnan(ref)
    g, r = got[f], ref[f]
    if r.numel() == 0:
        return
    scale = float(r.abs().max())
    err = (g - r).abs()
    assert bool((err <= rtol * r.abs() + atol * scale).all()), f"{what}: worst error {float(err.max())} (scale {scale})"


def _check_all(z, meta, name, losses, grads):
    ref = meta["cases"][name]["losses"]
    for k, v in ref.items():
        _close(torch.tensor(float(losses[k].detach() if torch.is_tensor(losses[k]) else losses[k])), torch.tensor(v), f"{name}/{k}", atol=0.0)
    for k, g in grads.items():
        _close(g, torch.from_numpy(z[f"{name}/grad/{k}"]), f"{name}/grad {k}")


def test_golden_covers_the_edge_batches(golden):
    _, meta = golden
    edges = {e for m in meta["cases"].values() for e in m["edges"]}
    assert {"giou", "bce", "pos", "sal_ties", "no_fg", "no_valid", "no_pos", "sal_zero"} <= edges
    assert {m["B"] for m in meta["cases"].values()} >= {1, 33}
    assert {m["eos_coef"] for m in meta["cases"].values()} == {0.1, 0.5}
    assert np.isnan(meta["cases"]["no_fg"]["losses"]["loss_b"]) and np.isnan(meta["cases"]["no_valid"]["losses"]["loss_f"])


@pytest.mark.parametrize("name", ["giou_ties", "bce_saturated", "bce_saturated_eos05", "positives", "b1", "b1_l16", "b33", "no_fg",
                                  "no_valid", "no_pos", "sal_zero", "mixed_eos05"])
def test_fp64_reference_and_oracle_match_the_reference(golden, name):
    from oracle import univtg_oracle as O

    z, meta = golden
    c = _case(z, meta, name)
    losses, (g,) = R.mr_reference(c, [R.TRAIN_W])
    _check_all(z, meta, name, losses, g)
    # the oracle, fp64 autograd through its own restatement
    leaves = {"pred_logits": c["pred_logits"].double().unsqueeze(-1).requires_grad_(True),
              "pred_spans": c["pred_spans"].double().requires_grad_(True),
              "vid_mem_proj": c["vid_mem_proj"].double().requires_grad_(True),
              "txt_mem_proj": c["txt_mem_proj"].double().unsqueeze(1).requires_grad_(True)}
    tg = {k: c[k] for k in ("timestamp", "timestamp_mask", "timestamp_window", "span_labels_nn", "saliency_scores")}
    if c["pos"] is not None:
        tg["saliency_pos_labels"] = c["pos"].unsqueeze(1)
    ol = O.criterion(leaves, tg, eos_coef=c["eos_coef"])
    O.weighted_total(ol, dict(zip(R.LOSS_NAMES, R.TRAIN_W))).backward()
    og = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).reshape(c[k].shape) for k, v in leaves.items()}
    _check_all(z, meta, name, ol, og)


def test_oracle_bce_gradient_is_finite_at_saturated_probabilities():
    from oracle import univtg_oracle as O

    p = torch.tensor([[1.0, 0.0, 1.0, 0.0]], dtype=torch.float64).unsqueeze(-1).requires_grad_(True)
    window = torch.tensor([[0.0, 1.0, 1.0, 0.0]])
    tg = {"timestamp_mask": torch.ones(1, 4), "timestamp_window": window, "saliency_scores": torch.zeros(1, 4)}
    out = {"pred_logits": p, "pred_spans": torch.zeros(1, 4, 2, dtype=torch.float64)}
    O.criterion(out, tg, eos_coef=1.0, losses=("labels",))["loss_f"].backward()
    g = 1.0 / float(torch.tensor(1e-12, dtype=torch.float32)) / 4  # torch clamps p (1 - p) at float32(1e-12) in any dtype
    assert p.grad.flatten().tolist() == pytest.approx([g, -g, 0.0, 0.0], rel=1e-15, abs=0.0)


# ---- host checks: every refusal happens before a pointer is read, so fake device addresses are enough ----
def _fake(off=0):
    return ctypes.c_void_p(0x7F0000000000 + off)


def _mr_fwd(B=4, Lv=75, d=64, xv=0, xt=0):
    lib = _lib.load_library()
    f = _fake
    return lib.univtg_loss_forward(f(), f(0x100), f(0x200 + xv), f(0x300 + xt), f(0x400), f(0x500), f(0x600), f(0x700), f(0x800),
                                   f(0x900), B, Lv, d, 0.1, 0.07, f(0xA00), f(0xB00), None)


def _mr_bwd(B=4, Lv=75, d=64, xv=0, xt=0, dxv=0, dxt=0):
    lib = _lib.load_library()
    f = _fake
    return lib.univtg_loss_backward(f(), f(0x200 + xv), f(0x300 + xt), f(0x900), B, Lv, d, f(0xB00), f(0xC00), f(0xD00),
                                    f(0xE00 + dxv), f(0xF00 + dxt), None)


def _qf_fwd(B=4, Lv=75, d=64, xv=0, xt=0):
    lib = _lib.load_library()
    f = _fake
    return lib.univtg_qfvs_loss_forward(f(), f(0x200 + xv), f(0x300 + xt), f(0x400), f(0x500), f(0x600), 1, B, Lv, d, 0.07, f(0xA00),
                                        f(0xB00), None)


def _qf_bwd(B=4, Lv=75, d=64, xv=0, xt=0, dxv=0, dxt=0):
    lib = _lib.load_library()
    f = _fake
    return lib.univtg_qfvs_loss_backward(f(), f(0x200 + xv), f(0x300 + xt), B, Lv, d, f(0xB00), f(0xC00), f(0xE00 + dxv),
                                         f(0xF00 + dxt), None)


SHAPES = [(dict(B=0), "B 0"), (dict(B=257), "257"), (dict(Lv=0), "Lv 0"), (dict(d=0), "d 0"), (dict(d=2), "d 2"),
          (dict(d=66), "d 66"), (dict(B=1, Lv=12287), "shared memory"), (dict(B=256, Lv=11777), "shared memory")]


@pytest.mark.parametrize("call", [_mr_fwd, _mr_bwd, _qf_fwd, _qf_bwd], ids=["mr_fwd", "mr_bwd", "qfvs_fwd", "qfvs_bwd"])
def test_loss_entry_points_refuse_bad_shapes(call):
    for kw, msg in SHAPES:
        if "257" in msg and call in (_qf_fwd, _qf_bwd):
            continue  # the QFVS kernels have no 256-sample limit
        assert call(**kw) != 0, kw
        assert msg in _lib.last_error(), (kw, _lib.last_error())


@pytest.mark.parametrize("call", [_mr_fwd, _mr_bwd, _qf_fwd, _qf_bwd], ids=["mr_fwd", "mr_bwd", "qfvs_fwd", "qfvs_bwd"])
def test_loss_entry_points_refuse_misaligned_rows(call):
    names = {"xv": "vid_mem_proj", "xt": "txt_mem_proj", "dxv": "d_vid_mem_proj", "dxt": "d_txt_mem_proj"}
    if call in (_mr_fwd, _qf_fwd):
        names = {k: v for k, v in names.items() if not k.startswith("d")}
    for k, name in names.items():
        for off in (4, 8, 12):
            assert call(**{k: off}) != 0, (k, off)
            assert f"{name} must be 16-byte aligned" in _lib.last_error(), (k, _lib.last_error())
            assert _lib.last_error().split(": ")[1].startswith(name)
