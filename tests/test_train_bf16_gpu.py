"""GPU parity of the bf16 training path (operand_format="bf16"): the whole step - forward, criterion, backward - against the
exact fp64 oracle and the bf16-emulating one, the loss-scale handling of the backward, FlatAdamW's update and 16-bit operand
refresh, the graphed step, and the skipped-update count of the optimizer in every format.

Gradient acceptance, per parameter tensor (rel = relative L2 error):
  * self-calibrating: rel(bf16 kernels, bf16-emulating oracle) <= R * rel(fp16 kernels, fp16-emulating oracle) + FLOOR, the
    fp16 run being the same batch through an fp16 model with the same weights.  bf16 keeps 8 significand bits to fp16's 11,
    so its rounding unit is 8x larger and R sits near 8-16;
  * absolute: rel(bf16 kernels, exact) <= REL_CAP and cosine(bf16 kernels, exact) >= COS_CAP.
Measured on an H100 80GB HBM3 (700 W power limit) over the nine cases below, and the bars (each <= 1.5x the measured worst):
  bar                                    measured worst                                           asserted
  R (rel_bf16 / rel_fp16, slope)         all tensors of the cfg2 / cfg4 / QFVS / tiny_ragged cases  16
                                         within 16 x + 7e-6 (ratios up to 266 only where fp16 is
                                         at 3e-5 and bf16 at 9e-3: the floor's range)
  FLOOR (rel_bf16 - 16 rel_fp16)         tiny_full 2.35e-2 (class_embed.layers.1.weight, head        3.5e-2
                                         gain 4), tiny_txt_pos 1.31e-2, tiny_hl 8.5e-3,             2e-2, 1.3e-2,
                                         the other six <= 7e-6                                      1e-3
  REL_CAP (rel_bf16 vs exact)            0.123 (tiny_ragged input_vid_proj.0.LayerNorm.weight)      0.18
  COS_CAP (cosine vs exact)              0.9925 (same tensor)                                       0.988
  (for comparison the fp16 kernels' worst rel vs exact over the same cases is 0.044)
A kernel that reads bf16 operands as fp16 (or the reverse) makes a gradient garbage, far beyond any of these bars.

Loss-scale equivariance: a power-of-two loss scale commutes with bf16 and fp32 rounding, so the parameter gradients at
grad_scale 1 and 2^10 agree bit for bit wherever no fp32 atomic reorders a sum; the tensors the backward reduces with atomics
(found from the launch plan, _atomic_params) get the suite's atomics tolerance.  With bf16's default scale of 1, this is what
shows a missing or doubled 1 / scale on a parameter gradient."""
import ctypes
import json
import os

import pytest
import torch

from oracle import univtg_oracle as O
from tests import attn_dropout_oracle as AO
from tests import txt_pos_oracle as TO
from tests.helpers import load_golden
from tests.test_train_gpu import _cos, _rel
from tests.test_train_graph_gpu import _batch, _close_trajectory, _eager_step, _graphed_call
from univtg_b200 import _lib, build_model, synth
from univtg_b200.graphs import GraphedTrainStep, rng_seed_at
from univtg_b200.optim import FlatAdamW

pytestmark = pytest.mark.gpu

OPQ = {"bf16": O.round_bf16, "fp16": O.round_fp16}
# gradient bars (see the module docstring).  FLOOR is per case: where R alone covers every tensor, 1e-3 of round-off allowance
R, REL_CAP, COS_CAP = 16.0, 0.18, 0.988
FLOOR = {"tiny_full": 3.5e-2, "tiny_txt_pos": 2e-2, "tiny_hl": 1.3e-2}
ATOMIC_TOL = dict(rtol=2e-3, atol=1e-6)  # fp32 atomics in the backward are order-dependent (tests/test_train_gpu.py)

GOLDEN = ("tiny_ragged", "tiny_full", "cfg2_b4_ragged", "cfg4_b4_ragged", "cfg2_full")
# name -> (config, batch, weight seed, input seed, model settings)
SYNTH = {
    # the reference's defaults, all three on: in-kernel input dropout, DropPath and attention dropout
    "cfg2_dropout": ("cfg2", 4, 77, 78, dict(input_dropout=0.5, droppath=0.1, dropout=0.1)),
    "tiny_txt_pos": ("tiny", 6, 61, 62, dict(use_txt_pos=True)),
    "tiny_hl": ("tiny", 6, 5, 9, dict(dset_type="hl")),
    "tiny_vs": ("tiny", None, 31, 32, dict(dset_type="vs")),
}
CASES = GOLDEN + tuple(SYNTH)


def _record(name, payload):
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "results")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, f"parity_bf16_{name}.json"), "w") as f:
            json.dump(payload, f, indent=1)
    except OSError:
        pass


def _cuda(d):
    return {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in d.items()}


def _case(name):
    """(cfg, state dict, raw inputs, targets, model settings, kind, head gain); raw inputs / targets are lists for 'vs' (three
    forwards and the frame mask as the last targets entry)."""
    if name in GOLDEN:
        cfg, sd, inp, tgt, z = load_golden(name)
        return cfg, sd, inp, tgt, dict(droppath=0.0, input_dropout=0.0), "plain", float(z["meta_head_gain"])
    cfg_name, batch, wseed, iseed, over = SYNTH[name]
    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=wseed)
    settings = dict(droppath=0.0, input_dropout=0.0)
    settings.update(over)
    if name == "tiny_vs":
        b = synth.make_qfvs_batch(cfg, iseed, 4, 24, (24, 24, 24, 10), 3, 5)
        return cfg, sd, list(b[:3]), list(b[3:6]) + [b[6]], settings, "vs", 1.0
    raw = synth.make_inputs(cfg, seed=iseed, ragged=True, batch=batch)
    tgt = synth.make_targets(raw, seed=iseed + 1)
    kind = "plain"
    if over.get("dropout", 0.0) > 0:
        kind = "drop"
    elif over.get("use_txt_pos"):
        kind = "txt_pos"
    elif over.get("dset_type") == "hl":
        kind = "hl"
        tgt = {"saliency_scores": tgt["saliency_scores"], "saliency_pos_labels": tgt["saliency_pos_labels"],
               "timestamp_mask": tgt["timestamp_mask"], "timestamp_window": 1 * (tgt["saliency_scores"] > 0)}
    return cfg, sd, raw, tgt, settings, kind, 1.0


def _build(cfg, sd, fmt, settings):
    if settings.get("dset_type") == "vs":
        from univtg_b200.qfvs import build_model as build
    else:
        build = build_model
    model, crit = build(synth.reference_args(cfg, device="cuda:0", operand_format=fmt, **settings))
    model.load_state_dict(sd, strict=True)
    return model.to("cuda:0").train(), crit.to("cuda:0").train()


def _kernel_step(cfg, sd, raw, tgt, settings, kind, fmt):
    """One forward + criterion + backward in `fmt`; returns (outputs, losses, {name: gradient or None}, model, criterion,
    draws)."""
    model, crit = _build(cfg, sd, fmt, settings)
    model.keep_last_draw = kind == "drop"
    torch.manual_seed(5)
    if kind == "vs":
        mask = tgt[3].cuda()
        outs = [model(**_cuda(inp)) for inp in raw]
        dicts = [crit(o, _cuda(t), mask) for o, t in zip(outs, tgt[:3])]
        loss = {k: dicts[0][k] + dicts[1][k] + dicts[2][k] for k in dicts[0]}
        out = outs[2]
    else:
        out = model(**_cuda(raw))
        loss = crit(out, _cuda(tgt))
    crit.weighted_total(loss).backward()
    torch.cuda.synchronize()
    draws = None
    if kind == "drop":
        scales, masks = model._last_draw
        draws = (scales.cpu(), [None if m is None else m.cpu() for m in masks], [m.cpu() for m in model._last_attn_draw])
    grads = {n: (None if p.grad is None else p.grad.detach().double().cpu()) for n, p in model.named_parameters()}
    out = {k: out[k].detach().double().cpu() for k in ("pred_logits", "pred_spans")}
    return out, {k: float(v.detach()) for k, v in loss.items()}, grads, model, crit, draws


def _oracle(cfg, sd, raw, tgt, kind, opq, draws, weights):
    """fp64 autograd through the oracle, on the GPU; opq: the 16-bit operand rounding to emulate (None: exact)."""
    leaves = {k: v.cuda().double().requires_grad_(True) for k, v in sd.items()}
    if kind == "vs":
        from oracle import qfvs_oracle as QO

        mask = tgt[3].cuda()
        dicts = [QO.criterion(O.forward(leaves, cfg, **_cuda(inp), opq=opq), _cuda(t), mask) for inp, t in zip(raw, tgt[:3])]
        loss = QO.gather(dicts, 1)
        out = None
    else:
        inp, tg = _cuda(raw), _cuda(tgt)
        if kind == "drop":
            scales, masks, amasks = draws
            out = AO.forward(leaves, cfg, **inp, dp_scale=scales.cuda(), drop_masks=[None if m is None else m.cuda() for m in masks],
                             attn_masks=[m.cuda() for m in amasks], opq=opq)
        elif kind == "txt_pos":
            out = TO.forward(leaves, cfg, **inp, opq=opq, use_txt_pos=True)
        else:
            out = O.forward(leaves, cfg, **inp, opq=opq)
        loss = O.criterion(out, tg, losses=("labels", "saliency") if kind == "hl" else ("spans", "labels", "saliency"))
    O.weighted_total(loss, weights).backward()
    grads = {k: (None if v.grad is None else v.grad.cpu()) for k, v in leaves.items()}
    out = None if out is None else {k: out[k].detach().cpu() for k in ("pred_logits", "pred_spans")}
    return out, {k: float(v.detach()) for k, v in loss.items()}, grads


@pytest.mark.parametrize("name", CASES)
def test_bf16_training_step_matches_oracle(name):
    cfg, sd, raw, tgt, settings, kind, gain = _case(name)
    out, loss, grads, model, crit, draws = _kernel_step(cfg, sd, raw, tgt, settings, kind, "bf16")
    assert model.grad_scale == 1.0
    weights = dict(crit.weight_dict)
    _, _, grads16, _, _, draws16 = _kernel_step(cfg, sd, raw, tgt, settings, kind, "fp16")
    if kind == "drop":  # the same torch seed: the same in-kernel draws in either format
        assert torch.equal(draws[0], draws16[0]) and all(torch.equal(a, b) for a, b in zip(draws[2], draws16[2]))
        assert all((a is None and b is None) or torch.equal(a, b) for a, b in zip(draws[1], draws16[1]))
    xout, xloss, xgrad = _oracle(cfg, sd, raw, tgt, kind, None, draws, weights)
    eout, eloss, egrad = _oracle(cfg, sd, raw, tgt, kind, OPQ["bf16"], draws, weights)
    _, _, hgrad = _oracle(cfg, sd, raw, tgt, kind, OPQ["fp16"], draws, weights)
    # outputs and losses: the bf16 bars of the forward tests
    if xout is not None:
        for k in ("pred_logits", "pred_spans"):
            torch.testing.assert_close(out[k], eout[k], rtol=2e-3 * gain, atol=5e-4 * gain, msg=lambda m: f"{name} {k} emulating: {m}")
            torch.testing.assert_close(out[k], xout[k], rtol=1e-2, atol=3e-3, msg=lambda m: f"{name} {k} exact: {m}")
    assert sorted(loss) == sorted(xloss)
    for k in xloss:
        assert abs(loss[k] - eloss[k]) <= 1e-3 * max(1.0, abs(eloss[k])), (name, k, loss[k], eloss[k])
        assert abs(loss[k] - xloss[k]) <= 1e-2 * max(1.0, abs(xloss[k])), (name, k, loss[k], xloss[k])
    rows = {}
    for n, g in grads.items():
        og = xgrad[n]
        if og is None or float(og.abs().max()) == 0.0:
            assert g is None or float(g.abs().max()) == 0.0, f"{name}: {n} must not receive a gradient"
            continue
        assert g is not None, f"{name}: {n} got no gradient"
        assert bool(torch.isfinite(g).all()), (name, n)
        rb, rh = _rel(g, egrad[n]), _rel(grads16[n], hgrad[n])
        rows[n] = dict(rel_bf16_emulating=rb, rel_fp16_emulating=rh, rel_bf16_exact=_rel(g, og), cos_bf16_exact=_cos(g, og),
                       rel_fp16_exact=_rel(grads16[n], og))
    _record(name, rows)
    floor = FLOOR.get(name, 1e-3)
    bad = {n: v for n, v in rows.items() if v["rel_bf16_emulating"] > R * v["rel_fp16_emulating"] + floor
           or v["rel_bf16_exact"] > REL_CAP or v["cos_bf16_exact"] < COS_CAP}
    assert not bad, f"{name}: bf16 gradient mismatch {bad}"


# ------------------------------------------------------------------------------------------------- loss-scale equivariance
def _atomic_params(model, cfg, inp):
    """Names of the parameters whose gradient the backward of this input shape reduces with fp32 atomics: every LayerNorm term,
    bias, token-type row, weightedpool.weight and final head conv (row kernels / GEMM column sums / head kernel), and each GEMM
    weight gradient whose launch the plan splits over K (choose_tile with the plan's problems, train.cu univtg_backward)."""
    lib = _lib.load_library()
    B, Lv, _ = inp["src_vid"].shape
    Lt = inp["src_txt"].shape[1]
    d, ff = cfg["hidden_dim"], cfg["dim_feedforward"]
    M, Mv, Mt, Mh = B * (Lv + Lt), B * Lv, B * Lt, B * (Lv + 1)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    kpad = lambda k: (k + 63) // 64 * 64  # noqa: E731

    def ksplit(probs, max_split):
        n = len(probs)
        Ms = (ctypes.c_int32 * n)(*[p[0] for p in probs])
        Ns = (ctypes.c_int32 * n)(*[p[1] for p in probs])
        Ks = (ctypes.c_int32 * n)(*[(p[2] + 63) // 64 for p in probs])
        bn, ks = ctypes.c_int32(0), ctypes.c_int32(0)
        _lib.check(lib.univtg_debug_choose_tile(Ms, Ns, Ks, n, sms, 64, max_split, ctypes.byref(bn), ctypes.byref(ks)), "choose_tile")
        return ks.value

    split = {}
    conv = ksplit([(d, d, Mh)] * 3, 8)
    for h in ("class_embed", "span_embed"):
        split[f"{h}.layers.0.weight"] = split[f"{h}.layers.1.weight"] = conv
    for l in range(cfg["enc_layers"]):
        pre = f"transformer.encoder.layers.{l}."
        split[pre + "linear1.weight"] = split[pre + "linear2.weight"] = ksplit([(d, ff, M), (ff, d, M)], 16)
        split[pre + "self_attn.out_proj.weight"] = ksplit([(d, d, M)], 16)
        split[pre + "self_attn.in_proj_weight"] = ksplit([(2 * d, d, M), (d, d, M)], 16)
    vdim, tdim = cfg["v_feat_dim"], cfg["t_feat_dim"]
    for i in range(cfg["n_input_proj"]):
        dinv, dint = (vdim, tdim) if i == 0 else (d, d)
        nv = kpad(dinv) if dinv % 8 else dinv
        split[f"input_vid_proj.{i}.net.1.weight"] = split[f"input_txt_proj.{i}.net.1.weight"] = ksplit([(d, nv, Mv), (d, dint, Mt)], 16)
    return {n for n, _ in model.named_parameters() if split.get(n, 2) > 1}


@pytest.mark.parametrize("name", ["tiny_ragged", "cfg2_b4_ragged", "cfg2_full"])
def test_bf16_gradients_are_loss_scale_equivariant(name):
    """L <= 128 and head size 128 in these cases: the attention backward writes dQ without atomics, so the atomics are the
    parameter-gradient reductions that _atomic_params lists."""
    cfg, sd, inp, tgt, _ = load_golden(name)
    assert inp["src_vid"].shape[1] + inp["src_txt"].shape[1] <= 128 and cfg["hidden_dim"] // cfg["nheads"] == 128
    model, crit = _build(cfg, sd, "bf16", dict(droppath=0.0, input_dropout=0.0))
    grads = []
    for scale in (1.0, 1024.0):
        model.grad_scale = scale
        for p in model.parameters():
            p.grad = None
        loss = crit(model(**_cuda(inp)), _cuda(tgt))
        crit.weighted_total(loss).backward()
        torch.cuda.synchronize()
        grads.append({n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None})
    atomic = _atomic_params(model, cfg, inp)
    assert sorted(grads[0]) == sorted(grads[1])
    exact = 0
    for n, g in grads[0].items():
        if n in atomic:
            torch.testing.assert_close(grads[1][n], g, **ATOMIC_TOL, msg=lambda m, n=n: f"{name} {n}: {m}")
        else:
            assert torch.equal(grads[1][n], g), (name, n, float((grads[1][n] - g).abs().max()))
            exact += 1
    assert exact >= 1 if name == "cfg2_full" else exact >= 4 * cfg["enc_layers"], (name, exact)


# ------------------------------------------------------------------------------------------------- optimizer and graph
def _train_inputs(cfg, batch, seed):
    raw = synth.make_inputs(cfg, seed=seed, ragged=True, batch=batch)
    tgt = synth.make_targets(raw, seed=seed + 1)
    return _cuda(raw), _cuda(tgt)


@pytest.mark.parametrize("cfg_name", ["tiny", "cfg1"])
def test_bf16_adamw_keeps_the_packed_operands_current(cfg_name):
    """Three bf16 FlatAdamW steps write the bf16 operand copies (kind 0 rows and kind 1 conv taps): a full re-pack from the
    fp32 parameters reproduces them byte for byte.  tiny: v_feat_dim 194, cfg1: 514 (rows straddle float4s)."""
    cfg = synth.CONFIGS[cfg_name]
    model, crit = _build(cfg, synth.make_state_dict(cfg, seed=3), "bf16", dict(droppath=0.0, input_dropout=0.0))
    inp, tgt = _train_inputs(cfg, 4, 41)
    opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-2, max_grad_norm=0.1)
    fmt = model._fmt(True)
    assert fmt == 1
    for _ in range(3):
        out = model(**inp)
        total = crit.weighted_total(crit(out, tgt))
        opt.zero_grad()
        total.backward()
        opt.step()
    kept = model._packed[fmt].clone()
    key = dict(model._packed_key)
    model._packed_key = {}
    model._ensure_packed(training=True)
    torch.cuda.synchronize()
    assert torch.equal(kept, model._packed[fmt])
    assert fmt in key and opt.step_count == 3


def _fill_grads(model, ref_params, gen, gscale=1e-3):
    flat, views = model._grad_buffer()
    flat.zero_()
    pos = {id(p): i for i, (_, p) in enumerate(model.named_parameters())}
    for v, p in zip(views, model._abi_params()):
        g = torch.randn(v.shape, device="cuda", generator=gen) * gscale
        v.copy_(g)
        ref_params[pos[id(p)]].grad = g.clone()


def test_bf16_flat_adamw_matches_torch_clip_plus_adamw():
    cfg = synth.CONFIGS["tiny"]
    model, _ = _build(cfg, synth.make_state_dict(cfg, seed=3), "bf16", dict(droppath=0.0, input_dropout=0.0))
    ref = [p.detach().clone().requires_grad_(True) for _, p in model.named_parameters()]
    opt_ref = torch.optim.AdamW(ref, lr=1e-3, weight_decay=1e-2)
    opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-2, max_grad_norm=0.1)
    gen = torch.Generator(device="cuda").manual_seed(11)
    for gscale in (3.0, 1e-4, 3.0, 1e-2):  # above / below the clip threshold
        _fill_grads(model, ref, gen, gscale)
        n_ref = torch.nn.utils.clip_grad_norm_(ref, 0.1)
        opt_ref.step()
        n = opt.step()
        assert abs(float(n) - float(n_ref)) <= 1e-5 * float(n_ref)
        for (n_, p), rp in zip(model.named_parameters(), ref):
            torch.testing.assert_close(p.detach(), rp.detach(), rtol=2e-5, atol=2e-7, msg=lambda m, n_=n_: f"{n_}: {m}")


DROPS = dict(input_dropout=0.5, droppath=0.1, dropout=0.1)


def _graph_models(cfg_name, n=2, qfvs=False, drops=DROPS, lr=1e-3):
    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=3)
    out = []
    for _ in range(n):
        model, crit = _build(cfg, sd, "bf16", dict(drops, dset_type="vs") if qfvs else dict(drops))
        out.append((model, crit, FlatAdamW(model, lr=lr, weight_decay=1e-2, max_grad_norm=0.1)))
    return out


@pytest.mark.parametrize("cfg_name", ["tiny", "cfg1"])
def test_bf16_six_replays_equal_six_eager_steps_with_the_replay_seeds(cfg_name):
    (mg, cg, og), (me, ce, oe) = _graph_models(cfg_name)
    gs = GraphedTrainStep(mg, cg, og)
    p0 = og._flat_p.clone()
    for k in range(1, 7):
        inp, tgt = _batch(cfg_name, 100 + k)
        _, lg = _graphed_call(gs, inp, tgt)  # losses and the update checked bit for bit against eager launches
        _, le = _eager_step(me, ce, oe, inp, tgt, rng_seed_at(gs.seed_base, k))
        torch.cuda.synchronize()
        assert og.step_count == oe.step_count == k and int(gs._step.item()) == k
        # the two trajectories differ in the parameters' last bits after step 1; bf16 operand rounding turns that into loss
        # differences 8x those of fp16 (measured: 2.2e-3 on cfg1): the fp16 test's rtol 2e-3 x 8
        torch.testing.assert_close(lg, le, rtol=1.6e-2, atol=1e-5)
    _close_trajectory(og._flat_p, oe._flat_p, p0)
    assert gs.num_graphs == 1


def test_bf16_qfvs_replays_equal_eager():
    cfg = synth.CONFIGS["tiny"]
    b = synth.make_qfvs_batch(cfg, 32, 4, 24, (24, 24, 24, 10), 3, 5)
    inp, tgt, mask = _cuda(b[0]), _cuda(b[3]), b[6].cuda()
    (mg, cg, og), (me, ce, oe) = _graph_models("tiny", qfvs=True)
    gs = GraphedTrainStep(mg, cg, og)
    p0 = og._flat_p.clone()
    for k in range(1, 4):
        _, lg = _graphed_call(gs, inp, tgt, mask)
        _, le = _eager_step(me, ce, oe, inp, tgt, rng_seed_at(gs.seed_base, k), mask)
        if k == 1:
            assert torch.equal(lg, le)  # same parameters, same masks
        torch.testing.assert_close(lg, le, rtol=1.6e-2, atol=1e-5)
    torch.cuda.synchronize()
    assert og.step_count == oe.step_count == 3
    _close_trajectory(og._flat_p, oe._flat_p, p0)


# ------------------------------------------------------------------------------------------------- skipped updates
@pytest.mark.parametrize("fmt", ["bf16", "fp16"])
def test_skipped_update_is_not_counted_without_dynamic_loss_scale(fmt):
    """A gradient buffer with one NaN: univtg_adamw_step leaves weights and moments untouched, and with a static loss scale
    (always in bf16; dynamic_loss_scale=False in fp16) the step count, skipped_steps and the checkpoint's 'step' still count
    real updates only - the next update equals torch.optim.AdamW that never saw the bad step."""
    cfg = synth.CONFIGS["tiny"]
    model, _ = _build(cfg, synth.make_state_dict(cfg, seed=3), fmt, dict(droppath=0.0, input_dropout=0.0))
    ref = [p.detach().clone().requires_grad_(True) for _, p in model.named_parameters()]
    opt_ref = torch.optim.AdamW(ref, lr=1e-3, weight_decay=1e-2)
    opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-2, max_grad_norm=0.0, dynamic_loss_scale=False)
    assert not opt.dynamic_loss_scale
    scale = model.grad_scale
    gen = torch.Generator(device="cuda").manual_seed(21)

    def check():
        for (n_, p), rp in zip(model.named_parameters(), ref):
            torch.testing.assert_close(p.detach(), rp.detach(), rtol=2e-5, atol=2e-7, msg=lambda m, n_=n_: f"{n_}: {m}")

    _fill_grads(model, ref, gen)
    opt.step()
    opt_ref.step()
    torch.cuda.synchronize()
    before = [p.detach().clone() for p in model._abi_params()]
    m0, v0 = opt._m.clone(), opt._v.clone()
    _fill_grads(model, [r.detach().clone() for r in ref], gen)  # (the reference optimizer never sees this batch)
    model._grad_buffer()[1][5].view(-1)[7] = float("nan")
    opt.step()
    torch.cuda.synchronize()
    assert float(opt._scratch[2]) == 1.0
    assert all(torch.equal(p.detach(), b) for p, b in zip(model._abi_params(), before))
    assert torch.equal(opt._m, m0) and torch.equal(opt._v, v0)
    sd = opt.state_dict()  # right after the skipped step: the checkpoint counts one update
    assert opt.step_count == 1 and opt.skipped_steps == 1
    assert {float(s["step"]) for s in sd["state"].values()} == {1.0} and sd["loss_scale"]["skipped_steps"] == 1
    for _ in range(3):
        _fill_grads(model, ref, gen)
        opt.step()
        opt_ref.step()
        torch.cuda.synchronize()
        check()  # a bias correction one step ahead moves these updates by > 10 %
    sd = opt.state_dict()
    assert opt.step_count == 4 and opt.skipped_steps == 1 and model.grad_scale == scale
    assert {float(s["step"]) for s in sd["state"].values()} == {4.0}
    ref_sd = opt_ref.state_dict()
    assert {float(s["step"]) for s in ref_sd["state"].values()} == {4.0}


def _nan_batch(inp):
    bad = {k: v.clone() for k, v in inp.items()}
    row = int(torch.nonzero(bad["src_vid_mask"][0]).flatten()[-1])  # a valid frame of sample 0
    bad["src_vid"][0, row, 3] = float("nan")
    return bad


def test_bf16_skipped_step_graph_eager_and_mixed_agree():
    """good batch, a batch with one NaN in a valid src_vid entry (its update is skipped), then good batches: graphed, eager
    and graph / eager / graph runs end with the same step count, parameters, moments and state_dict()."""
    runs = _graph_models("tiny", n=3, drops=dict(input_dropout=0.0, droppath=0.0, dropout=0.0))
    batches = [_batch("tiny", 500 + i) for i in range(5)]
    batches[1] = (_nan_batch(batches[1][0]), batches[1][1])
    (mg, cg, og), (me, ce, oe), (mm, cm, om) = runs
    gs, gm = GraphedTrainStep(mg, cg, og), GraphedTrainStep(mm, cm, om)
    p0 = og._flat_p.clone()
    for k, (inp, tgt) in enumerate(batches):
        gs(inp, tgt)
        _eager_step(me, ce, oe, inp, tgt, None)
        if k in (1, 3):
            _eager_step(mm, cm, om, inp, tgt, None)
        else:
            gm(inp, tgt)
        torch.cuda.synchronize()
        if k == 1:
            for opt in (og, oe, om):
                assert float(opt._scratch[2]) == 1.0, "the NaN batch must be skipped"
    sds = [o.state_dict() for o in (og, oe, om)]
    for opt, sd in zip((og, oe, om), sds):
        assert opt.step_count == 4 and opt.skipped_steps == 1, (opt.step_count, opt.skipped_steps)
        assert {float(s["step"]) for s in sd["state"].values()} == {4.0}
    assert int(gs._step.item()) == int(gm._step.item()) == 4
    for a in (og, om):
        _close_trajectory(a._flat_p, oe._flat_p, p0)
        for t in ("_m", "_v"):
            torch.testing.assert_close(getattr(a, t), getattr(oe, t), **ATOMIC_TOL)
    for sd in sds[1:]:
        assert sd["param_groups"] == sds[0]["param_groups"] and sd["loss_scale"] == sds[0]["loss_scale"]


def test_bf16_step_captured_whole_in_a_cuda_graph():
    """The whole eager step - forward, criterion, backward, FlatAdamW.step - captured in one torch CUDA graph with a static loss
    scale (bench.py's graph probe): the step reads no skip flag inside the capture, and the replays train."""
    cfg = synth.CONFIGS["tiny"]
    model, crit = _build(cfg, synth.make_state_dict(cfg, seed=3), "bf16", dict(droppath=0.0, input_dropout=0.0))
    opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-2, max_grad_norm=0.1)
    inp, tgt = _train_inputs(cfg, 4, 41)

    def step():
        total = crit.weighted_total(crit(model(**inp), tgt))
        opt.zero_grad(set_to_none=True)
        total.backward()
        opt.step()
        return total

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.synchronize()
    model.__dict__.pop("_grad_anchor", None)  # (the capture makes its own autograd anchor, as GraphedTrainStep's does)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=side):
        total = step()
    torch.cuda.current_stream().wait_stream(side)
    graph.replay()
    torch.cuda.synchronize()
    first = float(total)
    p0 = opt._flat_p.clone()
    for _ in range(8):
        graph.replay()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(opt._flat_p).all()) and not torch.equal(opt._flat_p, p0)
    assert float(total) < first
    step()  # an eager step after the replays consumes the warm-up's flag as usual
    torch.cuda.synchronize()
    assert opt.skipped_steps == 0
