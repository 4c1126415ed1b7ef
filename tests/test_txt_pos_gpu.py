"""Learned text positions (args.use_txt_pos) on the GPU: pos_t = Dropout(LayerNorm(x_t + P[l])) is computed by one row kernel after
the projectors and added to the text rows of every encoder layer's q/k operand; the backward accumulates the q/k-half dgrad of
the text rows over the layers and runs the LayerNorm / dropout backward into the three txt_position_embed gradients and the
stream gradient of x_t.  The yardstick is tests/txt_pos_oracle.py (pinned to the reference by tests/test_txt_pos_cpu.py), fed
the multipliers the kernels applied (read back through univtg_dropout_mask)."""
import ctypes

import pytest
import torch

from oracle import univtg_oracle as O
from tests import txt_pos_oracle as TO
from tests.test_train_gpu import WD, _cos, _grad_verdict, _record, _rel
from univtg_b200 import _lib, build_model, ddp, synth
from univtg_b200.optim import FlatAdamW

pytestmark = pytest.mark.gpu

TINY = synth.CONFIGS["tiny"]
OUT_KEYS = ("pred_logits", "pred_spans", "saliency_scores", "vid_mem_proj", "txt_mem_proj")
TP_NAMES = ("txt_position_embed.position_embeddings.weight", "txt_position_embed.LayerNorm.weight",
            "txt_position_embed.LayerNorm.bias")


def _model(cfg, seed=61, **over):
    args = dict(device="cuda:0", use_txt_pos=True, dropout=0.0, input_dropout=0.0, droppath=0.0)
    args.update(over)
    model, crit = build_model(synth.reference_args(cfg, **args))
    model.load_state_dict(synth.make_state_dict(cfg, seed=seed), strict=True)
    return model.to("cuda:0"), crit.to("cuda:0")


def _inputs(cfg, batch, seed=62):
    raw = synth.make_inputs(cfg, seed=seed, ragged=True, batch=batch)
    tgt = synth.make_targets(raw, seed=seed + 1)
    return raw, tgt, {k: v.cuda() for k, v in raw.items()}, {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in tgt.items()}


# ---------------------------------------------------------------------------------------------------------------- inference
EVAL_CASES = {
    "tiny": (TINY, 6, "fp16"),                     # dh = 128, L = 30: one key tile
    "tiny_long": (dict(TINY, l_vid=200), 3, "fp16"),  # L = 209: two key tiles
    "cfg1": (synth.CONFIGS["cfg1"], 3, "fp16"),    # dh = 32: SIMT attention, d = 256
    "cfg2_b32": (synth.CONFIGS["cfg2"], 32, "fp16"),  # the benchmarked shape, d = 1024
    "tiny_bf16": (TINY, 6, "bf16"),
}


@pytest.mark.parametrize("name", list(EVAL_CASES))
def test_eval_matches_oracle(name):
    cfg, batch, fmt = EVAL_CASES[name]
    raw, _, inp, _ = _inputs(cfg, batch)
    model, _ = _model(cfg, operand_format=fmt)
    model.eval()
    with torch.no_grad():
        out = model(**inp)
    sd = synth.make_state_dict(cfg, seed=61)
    opq = O.round_fp16 if fmt == "fp16" else O.round_bf16
    eo = TO.forward(sd, cfg, **raw, opq=opq, use_txt_pos=True)
    xo = TO.forward(sd, cfg, **raw, use_txt_pos=True)
    off = TO.forward(sd, cfg, **raw)
    loose = 10.0 if fmt == "bf16" else 1.0
    for k in ("pred_logits", "pred_spans", "saliency_scores"):
        got = out[k].double().cpu()
        torch.testing.assert_close(got, eo[k], rtol=2e-4 * loose, atol=5e-5 * loose, msg=lambda m: f"{name} {k} emulating: {m}")
        torch.testing.assert_close(got, xo[k], rtol=1e-3 * loose, atol=2e-4 * loose, msg=lambda m: f"{name} {k} exact: {m}")
    assert not torch.allclose(xo["pred_spans"], off["pred_spans"], rtol=1e-4, atol=1e-5)  # the positions matter here


def test_graph_replay_is_eager_and_follows_parameter_changes():
    cfg = TINY
    raw, tgt, inp, tgt_c = _inputs(cfg, 6)
    model, crit = _model(cfg)
    model.eval()

    def eager():
        model.use_cuda_graphs = False
        with torch.no_grad():
            return {k: v.clone() for k, v in model(**inp).items() if torch.is_tensor(v)}

    def graphed():
        model.use_cuda_graphs = True
        with torch.no_grad():
            o = model(**inp)
            o2 = model(**inp)  # a replay, not the capture
        return o2

    def same():
        e, g = eager(), graphed()
        for k in OUT_KEYS:
            assert torch.equal(e[k], g[k]), k
        return e

    base = same()
    tp = model.txt_position_embed
    with torch.no_grad():  # in-place edit of the table: same storage, new values
        tp.position_embeddings.weight.mul_(1.5)
    edited = same()
    assert not torch.equal(edited["pred_spans"], base["pred_spans"])
    model.load_state_dict(synth.make_state_dict(cfg, seed=61), strict=True)
    assert torch.equal(same()["pred_spans"], base["pred_spans"])
    # a FlatAdamW step re-seats every parameter as a view of its flat buffer and updates the text-position tensors
    opt = FlatAdamW(model, lr=1e-2, weight_decay=0.0)
    model.train()
    out = model(**inp)
    loss = crit(out, tgt_c)
    sum(loss[k] * crit.weight_dict[k] for k in loss).backward()
    before = tp.LayerNorm.bias.detach().clone()
    opt.step()
    torch.cuda.synchronize()
    assert not torch.equal(before, tp.LayerNorm.bias.detach())
    model.eval()
    stepped = same()
    assert not torch.equal(stepped["pred_spans"], base["pred_spans"])
    sd = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    ref = TO.forward(sd, cfg, **raw, opq=O.round_fp16, use_txt_pos=True)
    torch.testing.assert_close(stepped["pred_spans"].double().cpu(), ref["pred_spans"], rtol=2e-4, atol=5e-5)


# ---------------------------------------------------------------------------------------------------------------- training
# name: (config, batch, input_dropout, droppath, attention dropout, reference_rng_order)
TRAIN_CASES = {
    "tiny_p0": (TINY, 6, 0.0, 0.0, 0.0, False),
    "tiny_p05": (TINY, 6, 0.5, 0.0, 0.0, False),
    # L = 209: the atomic-dQ attention backward, whose fp32 -> 16-bit pass copies the text rows.  Input dropout stays off here: with
    # p = 0.5 the kernels agree with the fp16-emulating oracle to 0.35 %, but input_vid_proj.0's gradients sit 6.7 % from the
    # exact one (H100, 700 W) - fp16 operand rounding of the x2-scaled 194-wide video features, not the text positions
    "tiny_long": (dict(TINY, l_vid=200), 3, 0.0, 0.0, 0.0, False),
    "cfg1_p05": (synth.CONFIGS["cfg1"], 3, 0.5, 0.0, 0.0, False),
    "tiny_reference_order": (TINY, 6, 0.5, 0.1, 0.0, True),
    "cfg2_defaults": (synth.CONFIGS["cfg2"], 4, 0.5, 0.1, 0.1, False),
}
# gradient bar of _grad_verdict (within NEAR_TOL of one of the two oracles): the attention-dropout tests' values
NEAR_TOL = {"cfg2_defaults": 2.2e-2}


def _train_step(model, crit, inp, tgt_c, seed=5):
    model.train()
    crit.train()
    model.keep_last_draw = True
    torch.manual_seed(seed)
    out = model(**inp)
    loss = crit(out, tgt_c)
    sum(loss[k] * crit.weight_dict[k] for k in loss).backward()
    torch.cuda.synchronize()
    scales, masks = model._last_draw
    return out, loss, scales, masks, model._last_attn_draw, model._last_txt_pos_draw


def _oracle(cfg, raw, tgt, scales, masks, amasks, tmul, opq, seed=61):
    sd = synth.make_state_dict(cfg, seed=seed)
    leaves = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    o = TO.forward(leaves, cfg, **raw, dp_scale=None if scales is None else scales.cpu(),
                   drop_masks=[None if m is None else m.cpu() for m in masks],
                   attn_masks=None if amasks is None else [m.cpu() for m in amasks], opq=opq, use_txt_pos=True,
                   txt_pos_mul=None if tmul is None else tmul.cpu())
    ls = O.criterion(o, tgt)
    O.weighted_total(ls, WD).backward()
    return o, ls, {k: v.grad for k, v in leaves.items()}


@pytest.mark.parametrize("name", list(TRAIN_CASES))
def test_training_matches_oracle_fed_the_same_draws(name):
    cfg, batch, idrop, dpath, adrop, ref_order = TRAIN_CASES[name]
    raw, tgt, inp, tgt_c = _inputs(cfg, batch, 78)
    model, crit = _model(cfg, seed=77, input_dropout=idrop, droppath=dpath, dropout=adrop)
    model.reference_rng_order = ref_order
    out, loss, scales, masks, amasks, tmul = _train_step(model, crit, inp, tgt_c)
    B, Lt, d = batch, raw["src_txt"].shape[1], cfg["hidden_dim"]
    if idrop > 0:
        assert tuple(tmul.shape) == (B, Lt, d) and bool((tmul == 0).any())
    else:
        assert tmul is None
    eout, eloss, egrad = _oracle(cfg, raw, tgt, scales, masks, amasks, tmul, O.round_fp16, seed=77)
    xout, xloss, xgrad = _oracle(cfg, raw, tgt, scales, masks, amasks, tmul, None, seed=77)
    for k in ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj"):
        got = out[k].detach().double().cpu()
        tight = k.startswith("pred")
        torch.testing.assert_close(got, eout[k].detach(), rtol=2e-4 if tight else 5e-4, atol=5e-5 if tight else 5e-4,
                                   msg=lambda m: f"{name} {k} vs emulating oracle: {m}")
        torch.testing.assert_close(got, xout[k].detach(), rtol=1e-3, atol=1e-4 if tight else 2e-3,
                                   msg=lambda m: f"{name} {k} vs exact oracle: {m}")
    for k in xloss:
        lk, ek, xk = float(loss[k].detach()), float(eloss[k].detach()), float(xloss[k].detach())
        assert abs(lk - ek) <= 1e-4 * max(1.0, abs(ek)), (name, k)
        assert abs(lk - xk) <= 1e-3 * max(1.0, abs(xk)), (name, k)
    worst = {}
    for n_, prm in model.named_parameters():
        if xgrad[n_] is None or float(xgrad[n_].abs().max()) == 0.0:
            continue
        g = prm.grad.double().cpu()
        assert bool(torch.isfinite(g).all()), n_
        worst[n_] = (_rel(g, xgrad[n_]), _cos(g, xgrad[n_]), _rel(g, egrad[n_]))
    assert all(n_ in worst for n_ in TP_NAMES), sorted(worst)
    table = dict(model.named_parameters())[TP_NAMES[0]].grad
    assert float(table[Lt:].abs().max()) == 0.0  # rows beyond Lt get exactly zero
    _record(f"txt_pos_{name}", {k: {"rel_exact": v[0], "cos_exact": v[1], "rel_emulating": v[2]} for k, v in worst.items()})
    bad = _grad_verdict(worst, NEAR_TOL.get(name, 5e-2))
    assert not bad, f"{name}: gradient mismatch with text positions {bad}"


def test_dropout_multiplier_statistics_and_reproducibility():
    lib = _lib.load_library()
    cfg = TINY
    model, _ = _model(cfg, input_dropout=0.5)
    B, Lt, d, n = 64, 32, cfg["hidden_dim"], cfg["n_input_proj"]

    def draw(seed, index):
        rng = _lib.Rng(seed, 0.5, 0.0)
        m = torch.empty(B * Lt, d, device="cuda:0")
        _lib.check(lib.univtg_dropout_mask(ctypes.byref(rng), index, B * Lt, d, _lib.ptr(m), _lib.stream_ptr()), "univtg_dropout_mask")
        return m

    m = draw(1234567, 2 * n)
    assert bool(((m == 0) | (m == 2.0)).all())
    keep = (m != 0).float()
    N = keep.numel()
    assert abs(float(keep.mean()) - 0.5) < 4.0 * (0.25 / N) ** 0.5 + 2e-5
    tol = 4.0 * (0.25 / N) ** 0.5 * 2
    k = keep.bool()
    for a, b in ((k[:, :-1], k[:, 1:]), (k[:-1], k[1:]), (k[:, :-8], k[:, 8:])):  # columns, rows, the 8-column Philox block
        assert abs(float((a == b).float().mean()) - 0.5) < tol
    for other in range(2 * n):  # independent of every projector mask of the same step
        assert abs(float(((draw(1234567, other)[:, :d] != 0) == k).float().mean()) - 0.5) < tol
    # the same torch seed gives a bit-identical train-mode forward
    raw, tgt, inp, tgt_c = _inputs(cfg, 6)
    model.train()
    runs = []
    for _ in range(2):
        torch.manual_seed(9)
        with torch.no_grad():
            runs.append({k_: v.clone() for k_, v in model(**inp).items() if torch.is_tensor(v)})
    for k_ in OUT_KEYS:
        assert torch.equal(runs[0][k_], runs[1][k_]), k_


@pytest.mark.parametrize("fmt", ["fp16", "bf16"])
@pytest.mark.parametrize("nheads", [2, 8])
def test_eval_equals_train_without_dropout_and_one_more_launch(nheads, fmt):
    cfg = dict(TINY, nheads=nheads)
    model, _ = _model(cfg, seed=31, operand_format=fmt)
    plain, _ = _model(cfg, seed=31, operand_format=fmt, use_txt_pos=False)
    inp = {k: v.cuda() for k, v in synth.make_inputs(cfg, seed=32, ragged=True).items()}
    B, Lv, _ = inp["src_vid"].shape
    Lt = inp["src_txt"].shape[1]
    lib = _lib.load_library()

    def counted(m):
        torch.cuda.synchronize()
        n0 = lib.univtg_launch_count()
        o = m(**inp)
        torch.cuda.synchronize()
        return o, lib.univtg_launch_count() - n0

    model.eval()
    with torch.no_grad():
        model(**inp)
        ev, n_eval = counted(model)
    model.train()
    model(**inp)
    tr, n_train = counted(model)
    assert n_eval == n_train == model.num_forward_launches(B, Lv, Lt) == plain.num_forward_launches(B, Lv, Lt) + 1
    for k in OUT_KEYS:
        assert torch.equal(ev[k], tr[k].detach()), k


def test_flat_adamw_matches_clip_and_torch_adamw_and_state_dicts_interchange():
    cfg = TINY
    raw, tgt, inp, tgt_c = _inputs(cfg, 6)
    model, crit = _model(cfg)
    ref, _ = _model(cfg)
    opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-4, max_grad_norm=0.1, dynamic_loss_scale=False)
    topt = torch.optim.AdamW([p for _, p in ref.named_parameters()], lr=1e-3, weight_decay=1e-4)
    rp = dict(ref.named_parameters())
    for _ in range(3):
        model.train()
        opt.zero_grad()
        out = model(**inp)
        loss = crit(out, tgt_c)
        sum(loss[k] * crit.weight_dict[k] for k in loss).backward()
        torch.cuda.synchronize()
        for n_, p in model.named_parameters():  # the reference optimiser sees the same gradients
            rp[n_].grad = p.grad.detach().clone()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), 0.1)
        opt.step()
        topt.step()
        torch.cuda.synchronize()
    for n_, p in model.named_parameters():
        torch.testing.assert_close(p.detach(), rp[n_].detach(), rtol=2e-5, atol=2e-7, msg=lambda m, n_=n_: f"{n_}: {m}")
    assert not torch.equal(model.txt_position_embed.LayerNorm.weight.detach(),
                           synth.make_state_dict(cfg, seed=61)["txt_position_embed.LayerNorm.weight"].cuda())
    # FlatAdamW -> torch.optim.AdamW and back
    sd = opt.state_dict()
    names = [n_ for n_, _ in model.named_parameters()]
    for i in (names.index(t) for t in TP_NAMES):
        assert i in sd["state"], names[i]
    t2 = torch.optim.AdamW([p for _, p in ref.named_parameters()], lr=1e-3)
    t2.load_state_dict(sd)
    opt2 = FlatAdamW(model, lr=1e-3)
    opt2.load_state_dict(topt.state_dict())
    assert opt2.step_count == 3


def test_grad_stage_slices_cover_the_enlarged_buffer_once():
    model, _ = _model(TINY)
    flat, _ = model._grad_buffer()
    offs = model._grad_offsets()
    seen = torch.zeros(flat.numel(), dtype=torch.int32)
    for _, sl in ddp.grad_stage_slices(model):
        for lo, hi in sl:
            seen[lo:hi] += 1
    for i in range(len(offs) - 1):
        assert int(seen[offs[i]:offs[i + 1]].min()) == 1 and int(seen[offs[i]:offs[i + 1]].max()) == 1, i
    stages = ddp.grad_stage_slices(model)
    assert (offs[-4], offs[-1]) in stages[len(stages) - 2][1]


def test_refusals():
    cfg = TINY
    _, _, inp, tgt_c = _inputs(cfg, 3)
    model, _ = build_model(synth.reference_args(cfg, device="cuda:0", use_txt_pos=True, max_q_l=8))
    model.to("cuda:0")
    with pytest.raises(ValueError, match="exceed max_q_l = 8"):
        model(**inp)  # Lt = 9
    # the C ABI refuses the same, and a backward whose gradient count does not match the setting
    lib = _lib.load_library()
    model, crit = _model(cfg)
    model.train()
    out = model(**inp)
    loss = crit(out, tgt_c)
    plan = next(e for k, e in model._plans.items() if k[3] == 1)
    tp = model.txt_position_embed
    scratch = torch.empty(1 << 20, dtype=torch.uint8, device="cuda:0")
    st = _lib.TxtPos(tp.position_embeddings.weight.data_ptr(), 8, tp.LayerNorm.weight.data_ptr(), tp.LayerNorm.bias.data_ptr(),
                     None, scratch.data_ptr())
    assert lib.univtg_plan_set_txt_pos(plan.handle, ctypes.byref(st)) != 0
    assert "max_q_l = 8" in _lib.last_error()
    n = lib.univtg_num_params(ctypes.byref(model._cfg))
    model._arm_txt_pos(plan, None, torch.empty(1 << 20, dtype=torch.uint8, device="cuda:0"))
    one = torch.zeros(4, device="cuda:0")
    for count in (n, n + 2):  # the three text-position gradients missing, or one short
        arr = (ctypes.c_void_p * count)(*([one.data_ptr()] * count))
        rc = lib.univtg_backward(plan.handle, _lib.ptr(one), _lib.ptr(one), _lib.ptr(one), None, None, None, None, None, None, None,
                                 1.0, arr, count, _lib.stream_ptr())
        assert rc != 0 and f"expected {n + 3} gradient tensors" in _lib.last_error()
