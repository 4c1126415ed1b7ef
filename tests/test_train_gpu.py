"""GPU parity of the training path: criterion values, output gradients and parameter gradients against the fp64 oracle
(autograd through oracle/univtg_oracle.py) and against the reference's golden gradient summaries.

Tolerances (see DESIGN.md 'Precision'; measured with tools/train_diag.py): the forward's fp16 operand rounding alone moves
exact gradients by 1-3.5 % (ReLU / LayerNorm / InfoNCE with temperature 0.07 amplify it), the fp16 loss-scaled backward adds
0.1-2 %.  So: per-tensor relative L2 error <= 5e-2 and cosine >= 0.998 against exact fp64 gradients; loss values match the exact oracle to 1e-3 and the emulating one to
1e-4; the criterion kernels alone (fed with oracle outputs) match the oracle to fp32 round-off."""
import pytest
import torch

from tests.helpers import golden_out, load_golden
from univtg_b200 import build_model, synth

pytestmark = pytest.mark.gpu

WD = {"loss_b": 10.0, "loss_g": 1.0, "loss_f": 10.0, "loss_s_intra": 0.1, "loss_s_inter": 0.1}


def _models(cfg, sd, **over):
    model, crit = build_model(synth.reference_args(cfg, device="cuda:0", droppath=0.0, input_dropout=0.0, **over))
    model.load_state_dict(sd, strict=True)
    return model.to("cuda:0"), crit.to("cuda:0")


def _oracle_grads(cfg, sd, inp, tgt, dp_scale=None, emulate=False):
    from oracle import univtg_oracle as O

    leaves = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    out = O.forward(leaves, cfg, **inp, dp_scale=dp_scale, opq=O.round_fp16 if emulate else None)
    loss = O.criterion(out, tgt)
    total = O.weighted_total(loss, WD)
    total.backward()
    return out, loss, {k: (v.grad if v.grad is not None else None) for k, v in leaves.items()}


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _cos(a, b):
    return float((a.flatten() @ b.flatten()) / (a.norm() * b.norm()).clamp_min(1e-30))


@pytest.mark.parametrize("name", ["tiny_ragged", "tiny_full", "cfg2_b4_ragged"])
def test_criterion_kernels_match_oracle(name):
    """Loss kernels in isolation: feed the oracle's own outputs; values and output-gradients must match to fp32 round-off."""
    from oracle import univtg_oracle as O

    cfg, sd, inp, tgt, z = load_golden(name)
    out = O.forward(sd, cfg, **inp)
    leaves = {k: out[k].clone().requires_grad_(True) for k in ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj")}
    ref = O.criterion(leaves, tgt)
    O.weighted_total(ref, WD).backward()
    _, crit = _models(cfg, sd)
    cuda_out = {k: v.detach().float().cuda().requires_grad_(True) for k, v in leaves.items()}
    got = crit(cuda_out, {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in tgt.items()})
    for k in ref:
        assert abs(float(got[k]) - float(ref[k])) <= 2e-5 * max(1.0, abs(float(ref[k]))), (name, k, float(got[k]), float(ref[k]))
        assert abs(float(got[k]) - float(z["loss_" + k])) <= 2e-5 * max(1.0, abs(float(z["loss_" + k]))), (name, k)
    sum(got[k] * WD[k] for k in got).backward()
    for k, v in leaves.items():
        g = cuda_out[k].grad.double().cpu()
        assert _rel(g, v.grad) < 2e-4, (name, k, _rel(g, v.grad))


def _record(name, payload):
    """Measured parity numbers are also written to results/parity_<name>.json (scratch, ignored by git)."""
    import json
    import os

    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "results")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, f"parity_{name}.json"), "w") as f:
            json.dump(payload, f, indent=1)
    except OSError:
        pass


# Gradient acceptance (per parameter tensor, against fp64 autograd through the oracle).  Two references:
#   exact      fp64 everywhere.  16-bit operand rounding of the FORWARD alone moves exact gradients by 1 - 3.5 % (DESIGN.md
#              section 3: ReLU / LayerNorm / InfoNCE at temperature 0.07 amplify it) - a property of the format.
#   emulating  the same fp16 operand rounding in the forward, straight-through in its backward.  Its own gradient sits 1 - 3 % from
#              the exact one, on the other side of some tensors (measured, results/parity_grads_*.json): neither reference is
#              uniformly "closer to what the kernels should produce".
# Required: within 5 % (rel-L2) and cosine >= 0.998 of the exact reference, within 6 % of the emulating one, and within
# NEAR_TOL of at least one of them (what is left then is the fp16 loss-scaled backward + fp32 accumulation order).
NEAR_TOL = {"tiny_ragged": 2.5e-2, "tiny_full": 2.5e-2, "cfg2_b4_ragged": 1.6e-2, "cfg2_full": 1.2e-2, "cfg4_b4_ragged": 2e-2}


def _grad_verdict(worst, near_tol):
    return {k: v for k, v in worst.items() if v[0] > 5e-2 or v[1] < 0.998 or v[2] > 6e-2 or min(v[0], v[2]) > near_tol}


@pytest.mark.parametrize("name", ["tiny_ragged", "tiny_full", "cfg2_b4_ragged", "cfg4_b4_ragged", "cfg2_full"])
def test_full_training_step_gradients(name):
    """Forward + criterion + backward of one batch against the oracle's autograd.  cfg2_full is the benchmarked shape (B = 32,
    M = 3424: split-K weight gradients with fp32 reductions, 3-D-TMA MN-major operands); cfg4_b4_ragged has L = 182, i.e. two
    key tiles in the attention forward and the atomic dQ path in its backward."""
    cfg, sd, inp, tgt, z = load_golden(name)
    model, crit = _models(cfg, sd)
    model.train()
    crit.train()
    out = model(**{k: v.cuda() for k, v in inp.items()})
    loss = crit(out, {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in tgt.items()})
    total = sum(loss[k] * crit.weight_dict[k] for k in loss)
    total.backward()
    torch.cuda.synchronize()
    _, oloss, ograd = _oracle_grads(cfg, sd, inp, tgt)
    eout, eloss, egrad = _oracle_grads(cfg, sd, inp, tgt, emulate=True)
    for k in oloss:
        assert abs(float(loss[k]) - float(oloss[k])) <= 1e-3 * max(1.0, abs(float(oloss[k]))), (name, k)
        assert abs(float(loss[k]) - float(eloss[k])) <= 1e-4 * max(1.0, abs(float(eloss[k]))), (name, k)
        assert abs(float(loss[k]) - float(z["loss_" + k])) <= 1e-3 * max(1.0, abs(float(z["loss_" + k]))), (name, k)
    # train-mode forward (droppath = input_dropout = 0) against the emulating oracle and the reference fixture
    gain = float(z["meta_head_gain"])  # tiny_full: final conv weights x 4 (trained-checkpoint-like logits) amplify rounding alike
    for k in ("pred_logits", "pred_spans"):
        torch.testing.assert_close(out[k].detach().double().cpu(), eout[k].detach(), rtol=2e-4 * gain, atol=5e-5 * gain)
        torch.testing.assert_close(out[k].detach().float().cpu(), golden_out(z, k), rtol=1e-3, atol=1e-4)
    worst = {}
    for n_, p in model.named_parameters():
        og = ograd[n_]
        if og is None or float(og.abs().max()) == 0.0:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, f"{n_} must not receive a gradient"
            continue
        assert p.grad is not None, f"{n_} got no gradient"
        g = p.grad.double().cpu()
        assert bool(torch.isfinite(g).all()), n_
        worst[n_] = (_rel(g, og), _cos(g, og), _rel(g, egrad[n_]))
        # fixtures from the live reference (fp32): gradient norm and the first 16 entries of every parameter gradient
        gn = float(z["gnorm_" + n_])
        if gn > 1e-8:
            assert abs(float(g.norm()) - gn) <= 5e-2 * gn, (name, n_, float(g.norm()), gn)
        gh = torch.from_numpy(z["ghead_" + n_]).double()
        rms = gn / max(1.0, g.numel() ** 0.5)  # sixteen individual entries: allow 5 % of a typical entry each on top of 8 % relative
        assert float((g.flatten()[:16] - gh).norm()) <= 8e-2 * float(gh.norm()) + 5e-2 * rms * 4.0, (name, n_)
    _record("grads_" + name, {k: {"rel_exact": v[0], "cos_exact": v[1], "rel_emulating": v[2]} for k, v in worst.items()})
    bad = _grad_verdict(worst, NEAR_TOL[name])
    assert not bad, f"{name}: gradient mismatch (rel-L2 exact, cosine exact, rel-L2 emulating) {bad}"


def _train_inputs(cfg, batch, seed):
    raw = synth.make_inputs(cfg, seed=seed, ragged=True, batch=batch)
    tgt = synth.make_targets(raw, seed=seed + 1)
    return raw, tgt, {k: v.cuda() for k, v in raw.items()}, {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in tgt.items()}


@pytest.mark.parametrize("cfg_name,batch,mode", [("tiny", 6, "reference_order"), ("tiny", 6, "in_kernel"), ("cfg2", 4, "in_kernel"),
                                                 ("cfg2", 4, "reference_order")])
def test_input_dropout_and_droppath_match_oracle_fed_the_same_draws(cfg_name, batch, mode):
    """The benchmarked arm: train mode with input_dropout = 0.5 and droppath = 0.1 (reference defaults).
    mode 'in_kernel' (default of the plugin, what bench.py times): the multipliers are generated inside the LayerNorm / sine-pos
    kernels from a per-forward seed (Philox) and regenerated by the backward; the test reads them back through
    univtg_dropout_mask / univtg_droppath_scales.  mode 'reference_order': the glue draws them with the reference's own torch
    calls in the reference's order (F.dropout per projector layer - model/univtg.py:394 -, then one torch.rand((B,1,1)) per
    DropPath site - transformer_encoder_droppath.py:154-167).  Either way the oracle is fed the same tensors (its mask semantics
    are pinned to the live reference by tests/test_oracle_vs_reference.py): forward, losses and gradients must agree."""
    from oracle import univtg_oracle as O

    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=77)
    raw, tgt, inp, tgt_c = _train_inputs(cfg, batch, 78)
    model, crit = build_model(synth.reference_args(cfg, device="cuda:0", droppath=0.3 if cfg_name == "tiny" else 0.1, input_dropout=0.5))
    model.load_state_dict(sd, strict=True)
    model.to("cuda:0").train()
    crit.to("cuda:0")
    model.reference_rng_order = mode == "reference_order"
    model.keep_last_draw = True
    torch.manual_seed(5)
    out = model(**inp)
    scales, masks = model._last_draw
    loss = crit(out, tgt_c)
    sum(loss[k] * crit.weight_dict[k] for k in loss).backward()
    torch.cuda.synchronize()
    B, Lv, Lt, d = batch, raw["src_vid"].shape[1], raw["src_txt"].shape[1], cfg["hidden_dim"]
    shapes = [(B, Lv, cfg["v_feat_dim"]), (B, Lv, d), (B, Lt, cfg["t_feat_dim"]), (B, Lt, d)]
    keep = 1.0 - model.droppath
    if mode == "reference_order":  # the draws are the reference's own calls in the reference's order
        torch.manual_seed(5)
        redrawn = [torch.nn.functional.dropout(torch.ones(s, device="cuda"), 0.5, True) for s in shapes]
        redrawn_s = torch.stack([torch.floor(keep + torch.rand((B, 1, 1), device="cuda")).flatten() / keep for _ in range(2 * cfg["enc_layers"])])
        assert all(torch.equal(a, b) for a, b in zip(masks, redrawn)) and torch.equal(scales, redrawn_s)
    else:  # statistics of the in-kernel generator: multipliers in {0, 1/(1-p)}, keep rate 1-p, independent streams
        for m, shp in zip(masks, shapes):
            assert tuple(m.shape) == shp and bool(((m == 0) | (m == 2.0)).all())
            assert abs(float((m != 0).float().mean()) - 0.5) < 4.0 * 0.5 / (m.numel() ** 0.5) + 1e-3
        assert float((masks[1] != masks[0][..., :d]).float().mean()) > 0.3 if cfg["v_feat_dim"] >= d else True
        assert bool(((scales == 0) | ((scales - 1.0 / keep).abs() < 1e-6)).all())
        flat = masks[0].flatten()
        assert abs(float(((flat[1:] != 0) == (flat[:-1] != 0)).float().mean()) - 0.5) < 0.02  # neighbours uncorrelated
    assert (scales == 0).any() or cfg_name != "tiny"
    masks_c, scales_c = [m.cpu() for m in masks], scales.cpu()

    def run(emulate):
        leaves = {k: v.double().requires_grad_(True) for k, v in sd.items()}
        o = O.forward(leaves, cfg, **raw, dp_scale=scales_c, drop_masks=masks_c, opq=O.round_fp16 if emulate else None)
        ls = O.criterion(o, tgt)
        O.weighted_total(ls, WD).backward()
        return o, ls, {k: v.grad for k, v in leaves.items()}

    eout, eloss, egrad = run(True)
    xout, xloss, xgrad = run(False)
    for k in ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj"):
        got = out[k].detach().double().cpu()
        tight = k.startswith("pred")  # projector outputs: K = 2818 products accumulated in fp32 (tensor core) vs fp64 (oracle)
        torch.testing.assert_close(got, eout[k].detach(), rtol=2e-4 if tight else 5e-4, atol=5e-5 if tight else 5e-4,
                                   msg=lambda m: f"{k} vs emulating oracle: {m}")
        torch.testing.assert_close(got, xout[k].detach(), rtol=1e-3, atol=1e-4 if k.startswith("pred") else 2e-3,
                                   msg=lambda m: f"{k} vs exact oracle: {m}")
    for k in xloss:
        assert abs(float(loss[k]) - float(eloss[k])) <= 1e-4 * max(1.0, abs(float(eloss[k]))), k
        assert abs(float(loss[k]) - float(xloss[k])) <= 1e-3 * max(1.0, abs(float(xloss[k]))), k
    worst = {}
    for n_, p in model.named_parameters():
        if xgrad[n_] is None or float(xgrad[n_].abs().max()) == 0.0:
            continue
        g = p.grad.double().cpu()
        worst[n_] = (_rel(g, xgrad[n_]), _cos(g, xgrad[n_]), _rel(g, egrad[n_]))
    _record(f"dropout_{cfg_name}_{mode}", {k: {"rel_exact": v[0], "cos_exact": v[1], "rel_emulating": v[2]} for k, v in worst.items()})
    # the draws come from torch's CUDA generator, whose sequence depends on the GPU's SM count: on H100 the cfg2 draws leave the
    # worst tensor (layer 0 FFN1 weight) at 2.04 % from the emulating reference and 2.14 % from the exact one
    bad = _grad_verdict(worst, 3e-2 if cfg_name == "tiny" else 2.2e-2)
    assert not bad, f"{cfg_name}: gradient mismatch with dropout + DropPath on {bad}"
    # the default (batched) draws: deterministic under a seed, different from eval
    model.reference_rng_order = False
    torch.manual_seed(9)
    a = model(**inp)["pred_spans"].detach().clone()
    torch.manual_seed(9)
    b = model(**inp)["pred_spans"].detach().clone()
    model.eval()
    with torch.no_grad():
        c = model(**inp)["pred_spans"]
    assert torch.equal(a, b) and not torch.allclose(a, c)


def test_hl_loss_list_and_missing_saliency_labels():
    """dset_type 'hl': losses = ['labels', 'saliency'], targets without timestamp / span_labels_nn (model/univtg.py:438-439,
    main/dataset.py:1118-1126).  Also the branch without saliency_pos_labels: both saliency losses are the constant 0 and the
    backward must deliver exact zeros (not uninitialised scratch) to vid_mem_proj / txt_mem_proj."""
    from oracle import univtg_oracle as O

    cfg = synth.CONFIGS["tiny"]
    sd = synth.make_state_dict(cfg, seed=5)
    raw, full, inp, _ = _train_inputs(cfg, 6, 9)
    model, crit = build_model(synth.reference_args(cfg, device="cuda:0", droppath=0.0, input_dropout=0.0, dset_type="hl"))
    assert crit.losses == ["labels", "saliency"]
    model.load_state_dict(sd, strict=True)
    model.to("cuda:0").train()
    crit.to("cuda:0")
    tgt = {"saliency_scores": full["saliency_scores"], "saliency_pos_labels": full["saliency_pos_labels"],
           "timestamp_mask": full["timestamp_mask"], "timestamp_window": 1 * (full["saliency_scores"] > 0)}
    out = model(**inp)
    loss = crit(out, {k: v.cuda() for k, v in tgt.items()})
    assert sorted(loss) == ["loss_f", "loss_s_inter", "loss_s_intra"]
    sum(loss[k] * crit.weight_dict[k] for k in loss).backward()
    leaves = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    oloss = O.criterion(O.forward(leaves, cfg, **raw), tgt, losses=("labels", "saliency"))
    O.weighted_total(oloss, WD).backward()
    for k in oloss:
        assert abs(float(loss[k]) - float(oloss[k])) <= 1e-3 * max(1.0, abs(float(oloss[k]))), k
    for n_ in ("transformer.encoder.layers.0.linear1.weight", "input_vid_proj.0.net.1.weight", "class_embed.layers.0.weight",
               "weightedpool.weight"):
        g = dict(model.named_parameters())[n_].grad.double().cpu()
        assert _rel(g, leaves[n_].grad) < 6e-2, (n_, _rel(g, leaves[n_].grad))
    g_span = dict(model.named_parameters())["span_embed.layers.0.weight"].grad
    assert g_span is None or float(g_span.abs().max()) == 0.0  # no 'spans' loss -> no gradient into span_embed
    # no saliency_pos_labels: reference returns 0. for both saliency losses (model/univtg.py:236-237)
    for p in model.parameters():
        p.grad = None
    tgt2 = {k: v.cuda() for k, v in tgt.items() if k != "saliency_pos_labels"}
    out = model(**inp)
    torch.empty(64 << 20, dtype=torch.uint8, device="cuda").fill_(0xFF)  # poison the allocator's free blocks (NaN patterns)
    loss = crit(out, tgt2)
    assert float(loss["loss_s_inter"]) == 0.0 and float(loss["loss_s_intra"]) == 0.0
    sum(loss[k] * crit.weight_dict[k] for k in loss).backward()
    for n_, p in model.named_parameters():
        if p.grad is not None:
            assert bool(torch.isfinite(p.grad).all()), n_
    assert float(dict(model.named_parameters())["weightedpool.weight"].grad.abs().max()) == 0.0


def test_optimizer_step_decreases_loss():
    """A few AdamW steps of the reference training loop body (train_vlp_ddp.py:56-68) on one synthetic batch."""
    cfg = synth.CONFIGS["tiny"]
    model, crit = _models(cfg, synth.make_state_dict(cfg, seed=3))
    model.train()
    inp = {k: v.cuda() for k, v in synth.make_inputs(cfg, seed=4, ragged=True, batch=8).items()}
    tgt = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in synth.make_targets(synth.make_inputs(cfg, seed=4, ragged=True, batch=8), seed=5).items()}
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-4, weight_decay=1e-4)
    vals = []
    for _ in range(12):
        out = model(**inp)
        ld = crit(out, tgt)
        total = sum(ld[k] * crit.weight_dict[k] for k in ld)
        opt.zero_grad()
        total.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 0.1)
        opt.step()
        vals.append(float(total))
    assert vals[-1] < vals[0], vals


@pytest.mark.parametrize("gscale", [1e-4, 3.0])  # below / above the clip threshold of 0.1
def test_flat_adamw_matches_torch_clip_plus_adamw(gscale):
    """univtg_adamw_step == clip_grad_norm_ + torch.optim.AdamW (train_vlp_ddp.py:66-68) on the same gradients."""
    from univtg_b200.optim import FlatAdamW

    cfg = synth.CONFIGS["tiny"]
    model, _ = _models(cfg, synth.make_state_dict(cfg, seed=3))
    ref_params = [p.detach().clone().requires_grad_(True) for p in model._abi_params()]
    opt_ref = torch.optim.AdamW(ref_params, lr=1e-3, weight_decay=1e-2)
    opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-2, max_grad_norm=0.1)
    gen = torch.Generator(device="cuda").manual_seed(11)
    for _ in range(4):
        flat, views = model._grad_buffer()
        flat.zero_()
        for v, rp in zip(views, ref_params):
            g = torch.randn(v.shape, device="cuda", generator=gen) * gscale
            v.copy_(g)
            rp.grad = g.clone()
        n_ref = torch.nn.utils.clip_grad_norm_(ref_params, 0.1)
        opt_ref.step()
        n = opt.step()
        assert abs(float(n) - float(n_ref)) <= 1e-5 * float(n_ref)
        for p, rp in zip(model._abi_params(), ref_params):
            torch.testing.assert_close(p.detach(), rp.detach(), rtol=2e-5, atol=2e-7)


def _fill_grads(model, ref_params, gen, gscale=1e-3):
    """Same random gradients into the model's flat buffer and into `ref_params` (clones of named_parameters(), same order)."""
    flat, views = model._grad_buffer()
    flat.zero_()
    pos = {id(p): i for i, (_, p) in enumerate(model.named_parameters())}
    for v, p in zip(views, model._abi_params()):
        g = torch.randn(v.shape, device="cuda", generator=gen) * gscale
        v.copy_(g)
        ref_params[pos[id(p)]].grad = g.clone()


def test_flat_adamw_is_a_torch_optimizer_checkpoints_both_ways_and_follows_schedulers():
    """The reference drives its optimizer through lr schedulers (main/config.py:352-360) and writes / resumes
    optimizer.state_dict() (main/train_mr.py:151, main/config.py:371): FlatAdamW is a torch.optim.Optimizer whose checkpoints are
    interchangeable with those of torch.optim.AdamW built the reference's way (all named_parameters(), one group), and whose lr
    is the parameter group's."""
    from univtg_b200.optim import FlatAdamW

    cfg = synth.CONFIGS["tiny"]
    sd0 = synth.make_state_dict(cfg, seed=3)
    model, _ = _models(cfg, sd0)

    def clones(m):
        return [p.detach().clone().requires_grad_(True) for _, p in m.named_parameters()]

    def check(m, ref):
        for (n, p), rp in zip(m.named_parameters(), ref):
            torch.testing.assert_close(p.detach(), rp.detach(), rtol=2e-5, atol=2e-7, msg=lambda s, n=n: f"{n}: {s}")

    ref_params = clones(model)
    opt_ref = torch.optim.AdamW(ref_params, lr=1e-3, weight_decay=1e-2)
    opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-2, max_grad_norm=0.0, dynamic_loss_scale=False)
    assert isinstance(opt, torch.optim.Optimizer) and len(opt.param_groups) == 1
    assert [id(p) for p in opt.param_groups[0]["params"]] == [id(p) for _, p in model.named_parameters()]
    assert len(ref_params) > len(model._abi_params())  # txt_position_embed.*: in the group, never updated (no gradient)
    gen = torch.Generator(device="cuda").manual_seed(5)
    for _ in range(3):
        _fill_grads(model, ref_params, gen)
        opt_ref.step()
        opt.step()
    check(model, ref_params)
    # (1) this optimizer's checkpoint -> the reference's optimizer
    ck = opt.state_dict()
    assert set(ck["state"]) == set(opt_ref.state_dict()["state"]) and float(ck["state"][min(ck["state"])]["step"]) == 3.0
    other = clones(model)
    opt_t = torch.optim.AdamW(other, lr=5e-2, weight_decay=0.0)
    opt_t.load_state_dict(ck)
    assert opt_t.param_groups[0]["lr"] == 1e-3 and opt_t.param_groups[0]["weight_decay"] == 1e-2
    # (2) the reference's checkpoint -> a fresh FlatAdamW on a fresh model holding the same weights
    model2, _ = _models(cfg, sd0)
    with torch.no_grad():
        for p2, p in zip(model2.parameters(), model.parameters()):
            p2.copy_(p)
    opt2 = FlatAdamW(model2, lr=7e-2, weight_decay=0.0, max_grad_norm=0.0, dynamic_loss_scale=False)
    opt2.load_state_dict(opt_ref.state_dict())
    assert opt2.step_count == 3 and opt2.lr == 1e-3 and opt2.weight_decay == 1e-2
    # one more step everywhere on identical gradients: four optimizers, one trajectory
    _fill_grads(model, ref_params, torch.Generator(device="cuda").manual_seed(9))
    for o, rp in zip(other, ref_params):
        o.grad = None if rp.grad is None else rp.grad.clone()
    _fill_grads(model2, clones(model2), torch.Generator(device="cuda").manual_seed(9))
    opt_ref.step()
    opt.step()
    opt_t.step()
    opt2.step()
    check(model, ref_params)
    check(model2, ref_params)
    for o, rp in zip(other, ref_params):
        torch.testing.assert_close(o.detach(), rp.detach(), rtol=2e-5, atol=2e-7)
    # (3) schedulers write the group's lr and the kernel reads it: after the decay to 0 a step moves nothing
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=1, gamma=0.0)
    assert opt.param_groups[0]["initial_lr"] == 1e-3
    opt.param_groups[0]["weight_decay"] = 0.0
    opt.step()  # (schedulers want an optimizer step before their own)
    sched.step()
    assert opt.lr == 0.0
    before = [p.detach().clone() for p in model.parameters()]
    _fill_grads(model, ref_params, gen)
    opt.step()
    for p, b in zip(model.parameters(), before):
        assert torch.equal(p.detach(), b)
    with pytest.raises(RuntimeError):
        opt.add_param_group({"params": [torch.zeros(1, device="cuda", requires_grad=True)]})


def test_zero_grad_after_step_is_the_same_training_run():
    """FlatAdamW(zero_grad_after_step=True) moves the zero-fill of the flat gradient buffer from the front of the backward to a
    side stream behind the update: same trajectory as the default, gradients read zero after step(), and a loop that never calls
    zero_grad() is then the reference loop (train_vlp_ddp.py:63-68) too."""
    from univtg_b200.optim import FlatAdamW

    cfg = synth.CONFIGS["tiny"]
    raw, tgt, inp, ctgt = _train_inputs(cfg, 6, 31)
    runs, grads, late = [], [], []
    for pre, call_zero in ((False, True), (True, True), (True, False)):
        model, crit = _models(cfg, synth.make_state_dict(cfg, seed=3))
        model.train()
        opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-2, max_grad_norm=0.1, zero_grad_after_step=pre)
        start = [p.detach().clone() for p in model._abi_params()]
        for it in range(4):
            torch.manual_seed(7)
            out = model(**inp)
            total = crit.weighted_total(crit(out, ctgt))
            if call_zero:
                opt.zero_grad()
            total.backward()
            if it == 1:  # the first backward that relies on the early fill: a stale buffer would hold step 0's gradient on top
                grads.append(model._grad_buffer()[0].clone())
            if it == 3:
                late.append(model._grad_buffer()[0].clone())
            opt.step()
        torch.cuda.synchronize()
        if pre:
            assert float(model._grad_buffer()[0].abs().max()) == 0.0
        runs.append([p.detach().clone() for p in model._abi_params()])
    for g in grads[1:]:
        assert float((g - grads[0]).norm() / grads[0].norm()) < 5e-3  # (fp32 atomics + last-bit parameter differences after one update; 3.9e-3 on H100)
    for g in late[1:]:  # three updates later the parameters differ in their last bits (Adam amplifies rounding noise), the gradients barely
        assert float((g - late[0]).norm() / late[0].norm()) < 2e-2
    # trajectories: Adam normalises, so single elements whose gradient is ~0 move by a noticeable fraction of lr on rounding noise
    # alone - compare the four-step update of each tensor as a whole
    for other in runs[1:]:
        for a, b, p0 in zip(runs[0], other, start):
            moved = float((a - p0).norm())
            assert float((a - b).norm()) <= 0.2 * moved + 1e-7, (float((a - b).norm()), moved)


def test_training_loop_with_flat_adamw_decreases_loss_and_repacks():
    from univtg_b200.optim import FlatAdamW

    cfg = synth.CONFIGS["tiny"]
    model, crit = _models(cfg, synth.make_state_dict(cfg, seed=3))
    model.train()
    raw = synth.make_inputs(cfg, seed=4, ragged=True, batch=8)
    inp = {k: v.cuda() for k, v in raw.items()}
    tgt = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in synth.make_targets(raw, seed=5).items()}
    opt = FlatAdamW(model, lr=1e-4, weight_decay=1e-4, max_grad_norm=0.1)
    vals = []
    for _ in range(12):
        out = model(**inp)
        ld = crit(out, tgt)
        total = sum(ld[k] * crit.weight_dict[k] for k in ld)
        opt.zero_grad()
        total.backward()
        opt.step()
        vals.append(float(total))
    assert vals[-1] < vals[0], vals
    # the state_dict still exposes the (updated) parameters under the reference keys
    sd = model.state_dict()
    assert all(torch.isfinite(v).all() for v in sd.values())


def test_stage_events_fire_only_after_their_gradients_are_final():
    """Overlap path of univtg_b200.ddp: at stage event k the stage's slice of the flat gradient buffer is snapshotted on a
    side stream while the rest of the backward is still running; every snapshot must equal the final buffer bit for bit."""
    from univtg_b200 import ddp

    cfg = synth.CONFIGS["cfg2"]
    model, crit = _models(cfg, synth.make_state_dict(cfg, seed=3))
    model.train()
    raw = synth.make_inputs(cfg, seed=4, ragged=True, batch=16)
    inp = {k: v.cuda() for k, v in raw.items()}
    tgt = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in synth.make_targets(raw, seed=5).items()}

    class Snapshot(ddp.OverlappedGradExchange):
        def __init__(self, model):  # no process group: pretend world 2 and record instead of reducing
            self.group, self.world, self.backend = None, 2, "snapshot"
            self.stages = ddp.grad_stage_slices(model)
            self.events, self.comm_stream, self.snaps = None, None, []

        def _reduce(self, t):
            self.snaps.append((t, t.clone()))

    model.direct_grad = True
    model._grad_sync = Snapshot(model)
    for _ in range(2):
        model._grad_sync.snaps = []
        out = model(**inp)
        ld = crit(out, tgt)
        sum(ld[k] * crit.weight_dict[k] for k in ld).backward()
    torch.cuda.synchronize()
    snaps = model._grad_sync.snaps
    assert len(snaps) == cfg["enc_layers"] + 5  # heads, one per encoder layer, two slices for each of the two projector stages
    flat, _ = model._grad_buffer()
    assert sum(s.numel() for s, _ in snaps) == flat.numel()
    for i, (live, snap) in enumerate(snaps):
        assert torch.equal(live, snap), f"stage slice {i} changed after its event fired"
        assert float(snap.abs().sum()) > 0.0


def test_weighted_total_equals_reference_sum_expression():
    """SetCriterion.weighted_total == sum(loss_dict[k] * weight_dict[k]) (train_mr.py:56-58), values and gradients."""
    cfg = synth.CONFIGS["tiny"]
    model, crit = _models(cfg, synth.make_state_dict(cfg, seed=3))
    model.train()
    raw = synth.make_inputs(cfg, seed=4, ragged=True, batch=8)
    inp = {k: v.cuda() for k, v in raw.items()}
    tgt = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in synth.make_targets(raw, seed=5).items()}
    grads = []
    for fused in (False, True):
        torch.manual_seed(0)
        for p in model.parameters():
            p.grad = None
        ld = crit(model(**inp), tgt)
        total = crit.weighted_total(ld) if fused else sum(ld[k] * crit.weight_dict[k] for k in ld.keys() if k in crit.weight_dict)
        total.backward()
        grads.append((float(total), [None if p.grad is None else p.grad.detach().clone() for p in model.parameters()]))
    assert abs(grads[0][0] - grads[1][0]) <= 1e-5 * max(1.0, abs(grads[0][0]))
    assert sum(g is not None for g in grads[0][1]) >= len(model._abi_params())
    for a, b in zip(grads[0][1], grads[1][1]):
        assert (a is None) == (b is None)  # parameters outside the univtg path (never used by the reference either) get no gradient
        if a is not None:
            torch.testing.assert_close(a, b, rtol=2e-3, atol=1e-6)  # fp32 atomics in the backward are order-dependent


def test_fp16_overflow_skips_the_update_and_backs_the_loss_scale_off():
    """fp16 safety: with an absurd loss scale the 16-bit gradient operands overflow; the fused AdamW must leave weights and
    moments bit-identical (skipped step), the next step() halves model.grad_scale, and training recovers."""
    from univtg_b200.optim import FlatAdamW

    cfg = synth.CONFIGS["tiny"]
    model, crit = _models(cfg, synth.make_state_dict(cfg, seed=3))
    model.train()
    raw, tgt, inp, ctgt = _train_inputs(cfg, 6, 31)
    opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-2, max_grad_norm=0.1)

    def step():
        out = model(**inp)
        total = crit.weighted_total(crit(out, ctgt))
        opt.zero_grad()
        total.backward()
        opt.step()
        return float(total)

    step()  # a normal step: moments become non-zero
    torch.cuda.synchronize()
    before = [p.detach().clone() for p in model._abi_params()]
    m0, v0, n0 = opt._m.clone(), opt._v.clone(), opt.step_count
    model.grad_scale = 2.0 ** 60
    step()
    torch.cuda.synchronize()
    assert float(opt._scratch[2]) == 1.0
    for p, b in zip(model._abi_params(), before):
        assert torch.equal(p.detach(), b)
    assert torch.equal(opt._m, m0) and torch.equal(opt._v, v0)
    step()  # consumes the flag: scale halved, the skipped step does not count
    assert model.grad_scale == 2.0 ** 59 and opt.skipped_steps >= 1
    model.grad_scale = 1024.0
    l0 = step()
    for _ in range(8):
        l1 = step()
    torch.cuda.synchronize()
    assert opt.step_count <= n0 + 10  # skipped updates are not counted
    assert all(bool(torch.isfinite(p).all()) for p in model._abi_params()) and l1 < l0


@pytest.mark.parametrize("cfg_name", ["tiny", "cfg1"])
def test_adamw_keeps_the_packed_operands_current(cfg_name):
    """univtg_adamw_step writes the 16-bit GEMM operand copies itself (+ univtg_pack_vectors for the fp32 vectors): after a few
    steps the packed buffer must be byte-identical to a fresh univtg_pack_weights of the updated parameters."""
    from univtg_b200.optim import FlatAdamW

    cfg = synth.CONFIGS[cfg_name]  # tiny: v_feat_dim 194 (rows straddle float4s); cfg1: 514
    model, crit = _models(cfg, synth.make_state_dict(cfg, seed=3))
    model.train()
    raw, tgt, inp, ctgt = _train_inputs(cfg, 4, 41)
    opt = FlatAdamW(model, lr=1e-3, weight_decay=1e-2, max_grad_norm=0.1)
    for _ in range(3):
        out = model(**inp)
        total = crit.weighted_total(crit(out, ctgt))
        opt.zero_grad()
        total.backward()
        opt.step()
    fmt = model._fmt(True)
    kept = model._packed[fmt].clone()
    key = dict(model._packed_key)
    model._packed_key = {}
    model._ensure_packed(training=True)  # full re-pack from the fp32 parameters
    torch.cuda.synchronize()
    assert torch.equal(kept, model._packed[fmt])
    assert fmt in key  # and the step did not invalidate the key: the next forward packs nothing
