"""Ragged-shape robustness of the plugin (reference collate pads every batch to ITS maximum, main/dataset.py:1037-1052,
utils/tensor_utils.py:36-53, so (B, L_v, L_t) changes from batch to batch): LRU plan cache, ONE shared inference workspace,
pooled training workspaces, torch-like gradient accumulation."""
import pytest
import torch

from univtg_b200 import build_model, synth

pytestmark = pytest.mark.gpu
WD = {"loss_b": 10.0, "loss_g": 1.0, "loss_f": 10.0, "loss_s_intra": 0.1, "loss_s_inter": 0.1}
CFG = dict(synth.CONFIGS["tiny"], nheads=2)  # d = 256, dh = 128: wgmma attention, oracle finishes in well under a second


def _model(**over):
    model, crit = build_model(synth.reference_args(CFG, device="cuda:0", droppath=0.0, input_dropout=0.0, **over))
    model.load_state_dict(synth.make_state_dict(CFG, seed=3), strict=True)
    return model.to("cuda:0"), crit.to("cuda:0")


def _batch(B, Lv, Lt, seed):
    raw = synth.make_inputs(CFG, seed=seed, ragged=True, batch=B, l_vid=Lv, l_txt=Lt)
    tgt = synth.make_targets(raw, seed=seed + 1)
    return raw, tgt, {k: v.cuda() for k, v in raw.items()}, {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in tgt.items()}


def _step(model, crit, inp, tgt):
    out = model(**inp)
    ld = crit(out, tgt)
    total = sum(ld[k] * crit.weight_dict[k] for k in ld)
    total.backward()
    return out, ld


def test_fifty_ragged_batches_reuse_the_pooled_workspaces_and_stay_correct():
    from oracle import univtg_oracle as O

    model, crit = _model()
    model.train()
    model.PLAN_CACHE = 8  # force evictions
    g = torch.Generator().manual_seed(0)
    shapes = [(6, 150, 32)] + [(int(torch.randint(2, 7, (1,), generator=g)), int(torch.randint(8, 151, (1,), generator=g)),
                                int(torch.randint(3, 33, (1,), generator=g))) for _ in range(50)]
    checked = 0
    reserved0 = None
    for i, (B, Lv, Lt) in enumerate(shapes):
        raw, tgt, inp, ctgt = _batch(B, Lv, Lt, 100 + i)
        for p in model.parameters():
            p.grad = None
        out, ld = _step(model, crit, inp, ctgt)
        if i % 3 == 0:  # interleave inference forwards of yet another shape: they share ONE workspace with every other plan
            model.eval()
            with torch.no_grad():
                ev = model(**_batch(B, max(8, Lv - 3), Lt, 500 + i)[2])
            assert bool(torch.isfinite(ev["pred_spans"]).all())
            model.train()
        if i == 1:
            torch.cuda.synchronize()
            reserved0 = torch.cuda.memory_reserved()
        if i in (7, 23, 50):
            leaves = {k: v.double().requires_grad_(True) for k, v in synth.make_state_dict(CFG, seed=3).items()}
            oout = O.forward(leaves, CFG, **raw, opq=O.round_fp16)
            ol = O.criterion(oout, tgt)
            O.weighted_total(ol, WD).backward()
            for k in ("pred_logits", "pred_spans"):
                torch.testing.assert_close(out[k].detach().double().cpu(), oout[k].detach(), rtol=2e-4, atol=5e-5)
            for k in ol:
                assert abs(float(ld[k]) - float(ol[k])) <= 1e-4 * max(1.0, abs(float(ol[k]))), (i, k)
            named = dict(model.named_parameters())
            for n_ in ("transformer.encoder.layers.0.linear2.weight", "input_txt_proj.1.net.1.weight", "class_embed.layers.1.weight"):
                a, b = named[n_].grad.double().cpu(), leaves[n_].grad
                assert float((a - b).norm() / b.norm()) < 6e-2, (i, n_)
            checked += 1
    torch.cuda.synchronize()
    assert checked == 3
    assert len(model._plans) <= 8
    assert len(model.__dict__["_train_pool"]) == 1  # one pooled training workspace served all 51 shapes
    # device memory: nothing beyond allocator noise was reserved after the first (largest) shape
    assert torch.cuda.memory_reserved() - reserved0 <= 96 << 20, (torch.cuda.memory_reserved(), reserved0)


def test_poisoned_workspaces_give_identical_results():
    """Nothing but the rows univtg_prepare_workspace zeroes may be read before it is written: fill both workspaces with 0xFF
    (NaN patterns), re-establish the zero rows, and the outputs / gradients must be bit-identical."""
    from univtg_b200 import _lib
    import ctypes

    model, crit = _model()
    raw, tgt, inp, ctgt = _batch(5, 37, 11, 7)
    model.eval()
    with torch.no_grad():
        a = model(**inp)
    model._ws_infer.fill_(0xFF)
    model.__dict__["_ws_owner"] = None  # forces univtg_prepare_workspace on the next forward
    with torch.no_grad():
        b = model(**inp)
    for k in ("pred_logits", "pred_spans", "saliency_scores", "vid_mem_proj", "txt_mem_proj"):
        assert torch.equal(a[k], b[k]), k
    model.train()
    _step(model, crit, inp, ctgt)
    g1 = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    for p in model.parameters():
        p.grad = None
    pool = model.__dict__["_train_pool"]
    assert len(pool) == 1
    pool[0].fill_(0xFF)
    model.__dict__["_train_ws_shape"].clear()
    _step(model, crit, inp, ctgt)
    lib = _lib.load_library()
    assert lib is not None and ctypes is not None
    for n, p in model.named_parameters():
        if p.grad is not None:
            assert bool(torch.isfinite(p.grad).all()), n
            # split-K / column-sum reductions use fp32 atomics: order-dependent in the last bits only
            torch.testing.assert_close(p.grad, g1[n], rtol=2e-3, atol=1e-6)


def test_two_forwards_before_backward_and_gradient_accumulation():
    """Micro-batching the way torch users write it: two training forwards, ONE summed loss, one backward; and two backwards
    without zero_grad() accumulate - in autograd mode and in direct_grad mode (FlatAdamW / flat all-reduce)."""
    from univtg_b200.optim import FlatAdamW

    model, crit = _model()
    model.train()
    _, _, inp1, tgt1 = _batch(4, 30, 9, 11)
    _, _, inp2, tgt2 = _batch(4, 30, 9, 13)  # same shape: round 1 would have overwritten the first forward's activations

    def grads():
        out = {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}
        for p in model.parameters():
            p.grad = None
        return out

    _step(model, crit, inp1, tgt1)
    ga = grads()
    _step(model, crit, inp2, tgt2)
    gb = grads()
    o1, o2 = model(**inp1), model(**inp2)
    l1, l2 = crit(o1, tgt1), crit(o2, tgt2)
    (sum(l1[k] * crit.weight_dict[k] for k in l1) + sum(l2[k] * crit.weight_dict[k] for k in l2)).backward()
    gsum = grads()
    for n in ga:
        torch.testing.assert_close(gsum[n], ga[n] + gb[n], rtol=3e-3, atol=1e-6, msg=lambda m: f"{n}: {m}")
    # direct_grad mode: .grad are views of the flat buffer
    opt = FlatAdamW(model, lr=1e-4)
    opt.zero_grad()
    _step(model, crit, inp1, tgt1)
    _step(model, crit, inp2, tgt2)  # no zero_grad in between -> accumulates
    for n, p in model.named_parameters():
        if n in ga:
            torch.testing.assert_close(p.grad, ga[n] + gb[n], rtol=3e-3, atol=1e-6, msg=lambda m: f"direct {n}: {m}")
    opt.zero_grad()
    _step(model, crit, inp2, tgt2)
    for n, p in model.named_parameters():
        if n in gb:
            torch.testing.assert_close(p.grad, gb[n], rtol=3e-3, atol=1e-6)


def test_pinned_plan_survives_eviction_and_plan_ids_are_not_reused_for_arming():
    """A plan held by a live autograd context is never destroyed by the LRU; the gradient exchange arms every NEW plan entry
    even when CPython recycles the id() of an evicted one (round-1 advisor finding)."""
    from univtg_b200 import ddp

    model, crit = _model()
    model.train()
    model.PLAN_CACHE = 2
    _, _, inp0, tgt0 = _batch(3, 20, 8, 21)
    out0 = model(**inp0)  # holds plan (3, 20, 8)
    held = model._plans[(3, 20, 8, 1)]
    assert held.pins == 1

    class Recorder(ddp.OverlappedGradExchange):
        def __init__(self, model):
            self.group, self.world, self.backend = None, 2, "record"
            self.stages = ddp.grad_stage_slices(model)
            self.events, self.comm_stream, self.reduced = None, None, 0

        def _reduce(self, t):
            self.reduced += 1

    model.direct_grad = True
    model._grad_sync = Recorder(model)
    armed = []
    for i in range(6):  # six more shapes through a 2-entry cache
        _, _, inp, tgt = _batch(2, 10 + i, 5, 30 + i)
        _step(model, crit, inp, tgt)
        plan = model._plans[(2, 10 + i, 5, 1)]
        assert plan.grad_events_owner is model._grad_sync
        armed.append(plan)
    assert held.handle is not None and (3, 20, 8, 1) in model._plans
    ld = crit(out0, tgt0)
    sum(ld[k] * crit.weight_dict[k] for k in ld).backward()
    torch.cuda.synchronize()
    assert held.pins == 0
    assert all(torch.isfinite(p.grad).all() for p in model.parameters() if p.grad is not None)
