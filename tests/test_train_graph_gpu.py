"""GPU checks of the graphed training step (univtg_b200.graphs.GraphedTrainStep) against the eager step.

What can be bit-identical is checked bit for bit:
  * the seed: replay k draws the masks of univtg_rng_seed_at(seed_base, k), so its losses equal, bit for bit, an eager training
    forward of the same parameters whose plan reads that seed (forward and criterion are deterministic);
  * the update: the parameters, moments and 16-bit operands a replay leaves equal univtg_adamw_step + univtg_pack_vectors applied
    eagerly to a snapshot taken before the replay, with the gradients the replay computed, at the step the host counts.
The gradients themselves come out of the backward's fp32 atomics, whose order changes from run to run, so two eager runs are
not bit-identical either: whole trajectories against a separate eager model are compared like
tests/test_train_gpu.py::test_zero_grad_after_step_is_the_same_training_run does."""
import ctypes

import pytest
import torch

from univtg_b200 import _lib, build_model, synth
from univtg_b200.graphs import GraphedTrainStep, rng_seed_at
from univtg_b200.optim import FlatAdamW

pytestmark = pytest.mark.gpu

DROPS = dict(input_dropout=0.5, droppath=0.1, dropout=0.1)


def _models(cfg_name, use_txt_pos=False, n=2, qfvs=False, **over):
    cfg = synth.CONFIGS[cfg_name]
    sd = synth.make_state_dict(cfg, seed=3)
    out = []
    for _ in range(n):
        if qfvs:
            from univtg_b200.qfvs import build_model as qfvs_build

            model, crit = qfvs_build(synth.reference_args(cfg, device="cuda:0", dset_type="vs", use_txt_pos=use_txt_pos, **DROPS))
        else:
            model, crit = build_model(synth.reference_args(cfg, device="cuda:0", use_txt_pos=use_txt_pos, **DROPS))
        model.load_state_dict(sd, strict=True)
        model = model.to("cuda:0").train()
        crit = crit.to("cuda:0")
        opt = FlatAdamW(model, **dict(dict(lr=1e-3, weight_decay=1e-2, max_grad_norm=0.1), **over))
        out.append((model, crit, opt))
    return out


def _batch(cfg_name, seed, batch=4, l_vid=None, l_txt=None):
    cfg = synth.CONFIGS[cfg_name]
    raw = synth.make_inputs(cfg, seed=seed, ragged=True, batch=batch, l_vid=l_vid, l_txt=l_txt)
    tgt = synth.make_targets(raw, seed=seed + 1)
    return {k: v.cuda() for k, v in raw.items()}, {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in tgt.items()}


def _seeded(model, inp, seed):
    """Context: the plan of this input shape reads `seed` from device memory (None: the host seed of the eager step)."""
    lib = _lib.load_library()

    class _Ctx:
        def __enter__(self):
            B, Lv, _ = inp["src_vid"].shape
            model._ensure_packed(training=True)
            self.plan = model._get_plan(B, Lv, inp["src_txt"].shape[1], True)
            self.t = None
            if seed is not None:
                self.t = torch.tensor([seed - (1 << 64) if seed >= (1 << 63) else seed], dtype=torch.int64, device="cuda:0")
                _lib.check(lib.univtg_plan_set_seed_source(self.plan.handle, ctypes.c_void_p(self.t.data_ptr())), "seed source")
            return self

        def __exit__(self, *exc):
            torch.cuda.synchronize()
            lib.univtg_plan_set_seed_source(self.plan.handle, None)

    return _Ctx()


def _eager_step(model, crit, opt, inp, tgt, seed, mask=None):
    with _seeded(model, inp, seed):
        out = model(**inp)
        ld = crit(out, tgt) if mask is None else crit(out, tgt, mask)
        total = crit.weighted_total(ld)
        opt.zero_grad()
        total.backward()
        opt.step()
    return total.detach().clone(), ld.vector.detach().clone()


def _probe_losses(model, crit, inp, tgt, seed, mask=None):
    """Training forward + criterion (no backward, nothing updated) drawing from `seed`."""
    with _seeded(model, inp, seed):
        out = model(**inp)
        ld = crit(out, tgt) if mask is None else crit(out, tgt, mask)
        vec = ld.vector.detach().clone()
    del out, ld
    return vec


def _snapshot(model, opt):
    fmt = model._fmt(True)
    return dict(p=opt._flat_p.clone(), m=opt._m.clone(), v=opt._v.clone(), packed=model._packed[fmt].clone())


def _eager_update(model, opt, snap, step):
    """univtg_adamw_step + univtg_pack_vectors on the snapshot, with the gradients now in the flat buffer."""
    lib = _lib.load_library()
    fmt = model._fmt(True)
    cfg = model._cfgs[fmt]
    flat_g, _ = model._grad_buffer()
    g = flat_g.clone()
    scratch = torch.zeros(2048, dtype=torch.float32, device="cuda:0")
    _lib.check(lib.univtg_adamw_step(_lib.ptr(snap["p"]), _lib.ptr(g), _lib.ptr(snap["m"]), _lib.ptr(snap["v"]), g.numel(), opt.lr,
                                     opt.betas[0], opt.betas[1], opt.eps, opt.weight_decay, int(step), opt.max_grad_norm, 0,
                                     _lib.ptr(scratch), ctypes.byref(cfg), _lib.ptr(snap["packed"]), _lib.stream_ptr()), "adamw")
    base = opt._flat_p.data_ptr()
    ptrs = [snap["p"].data_ptr() + (p.data_ptr() - base) for p in model._packed_params()]
    arr = (ctypes.c_void_p * len(ptrs))(*ptrs)
    _lib.check(lib.univtg_pack_vectors(ctypes.byref(cfg), arr, len(arr), _lib.ptr(snap["packed"]), _lib.stream_ptr()), "pack_vectors")
    torch.cuda.synchronize()
    return snap, float(scratch[2])


def _check_update_bitwise(model, opt, snap, step_count):
    ref, skipped = _eager_update(model, opt, snap, step_count)
    fmt = model._fmt(True)
    assert torch.equal(opt._flat_p, ref["p"])
    assert torch.equal(opt._m, ref["m"]) and torch.equal(opt._v, ref["v"])
    assert torch.equal(model._packed[fmt], ref["packed"])
    return skipped


def _graphed_call(gs, inp, tgt, mask=None, check=True):
    """One graphed step, checked bit for bit: losses against an eager forward with the replay's seed, update against the eager
    update of the replay's gradients."""
    model, crit, opt = gs.model, gs.criterion, gs.optimizer
    k = gs.replays + 1
    probe = _probe_losses(model, crit, inp, tgt, rng_seed_at(gs.seed_base, k), mask) if check else None
    snap = _snapshot(model, opt) if check else None  # (after the probe: its forward packs the operands on first use)
    total, losses = gs(inp, tgt, mask) if mask is not None else gs(inp, tgt)
    torch.cuda.synchronize()
    assert gs.replays == k
    if check:
        assert torch.equal(losses.vector, probe), (losses.vector, probe)
        assert torch.equal(total, crit.weighted_total(losses))
        skipped = float(opt._scratch[2]) != 0.0
        # the step this update ran at: the device counter before the replay + 1 (= the host count unless a skip is pending)
        step_now = int(gs._step.item())
        _check_update_bitwise(model, opt, snap, step_now if not skipped else step_now + 1)
    return total.detach().clone(), losses.vector.detach().clone()


def _close_trajectory(pa, pb, p0):
    moved = float((pa - p0).norm())
    assert float((pa - pb).norm()) <= 0.2 * moved + 1e-7, (float((pa - pb).norm()), moved)


@pytest.mark.parametrize("cfg_name", ["tiny", "cfg1"])
@pytest.mark.parametrize("use_txt_pos", [False, True])
def test_six_replays_equal_six_eager_steps_with_the_replay_seeds(cfg_name, use_txt_pos):
    (mg, cg, og), (me, ce, oe) = _models(cfg_name, use_txt_pos)
    gs = GraphedTrainStep(mg, cg, og)
    p0 = og._flat_p.clone()
    for k in range(1, 7):
        inp, tgt = _batch(cfg_name, 100 + k)
        tg, lg = _graphed_call(gs, inp, tgt)
        te, le = _eager_step(me, ce, oe, inp, tgt, rng_seed_at(gs.seed_base, k))
        torch.cuda.synchronize()
        assert og.step_count == oe.step_count == k and int(gs._step.item()) == k
        torch.testing.assert_close(lg, le, rtol=2e-3, atol=1e-5)  # (parameters differ in their last bits after step 1)
    _close_trajectory(og._flat_p, oe._flat_p, p0)
    assert gs.num_graphs == 1 and len(gs.captures) == 1


@pytest.mark.parametrize("cfg_name", ["tiny", "cfg1"])
def test_device_seed_equals_the_same_host_seed(cfg_name):
    """univtg_plan_set_seed_source(s) draws exactly the masks of rng.seed = s: forward outputs bit for bit, gradients to the
    backward's atomics noise - so the oracle-pinned dropout tests of the host seed carry over."""
    ((model, crit, opt),) = _models(cfg_name, n=1)
    inp, tgt = _batch(cfg_name, 7)
    res = []
    for use_dev in (False, True):
        state = torch.get_rng_state()
        seed = int(torch.empty((), dtype=torch.int64).random_().item()) & 0xFFFFFFFFFFFFFFFF  # what the eager forward draws
        torch.set_rng_state(state)
        with _seeded(model, inp, seed if use_dev else None):
            out = model(**inp)
            total = crit.weighted_total(crit(out, tgt))
            opt.zero_grad()
            total.backward()
        torch.set_rng_state(state)
        res.append(({k: out[k].detach().clone() for k in ("pred_logits", "pred_spans", "vid_mem_proj", "txt_mem_proj",
                                                           "saliency_scores")}, model._grad_buffer()[0].clone()))
        opt.zero_grad()
    (o0, g0), (o1, g1) = res
    for k in o0:
        assert torch.equal(o0[k], o1[k]), k
    assert float((g0 - g1).norm() / g0.norm()) < 1e-4
    # a different seed gives different masks
    with _seeded(model, inp, 12345):
        o2 = model(**inp)["pred_logits"].detach().clone()
    assert not torch.equal(o2, o0["pred_logits"])


def test_two_replays_of_one_batch_draw_different_masks():
    ((model, crit, opt),) = _models("tiny", n=1, lr=0.0)
    gs = GraphedTrainStep(model, crit, opt)
    inp, tgt = _batch("tiny", 11)
    p0 = opt._flat_p.clone()
    _, l1 = _graphed_call(gs, inp, tgt)
    _, l2 = _graphed_call(gs, inp, tgt)
    assert not torch.equal(l1, l2)
    assert torch.equal(opt._flat_p, p0)  # lr = 0: decay 1 - 0 * wd = 1, no step


@pytest.mark.parametrize("sched", ["lambda", "step"])
def test_lr_schedule_between_replays_matches_eager(sched):
    runs = _models("tiny")
    scheds = []
    for _, _, opt in runs:
        if sched == "lambda":
            scheds.append(torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 1.0 / (1 + e)))
        else:
            scheds.append(torch.optim.lr_scheduler.StepLR(opt, step_size=2, gamma=0.3))
    (mg, cg, og), (me, ce, oe) = runs
    gs = GraphedTrainStep(mg, cg, og)
    p0 = og._flat_p.clone()
    lrs = []
    for k in range(1, 6):
        inp, tgt = _batch("tiny", 200 + k)
        _graphed_call(gs, inp, tgt)
        _eager_step(me, ce, oe, inp, tgt, rng_seed_at(gs.seed_base, k))
        lrs.append(og.lr)
        assert float(gs._lr.item()) == float(torch.tensor(og.lr, dtype=torch.float32))
        for s in scheds:
            s.step()
    assert len(set(lrs)) > 1 and og.lr == oe.lr
    _close_trajectory(og._flat_p, oe._flat_p, p0)


def test_fp16_overflow_skips_backs_off_and_recaptures_like_eager():
    (mg, cg, og), (me, ce, oe) = _models("tiny", lr=1e-3)
    gs = GraphedTrainStep(mg, cg, og)
    inp, tgt = _batch("tiny", 31, batch=6)
    seeds = lambda k: rng_seed_at(gs.seed_base, k)  # noqa: E731
    _graphed_call(gs, inp, tgt)
    _eager_step(me, ce, oe, inp, tgt, seeds(1))
    for m in (mg, me):
        m.grad_scale = 2.0 ** 60
    snap = _snapshot(mg, og)
    dev_step = int(gs._step.item())
    _graphed_call(gs, inp, tgt, check=False)
    _eager_step(me, ce, oe, inp, tgt, seeds(2))
    torch.cuda.synchronize()
    assert float(og._scratch[2]) == 1.0 and float(oe._scratch[2]) == 1.0
    assert torch.equal(og._flat_p, snap["p"]) and torch.equal(og._m, snap["m"]) and torch.equal(og._v, snap["v"])
    assert torch.equal(mg._packed[mg._fmt(True)], snap["packed"])
    assert int(gs._step.item()) == dev_step
    assert gs.num_graphs == 2  # a second graph for the new scale
    _graphed_call(gs, inp, tgt, check=False)  # consumes replay 2's flag: the scale backs off here, as in eager
    _eager_step(me, ce, oe, inp, tgt, seeds(3))
    assert mg.grad_scale == me.grad_scale == 2.0 ** 59
    assert og.skipped_steps == oe.skipped_steps >= 1 and og.step_count == oe.step_count
    for m in (mg, me):
        m.grad_scale = 1024.0
    for k in range(4, 8):
        _graphed_call(gs, inp, tgt)
        _eager_step(me, ce, oe, inp, tgt, seeds(k))
    torch.cuda.synchronize()
    assert og.step_count == oe.step_count and og.skipped_steps == oe.skipped_steps and mg.grad_scale == me.grad_scale
    assert int(gs._step.item()) == og.step_count
    _close_trajectory(og._flat_p, oe._flat_p, snap["p"])


def test_alternating_shapes_share_one_workspace_and_evict_lru():
    ((model, crit, opt),) = _models("tiny", n=1)
    gs = GraphedTrainStep(model, crit, opt, max_graphs=2)
    shapes = [(60, 12), (40, 20), (75, 32)]
    batches = [_batch("tiny", 300 + i, l_vid=lv, l_txt=lt) for i, (lv, lt) in enumerate(shapes)]
    sizes = []
    for it in range(7):
        inp, tgt = batches[it % 3]
        _graphed_call(gs, inp, tgt)
        assert gs.num_graphs <= 2
        sizes.append(gs.workspace_bytes())
    assert len(gs.captures) == 7  # three shapes cycling through two slots: every call misses
    lib = _lib.load_library()
    need = max(lib.univtg_train_workspace_bytes(ctypes.byref(model._cfg), ctypes.byref(_lib.Shape(4, lv, lt, 1))) for lv, lt in shapes)
    assert sizes[-1] == need and len(set(sizes[2:])) == 1
    gs2 = GraphedTrainStep(model, crit, opt, max_graphs=3)
    for it in range(3):  # (a shape larger than any before grows the shared workspace and drops the graphs made so far)
        _graphed_call(gs2, *batches[it])
    n_cap = len(gs2.captures)
    for it in range(6):
        _graphed_call(gs2, *batches[it % 3])
    assert len(gs2.captures) - n_cap <= 2 and gs2.num_graphs == 3
    n_cap = len(gs2.captures)
    for it in range(6):  # all three held: nothing is captured any more
        _graphed_call(gs2, *batches[it % 3])
    assert len(gs2.captures) == n_cap and gs2.workspace_bytes() == need


def test_graph_eager_graph_equals_all_eager_and_state_dict_round_trip():
    (mg, cg, og), (me, ce, oe) = _models("tiny")
    gs = GraphedTrainStep(mg, cg, og)
    p0 = og._flat_p.clone()
    b = [_batch("tiny", 400 + i) for i in range(4)]
    extra = 0x1234567890ABCDEF
    _graphed_call(gs, *b[0])
    _eager_step(me, ce, oe, *b[0], rng_seed_at(gs.seed_base, 1))
    _eager_step(mg, cg, og, *b[1], extra)
    _eager_step(me, ce, oe, *b[1], extra)
    _graphed_call(gs, *b[2])
    _eager_step(me, ce, oe, *b[2], rng_seed_at(gs.seed_base, 2))
    torch.cuda.synchronize()
    assert og.step_count == oe.step_count == 3 and int(gs._step.item()) == 3
    _close_trajectory(og._flat_p, oe._flat_p, p0)
    sg, se = og.state_dict(), oe.state_dict()
    assert sg["param_groups"] == se["param_groups"] and sg["loss_scale"] == se["loss_scale"]
    assert sg["state"].keys() == se["state"].keys()
    for i in sg["state"]:
        assert float(sg["state"][i]["step"]) == float(se["state"][i]["step"]) == 3.0
    og.load_state_dict(sg)
    n_cap = len(gs.captures)
    _graphed_call(gs, *b[3])  # load_state_dict dropped the graphs: re-captured, and still bit-exact
    assert len(gs.captures) == n_cap + 1 and og.step_count == 4 and int(gs._step.item()) == 4


def test_qfvs_criterion_replay_equals_eager():
    cfg = synth.CONFIGS["tiny"]
    b = synth.make_qfvs_batch(cfg, 32, 4, 24, (24, 24, 24, 10), 3, 5)
    inp = {k: v.cuda() for k, v in b[0].items()}
    tgt = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in b[3].items()}
    mask = b[6].cuda()
    (mg, cg, og), (me, ce, oe) = _models("tiny", qfvs=True)
    gs = GraphedTrainStep(mg, cg, og)
    p0 = og._flat_p.clone()
    _, lg = _graphed_call(gs, inp, tgt, mask)
    _, le = _eager_step(me, ce, oe, inp, tgt, rng_seed_at(gs.seed_base, 1), mask)
    assert torch.equal(lg, le)  # same parameters, same masks: the losses agree bit for bit
    torch.cuda.synchronize()
    _close_trajectory(og._flat_p, oe._flat_p, p0)


def test_refusals_raise_before_any_capture(monkeypatch):
    ((model, crit, opt),) = _models("tiny", n=1)
    gs = GraphedTrainStep(model, crit, opt)
    inp, tgt = _batch("tiny", 5)

    def refused(exc=NotImplementedError, match=None):
        with pytest.raises(exc, match=match):
            gs(inp, tgt)
        assert len(gs.captures) == 0 and gs.replays == 0

    model.reference_rng_order = True
    refused(match="reference_rng_order")
    model.reference_rng_order = False
    model.keep_last_draw = True
    refused(match="keep_last_draw")
    model.keep_last_draw = False
    model._grad_sync = object()  # an armed ddp.OverlappedGradExchange
    refused(match="OverlappedGradExchange")
    model._grad_sync = None
    monkeypatch.setattr(torch.distributed, "is_initialized", lambda: True)
    monkeypatch.setattr(torch.distributed, "get_world_size", lambda *a, **k: 2)
    refused(match="world size")
    monkeypatch.undo()
    out = model(**inp)  # a backward whose gradients no step consumed: accumulation
    crit.weighted_total(crit(out, tgt)).backward()
    refused(match="accumulation")
    opt.zero_grad()
    model.operand_format = 2
    refused(match="fp16x3")
    with pytest.raises(NotImplementedError, match="fp16x3"):
        GraphedTrainStep(model, crit, opt)
    model.operand_format = 0
    with pytest.raises(TypeError):
        GraphedTrainStep(model, crit, torch.optim.SGD([torch.zeros(1, requires_grad=True)], lr=0.1))
    _graphed_call(gs, inp, tgt)  # and after all that the step runs


def test_adamw_step_dev_is_bit_identical_to_adamw_step_and_skips_without_counting():
    """univtg_adamw_step_dev (lr and step in device memory, bias corrections from the table) against univtg_adamw_step on the same
    gradients, over steps 1 .. 40 with a changing lr, a non-finite gradient (skipped: nothing moves, the device step stays) and
    steps past the table (its last row)."""
    from univtg_b200.graphs import bias_correction_table

    lib = _lib.load_library()
    n = 4 * 40000
    g0 = torch.Generator(device="cpu").manual_seed(5)
    p = torch.randn(n, generator=g0).cuda()
    a = dict(p=p.clone(), m=torch.zeros(n, device="cuda"), v=torch.zeros(n, device="cuda"), s=torch.zeros(2048, device="cuda"))
    b = dict(p=p.clone(), m=torch.zeros(n, device="cuda"), v=torch.zeros(n, device="cuda"), s=torch.zeros(2048, device="cuda"))
    table = bias_correction_table(0.9, 0.98, 25).cuda()  # shorter than saturation on purpose: steps 26.. reuse row 25
    full = bias_correction_table(0.9, 0.98)
    lr_dev = torch.zeros(1, device="cuda")
    step_dev = torch.zeros(1, dtype=torch.int32, device="cuda")
    host_step = 0
    for it in range(1, 41):
        g = torch.randn(n, generator=g0).cuda() * (10.0 ** (it % 3 - 2))
        if it == 7:
            g[123] = float("inf")
        lr = 1e-3 * (1.0 + 0.1 * it)
        lr_dev.fill_(lr)
        _lib.check(lib.univtg_adamw_step_dev(_lib.ptr(a["p"]), _lib.ptr(g), _lib.ptr(a["m"]), _lib.ptr(a["v"]), n, _lib.ptr(lr_dev), 0.9,
                                             0.98, 1e-8, 1e-2, _lib.ptr(step_dev), 0.1, 0, _lib.ptr(a["s"]), None, None,
                                             _lib.ptr(table), 25, _lib.stream_ptr()), "adamw_step_dev")
        if it == 7:
            torch.cuda.synchronize()
            assert float(a["s"][2]) == 1.0 and int(step_dev.item()) == host_step
            assert torch.equal(a["p"], b["p"]) and torch.equal(a["m"], b["m"])
            continue
        host_step += 1
        _lib.check(lib.univtg_adamw_step(_lib.ptr(b["p"]), _lib.ptr(g), _lib.ptr(b["m"]), _lib.ptr(b["v"]), n, lr, 0.9, 0.98, 1e-8,
                                         1e-2, host_step, 0.1, 0, _lib.ptr(b["s"]), None, None, _lib.stream_ptr()), "adamw_step")
        torch.cuda.synchronize()
        assert int(step_dev.item()) == host_step
        if host_step <= 25 or tuple(full[host_step - 1].tolist()) == tuple(table[-1].tolist()):
            assert torch.equal(a["p"], b["p"]) and torch.equal(a["m"], b["m"]) and torch.equal(a["v"], b["v"])
            assert torch.equal(a["s"][1], b["s"][1])
    assert host_step == 39
