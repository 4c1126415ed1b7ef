"""GPU parity of query-focused video summarisation (univtg_b200.qfvs): the criterion kernels against fp64 autograd through
oracle/qfvs_oracle.py, the training step of main/train_qfvs.py:179-204 (three forwards, three criterion calls, one backward)
against the oracle, and the evaluation's top-k shot selection (main/inference_qfvs.py:114-138).  The bars are those of
tests/test_train_gpu.py."""
import gc

import pytest
import torch

from tests.test_train_gpu import _grad_verdict
from univtg_b200 import synth
from univtg_b200.qfvs import build_model

pytestmark = pytest.mark.gpu

# (config, S, Lf, seg_len, L1, L2): the golden tiny case, and cfg2 dims at the reference's max_segment_num x max_frame_num
SHAPES = {"tiny": ("tiny", 4, 24, (24, 24, 24, 10), 3, 5),
          "cfg2_s20": ("cfg2", 20, 200, (200,) * 18 + (131, 0), 8, 8)}
NEAR_TOL = {"tiny": 2.5e-2, "cfg2_s20": 2e-2}


def _batch(name, seed=32, device="cuda"):
    cfg_name, S, Lf, seg_len, L1, L2 = SHAPES[name]
    cfg = synth.CONFIGS[cfg_name]
    b = synth.make_qfvs_batch(cfg, seed, S, Lf, seg_len, L1, L2)
    mv = lambda d: {k: v.to(device) for k, v in d.items()}  # noqa: E731
    return cfg, [mv(x) for x in b[:6]] + [b[6].to(device)]


def _models(cfg, seed=31):
    model, crit = build_model(synth.reference_args(cfg, device="cuda:0", dset_type="vs", droppath=0.0, input_dropout=0.0))
    model.load_state_dict(synth.make_state_dict(cfg, seed=seed), strict=True)
    return model.to("cuda:0"), crit.to("cuda:0")


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _cos(a, b):
    return float((a.flatten() @ b.flatten()) / (a.norm() * b.norm()).clamp_min(1e-30))


def _total(d, wd):
    return sum(d[k] * wd[k] for k in d.keys() if k in wd)


def _edge_targets(tg, count):
    zero = torch.zeros_like(tg["saliency_scores"])
    beyond = zero.clone()
    beyond[0, count - 3:count + 5] = 1.0
    return {"base": tg, "all_zero": dict(tg, saliency_scores=zero), "beyond_count": dict(tg, saliency_scores=beyond),
            "no_pos_labels": {k: v for k, v in tg.items() if k != "saliency_pos_labels"}}


@pytest.mark.parametrize("name", list(SHAPES))
def test_criterion_kernels_match_oracle(name):
    """The criterion alone, fed the exact oracle's outputs: losses to fp32 round-off, output gradients within 2e-4 (rel-L2);
    exact zeros where the reference returns 0."""
    from oracle import qfvs_oracle as QO
    from oracle import univtg_oracle as O

    cfg, b = _batch(name)
    inputs, targets, mask = b[:3], b[3:6], b[6]
    sd = {k: v.cuda() for k, v in synth.make_state_dict(cfg, seed=31).items()}
    _, crit = _models(cfg)
    with torch.no_grad():
        out = O.forward(sd, cfg, **inputs[2])
    count = int(mask.sum())
    cases = _edge_targets(targets[2], count)
    pl = out["pred_logits"].clone()
    kept = torch.nonzero(mask.reshape(-1)).flatten()
    t_kept = targets[2]["saliency_scores"][0, :count]
    for j in range(4):  # pred_logits exactly 0 / 1 against targets 0 / 1: the BCE's log clamp at -100
        pl.view(-1)[kept[int(torch.nonzero(t_kept == j % 2).flatten()[j])]] = float(j // 2)
    cases["clamp"] = targets[2]
    for case, tg in cases.items():
        leaves = {"pred_logits": pl if case == "clamp" else out["pred_logits"], "vid_mem_proj": out["vid_mem_proj"],
                  "txt_mem_proj": out["txt_mem_proj"]}
        leaves = {k: v.clone().requires_grad_(True) for k, v in leaves.items()}
        sal = QO.saliency_scores(leaves["vid_mem_proj"], leaves["txt_mem_proj"], inputs[2]["src_vid_mask"])
        ref = QO.criterion({"pred_logits": leaves["pred_logits"], "saliency_scores": sal}, tg, mask)
        rt = _total(ref, crit.weight_dict)
        if rt.requires_grad:
            rt.backward()
        got_leaves = {k: v.detach().float().requires_grad_(True) for k, v in leaves.items()}
        got = crit(dict(got_leaves, src_vid_mask=inputs[2]["src_vid_mask"]), tg, mask)
        assert sorted(got) == sorted(ref)
        for k in ref:
            r = float(ref[k])
            if r == 0.0:
                assert float(got[k]) == 0.0, (name, case, k)
            else:
                assert abs(float(got[k]) - r) <= 2e-5 * max(1.0, abs(r)), (name, case, k, float(got[k]), r)
        crit.weighted_total(got).backward()
        for k, v in leaves.items():
            g = got_leaves[k].grad.double()
            if v.grad is None or float(v.grad.abs().max()) == 0.0:
                assert float(g.abs().max()) == 0.0, (name, case, k)
            else:
                assert _rel(g, v.grad) < 2e-4, (name, case, k, _rel(g, v.grad))


def test_criterion_runs_without_host_synchronisation():
    """Forward and backward of three criterion calls with torch's sync debug mode raising on any host synchronisation."""
    cfg, b = _batch("tiny")
    model, crit = _models(cfg)
    model.train()
    outs = [{k: (v.detach().requires_grad_(True) if v.is_floating_point() and k != "src_vid_mask" else v) for k, v in model(**inp).items()}
            for inp in b[:3]]  # leaves: the backward below is the criterion's alone
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        dicts = [crit(o, t, b[6]) for o, t in zip(outs, b[3:6])]
        total = _total({k: dicts[0][k] + dicts[1][k] + dicts[2][k] for k in dicts[0]}, crit.weight_dict)
        total.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(total).item()
    assert all(o["vid_mem_proj"].grad is not None and o["pred_logits"].grad is not None for o in outs)


def _oracle_step(cfg, inputs, targets, mask, gather, wd, emulate):
    from oracle import qfvs_oracle as QO
    from oracle import univtg_oracle as O

    leaves = {k: v.cuda().double().requires_grad_(True) for k, v in synth.make_state_dict(cfg, seed=31).items()}
    opq = O.round_fp16 if emulate else None
    dicts = [QO.criterion(O.forward(leaves, cfg, **inp, opq=opq), tg, mask) for inp, tg in zip(inputs, targets)]
    ld = QO.gather(dicts, gather)
    _total(ld, wd).backward()
    return ld, {k: v.grad for k, v in leaves.items()}


@pytest.mark.parametrize("gather", [1, 0])
@pytest.mark.parametrize("name", list(SHAPES))
def test_full_training_step_gradients(name, gather):
    cfg, b = _batch(name)
    inputs, targets, mask = b[:3], b[3:6], b[6]
    model, crit = _models(cfg)
    model.train()
    outs = [model(**inp) for inp in inputs]
    dicts = [crit(o, t, mask) for o, t in zip(outs, targets)]
    ld = {k: dicts[0][k] + dicts[1][k] + dicts[2][k] for k in dicts[0]} if gather > 0 else dicts[2]
    _total(ld, crit.weight_dict).backward()
    torch.cuda.synchronize()
    xl, xg = _oracle_step(cfg, inputs, targets, mask, gather, crit.weight_dict, False)
    el, eg = _oracle_step(cfg, inputs, targets, mask, gather, crit.weight_dict, True)
    for k in xl:
        assert abs(float(ld[k]) - float(xl[k])) <= 1e-3 * max(1.0, abs(float(xl[k]))), (name, k, float(ld[k]), float(xl[k]))
        assert abs(float(ld[k]) - float(el[k])) <= 1e-4 * max(1.0, abs(float(el[k]))), (name, k, float(ld[k]), float(el[k]))
    worst = {}
    for n_, p in model.named_parameters():
        og = xg[n_]
        if og is None or float(og.abs().max()) == 0.0:
            assert p.grad is None or float(p.grad.abs().max()) == 0.0, f"{n_} must not receive a gradient"
            continue
        g = p.grad.double()
        assert bool(torch.isfinite(g).all()), n_
        worst[n_] = (_rel(g, og), _cos(g, og), _rel(g, eg[n_]))
    bad = _grad_verdict(worst, NEAR_TOL[name])
    assert not bad, f"{name} gather={gather}: gradient mismatch (rel-L2 exact, cosine exact, rel-L2 emulating) {bad}"


def test_unused_forwards_return_their_workspaces():
    """qfvs_loss_gather = 0: two of the three forwards never see a backward; their workspace leases go back to the pool."""
    cfg, b = _batch("tiny")
    model, crit = _models(cfg)
    model.train()

    def step():
        outs = [model(**inp) for inp in b[:3]]
        dicts = [crit(o, t, b[6]) for o, t in zip(outs, b[3:6])]
        _total(dicts[2], crit.weight_dict).backward()

    for _ in range(5):
        step()
        gc.collect()
    torch.cuda.synchronize()
    assert len(model.__dict__.get("_train_pool", [])) <= 3


def test_flat_adamw_lowers_the_gathered_loss():
    from univtg_b200.optim import FlatAdamW

    cfg, b = _batch("tiny")
    model, crit = _models(cfg)
    model.train()
    opt = FlatAdamW(model, lr=5e-4, weight_decay=1e-4, max_grad_norm=0.1)
    vals = []
    for _ in range(10):
        outs = [model(**inp) for inp in b[:3]]
        dicts = [crit(o, t, b[6]) for o, t in zip(outs, b[3:6])]
        total = _total({k: dicts[0][k] + dicts[1][k] + dicts[2][k] for k in dicts[0]}, crit.weight_dict)
        opt.zero_grad()
        total.backward()
        opt.step()
        vals.append(float(total))
    assert vals[-1] < vals[0], vals


def _scores(outs, mask_sf, output_type, score_gather):
    """main/inference_qfvs.py:114-131: per query, the masked output(s), summed over the three queries when qfvs_score_gather."""
    types = output_type if isinstance(output_type, list) else [output_type]
    per_q = [sum(o[t].squeeze().masked_select(mask_sf) for t in types) for o in outs]
    return per_q[0] + per_q[1] + per_q[2] if score_gather else per_q[2]


def test_evaluation_selects_the_oracle_shots():
    """The scoring body of main/inference_qfvs.py:114-138 on the port's eval outputs picks the exact oracle's top-k shots
    whenever the oracle's margin at the cut-off exceeds the fp16 tolerance."""
    from oracle import univtg_oracle as O

    compared = 0
    for name in SHAPES:
        cfg, b = _batch(name)
        inputs, mask = b[:3], b[6]
        S, Lf = inputs[0]["src_vid_mask"].shape
        mask_sf = mask.reshape(S, Lf)
        model, _ = _models(cfg)
        model.eval()
        sd = {k: v.cuda().double() for k, v in synth.make_state_dict(cfg, seed=31).items()}
        with torch.no_grad():
            outs = [model(**inp) for inp in inputs]
            ref = [O.forward(sd, cfg, **inp) for inp in inputs]
        for output_type in ("pred_logits", "saliency_scores", ["pred_logits", "saliency_scores"]):
            for score_gather in (0, 1):
                got = _scores(outs, mask_sf, output_type, score_gather)
                exp = _scores(ref, mask_sf, output_type, score_gather)
                # the fp16 forward bar (DESIGN.md section 3: rtol 1e-3 / atol 1e-4 on scores of magnitude <= 1) per summed term
                tol = 2e-3 * (3 if score_gather else 1) * (2 if isinstance(output_type, list) else 1)
                assert float((got.double() - exp).abs().max()) < tol, (name, output_type, score_gather)
                # every cut-off k: top-k sets agree iff the largest of our ranks among the oracle's k best is k - 1
                order_exp = exp.argsort(descending=True)
                rank_got = torch.empty_like(order_exp)
                rank_got[got.argsort(descending=True)] = torch.arange(got.numel(), device=got.device)
                same = rank_got[order_exp].cummax(0).values == torch.arange(got.numel(), device=got.device)
                srt = exp[order_exp]
                clear = (srt[:-1] - srt[1:]) > 2 * tol  # margin at cut-off k = i + 1
                assert bool(same[:-1][clear].all()), (name, output_type, score_gather)
                compared += int(clear.sum())
                for top_percent in (0.1, 0.2, 0.5):  # the reference's own topk call where its cut-off is clear
                    k = int(got.shape[0] * top_percent)
                    if k >= 1 and bool(clear[k - 1]):
                        assert set(got.topk(k)[1].tolist()) == set(exp.topk(k)[1].tolist()), (name, output_type, top_percent)
    print("clear cut-offs compared:", compared)
    assert compared >= 20, compared
