"""Per-launch cost of the tensor-core GEMM (gemm_wgmma_kernel) at the product's own launches.

Two views, both with CUDA events:
  * groups: every GEMM launch of the cfg2 (B = 32) and cfg5 forwards and of the cfg2 train step's backward, as the plan issues it:
    the same problem list per launch (the QKV, projector and conv-2 launches are groups of two or three problems), the same
    operand layouts (data gradients read an MN-major weight, weight gradients two MN-major operands) and the width / split-K
    factor the plan asks choose_tile for (univtg_debug_choose_tile with the same problems, step 16 for K-major B and 64 for
    MN-major B, and the plan's split limit).  Each launch is timed through univtg_op_gemm_group at the chosen width and at its
    legal neighbours (+-16, +-32; +-64 for MN-major B), as the mean over >= 200 back-to-back launches after warm-up, with
    the main stores of the plan's epilogue (bias, ReLU / GELU, 16-bit or fp32 output, split-K fp32 accumulation).  Not
    reproduced: the conv launches' row-shifted taps (timed as one GEMM with K = 3 taps x channels and the same k-block count),
    row remapping, residual / mask / column-sum options and the training forward's pre-activation and GELU' stores.
    Reported: us per launch, TFLOP/s, share of the data-sheet 989 TFLOP/s (dense fp16, H100 SXM at 700 W), and the sum of
    count x us per step next to the plan's own GEMM time.
  * merged: each backward launch that runs a data gradient together with the weight gradients reading the same operand, against
    the separate launches it replaces (one encoder layer and projector layer 1 at cfg2), both at the plan's widths and splits.
  * plan: the summed GEMM launch times of one cfg2 and cfg5 forward and one cfg2 train step, from the plan's per-launch event
    timeline.

    python tools/gemm_cost.py [--launches 200] [--out results/gemm_cost.json]

Set UNIVTG_LIB to time another build of the same ABI.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from univtg_b200 import _lib, synth  # noqa: E402

PEAK_TFLOPS = 989.0


def kpad(k):
    return (k + 63) // 64 * 64


def P(M, N, K, a_mn=0, b_mn=0, **o):
    """one problem: C[M, N] = sum_k A(m, k) B(n, k); o: act, out16, out32, bias, acc (split-K accumulation into out32)"""
    return dict(M=M, N=N, K=K, a_mn=a_mn, b_mn=b_mn, **o)


def forward_groups(cfg_name):
    """(name, launches per forward, problems, step, max_split) of the inference forward (api.cu: univtg_plan_create and the
    forward's launches)."""
    c = synth.CONFIGS[cfg_name]
    B, Lv, Lt, d, ff, n = c["batch"], c["l_vid"], c["l_txt"], c["hidden_dim"], c["dim_feedforward"], c["enc_layers"]
    M, Mv, Mt, Mh = B * (Lv + Lt), B * Lv, B * Lt, B * (Lv + 1)
    kv, kt = kpad(c["v_feat_dim"]), kpad(c["t_feat_dim"])
    f = f"{cfg_name} fwd"
    return [
        (f"{f} proj0 (vid + txt)", 1, [P(Mv, d, kv, act=1, bias=1, out32=1), P(Mt, d, kt, act=1, bias=1, out32=1)], 16, 1),
        (f"{f} proj1 (vid + txt)", 1, [P(Mv, d, d, bias=1, out32=1, out16=1), P(Mt, d, d, bias=1, out32=1, out16=1)], 16, 1),
        (f"{f} qkv (2d + d)", n, [P(M, 2 * d, d, bias=1, out16=1), P(M, d, d, bias=1, out16=1)], 16, 1),
        (f"{f} out-proj", n, [P(M, d, d, bias=1, out16=1)], 16, 1),
        (f"{f} ffn1", n, [P(M, ff, d, act=2, bias=1, out16=1)], 16, 1),
        (f"{f} ffn2", n, [P(M, d, ff, bias=1, out16=1)], 16, 1),
        (f"{f} conv1", 1, [P(Mh, 2 * d, 3 * d, act=1, bias=1, out16=1)], 16, 1),
        (f"{f} conv2 (class + span)", 1, [P(Mh, d, 3 * d, act=1, bias=1, out16=1)] * 2, 16, 1),
    ]


def backward_groups(cfg_name, separate=False):
    """the backward's launches (train.cu: univtg_backward): data gradients A K-major x B MN-major, weight gradients both
    MN-major with split-K into a pre-zeroed fp32 output.  The last entry of each tuple is the weight gradients' split limit.
    separate: the earlier plan, in which data and weight gradients had launches of their own."""
    c = synth.CONFIGS[cfg_name]
    B, Lv, Lt, d, ff, n = c["batch"], c["l_vid"], c["l_txt"], c["hidden_dim"], c["dim_feedforward"], c["enc_layers"]
    M, Mv, Mt, Mh = B * (Lv + Lt), B * Lv, B * Lt, B * (Lv + 1)
    kv, kt = kpad(c["v_feat_dim"]), kpad(c["t_feat_dim"])
    f = f"{cfg_name} bwd"
    dg = dict(a_mn=0, b_mn=1, out32=1)
    wg = dict(a_mn=1, b_mn=1, out32=1, acc=1)
    g = [
        (f"{f} conv wgrad (3 taps)", 2, [P(d, d, Mh, **wg)] * 3, 64, 8),
        (f"{f} conv2 dgrad (class + span)", 1, [P(Mh, d, 3 * d, **dg)] * 2, 64, 1),
        (f"{f} conv1 dgrad", 1, [P(Mh, d, 6 * d, **dg)], 64, 1),
    ]
    if not separate:
        g += [
            (f"{f} ffn2 dgrad + w2 wgrad", n, [P(M, ff, d, **dg), P(d, ff, M, **wg)], 64, 4),
            (f"{f} ffn1 dgrad + w1 wgrad", n, [P(M, d, ff, **dg), P(ff, d, M, **wg)], 64, 4),
            (f"{f} out-proj dgrad + wgrad", n, [P(M, d, d, **dg), P(d, d, M, **wg)], 64, 4),
            (f"{f} qkv dgrad + wgrad (2d + d)", n, [P(M, d, 3 * d, **dg), P(2 * d, d, M, **wg), P(d, d, M, **wg)], 64, 4),
            (f"{f} proj0 wgrad (vid + txt)", 1, [P(d, kv, Mv, **wg), P(d, kt, Mt, **wg)], 64, 16),
            (f"{f} proj0 dgrad (vid + txt)", 1, [P(Mv, kv, d, **dg), P(Mt, kt, d, **dg)], 64, 1),
            (f"{f} proj1 wgrad + dgrad (vid + txt)", 1, [P(d, d, Mv, **wg), P(d, d, Mt, **wg), P(Mv, d, d, **dg), P(Mt, d, d, **dg)], 64, 4),
        ]
        return g
    g += [
        (f"{f} ffn2 dgrad", n, [P(M, ff, d, **dg)], 64, 1),
        (f"{f} ffn wgrad (w2 + w1)", n, [P(d, ff, M, **wg), P(ff, d, M, **wg)], 64, 16),
        (f"{f} ffn1 dgrad", n, [P(M, d, ff, **dg)], 64, 1),
        (f"{f} out-proj dgrad", n, [P(M, d, d, **dg)], 64, 1),
        (f"{f} out-proj wgrad", n, [P(d, d, M, **wg)], 64, 16),
        (f"{f} qkv dgrad", n, [P(M, d, 3 * d, **dg)], 64, 1),
        (f"{f} qkv wgrad (2d + d)", n, [P(2 * d, d, M, **wg), P(d, d, M, **wg)], 64, 16),
    ]
    for i, (nv, nt) in enumerate(((kv, kt), (d, d))):
        g.append((f"{f} proj{i} wgrad (vid + txt)", 1, [P(d, nv, Mv, **wg), P(d, nt, Mt, **wg)], 64, 16))
        g.append((f"{f} proj{i} dgrad (vid + txt)", 1, [P(Mv, nv, d, **dg), P(Mt, nt, d, **dg)], 64, 1))
    return g


def choose(probs, num_sms, step, max_split):
    """width and per-problem split-K factors (problems without split-K accumulation: limit 1)"""
    lib = _lib.load_library()
    n = len(probs)
    Ms = (ctypes.c_int32 * n)(*[p["M"] for p in probs])
    Ns = (ctypes.c_int32 * n)(*[p["N"] for p in probs])
    Ks = (ctypes.c_int32 * n)(*[(p["K"] + 63) // 64 for p in probs])
    lim = (ctypes.c_int32 * n)(*[max_split if p.get("acc") else 1 for p in probs])
    bn, ks = ctypes.c_int32(0), (ctypes.c_int32 * n)()
    _lib.check(lib.univtg_debug_choose_tile_group(Ms, Ns, Ks, lim, n, num_sms, step, ctypes.byref(bn), ks), "choose_tile")
    return bn.value, list(ks)


def time_group(probs, bn, ksplit, launches):
    lib = _lib.load_library()
    keep, arr = [], (_lib.GemmProblem * len(probs))()
    for i, q in enumerate(probs):
        M, N, K = q["M"], q["N"], q["K"]
        g = torch.Generator().manual_seed(M + N + K + i)
        a = (torch.randn(K, M, generator=g) if q["a_mn"] else torch.randn(M, K, generator=g)).half().cuda()
        b = (torch.randn(K, N, generator=g) if q["b_mn"] else torch.randn(N, K, generator=g)).mul(0.05).half().cuda()
        p = arr[i]
        p.a, p.lda, p.a_mn = a.data_ptr(), (M if q["a_mn"] else K), q["a_mn"]
        p.b, p.ldb, p.b_mn = b.data_ptr(), (N if q["b_mn"] else K), q["b_mn"]
        p.M, p.N, p.K, p.ksplit = M, N, K, (ksplit[i] if q.get("acc") else 1)
        p.a_fmt, p.b_fmt, p.out_fmt, p.alpha, p.colsum_scale = -1, -1, -1, 1.0, 1.0
        p.act = q.get("act", 0)
        keep += [a, b]
        if q.get("bias"):
            bias = torch.randn(N, generator=g).cuda()
            p.bias = bias.data_ptr()
            keep.append(bias)
        if q.get("out32"):
            o32 = torch.zeros(M, N, device="cuda")
            p.out32, p.ld32, p.accumulate = o32.data_ptr(), N, 1 if q.get("acc") else 0
            keep.append(o32)
        if q.get("out16"):
            o16 = torch.empty(M, N, dtype=torch.float16, device="cuda")
            p.out16, p.ld16 = o16.data_ptr(), N
            keep.append(o16)
    full = ctypes.c_int32(-1)
    stream = _lib.stream_ptr()

    def launch():
        _lib.check(lib.univtg_op_gemm_group(arr, len(probs), 0, bn, 1, ctypes.byref(full), stream), "op_gemm_group")

    for _ in range(20):
        launch()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / launches * 1e3
    tf = sum(2.0 * q["M"] * q["N"] * q["K"] for q in probs) / (us * 1e-6) / 1e12
    return dict(us=round(us, 3), tflops=round(tf, 1), peak_share=round(tf / PEAK_TFLOPS, 4), full=full.value)


def merged_comparison(num_sms, launches):
    """each merged backward launch of cfg2 against the separate launches it replaces (per encoder layer: the FFN pair of launches
    against FFN2 dgrad, the FFN weight-gradient launch and FFN1 dgrad)"""
    new = {name.split(" bwd ")[1]: (probs, step, ms) for name, _, probs, step, ms in backward_groups("cfg2")}
    old = {name.split(" bwd ")[1]: (probs, step, ms) for name, _, probs, step, ms in backward_groups("cfg2", separate=True)}

    def t(entry):
        probs, step, ms = entry
        bn, ks = choose(probs, num_sms, step, ms)
        return time_group(probs, bn, ks, launches)["us"], bn, ks

    pairs = [("ffn (two launches)", ["ffn2 dgrad + w2 wgrad", "ffn1 dgrad + w1 wgrad"], ["ffn2 dgrad", "ffn wgrad (w2 + w1)", "ffn1 dgrad"]),
             ("out-proj", ["out-proj dgrad + wgrad"], ["out-proj dgrad", "out-proj wgrad"]),
             ("qkv", ["qkv dgrad + wgrad (2d + d)"], ["qkv dgrad", "qkv wgrad (2d + d)"]),
             ("proj1", ["proj1 wgrad + dgrad (vid + txt)"], ["proj1 wgrad (vid + txt)", "proj1 dgrad (vid + txt)"])]
    rows = []
    for name, merged, separate in pairs:
        m = [t(new[k]) for k in merged]
        s = [t(old[k]) for k in separate]
        mu, su = sum(x[0] for x in m), sum(x[0] for x in s)
        rows.append(dict(name=name, merged_us=round(mu, 3), separate_us=round(su, 3),
                         merged=[dict(launch=k, us=round(x[0], 3), bn=x[1], ksplit=x[2]) for k, x in zip(merged, m)],
                         separate=[dict(launch=k, us=round(x[0], 3), bn=x[1], ksplit=x[2]) for k, x in zip(separate, s)]))
        print(f"merged {name:20s} {mu:8.2f} us  separate {su:8.2f} us ({mu / su - 1:+.1%})  "
              f"merged {[(x[1], x[2]) for x in m]} separate {[(x[1], x[2]) for x in s]}", flush=True)
    return rows


def plan_gemm_ms(cfg_name, train):
    from univtg_b200 import build_model

    cfg = synth.CONFIGS[cfg_name]
    args = synth.reference_args(cfg, device="cuda:0")
    model, crit = build_model(args)
    model.load_state_dict(synth.make_state_dict(cfg, seed=0), strict=True)
    model.cuda()
    crit.cuda()
    inp = {k: v.cuda() for k, v in synth.make_inputs(cfg, seed=1).items()}
    B, Lv, Lt = cfg["batch"], cfg["l_vid"], cfg["l_txt"]
    res = []
    if train:
        from univtg_b200.optim import FlatAdamW

        model.train()
        crit.train()
        tgt = {k: (v.cuda() if torch.is_tensor(v) else v) for k, v in synth.make_targets(synth.make_inputs(cfg, seed=1), seed=2).items()}
        opt = FlatAdamW(model, lr=1e-4)
    for _ in range(5):
        if train:
            def run():
                opt.zero_grad(set_to_none=True)
                total = crit.weighted_total(crit(model(**inp), tgt))
                total.backward()
            tl = model.profile_train_step(B, Lv, Lt, run)
        else:
            model.eval()
            with torch.no_grad():
                tl = model.profile_forward(inp)
        g = [ms for k, ms in tl if k == 1]
        res.append((sum(g), len(g)))
    res.sort()
    ms, n = res[len(res) // 2]
    return dict(gemm_ms=round(ms, 4), launches=n)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clk = [s.strip() for s in q.split(",")]
        return dict(name=name, power_limit=power, max_sm_clock=clk)
    except Exception as ex:  # the timings stay valid; the card is then named by torch alone
        return dict(name=torch.cuda.get_device_name(), error=repr(ex)[:200])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "gemm_cost.json"))
    ap.add_argument("--no-plan", action="store_true", help="skip the product-plan timelines")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_cost.py needs a GPU"
    assert args.launches >= 200, "at least 200 launches per point"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows, per_step = [], {}
    sets = (("cfg2_fwd", forward_groups("cfg2")), ("cfg5_fwd", forward_groups("cfg5")), ("cfg2_bwd", backward_groups("cfg2")))
    for set_name, groups in sets:
        total = 0.0
        for name, count, probs, step, max_split in groups:
            bn0, ks = choose(probs, sms, step, max_split)
            widths = sorted({w for w in (bn0 - 2 * step, bn0 - step, bn0, bn0 + step, bn0 + 2 * step) if 32 <= w <= 256 and w % step == 0}
                            if step == 64 else {w for w in (bn0 - 32, bn0 - 16, bn0, bn0 + 16, bn0 + 32) if 32 <= w <= 256})
            pts = {w: time_group(probs, w, ks, args.launches) for w in widths}
            total += count * pts[bn0]["us"]
            rows.append(dict(set=set_name, name=name, count=count, problems=probs, chosen_bn=bn0, ksplit=ks, widths=pts))
            best = min(pts, key=lambda w: pts[w]["us"])
            shp = " + ".join(f"{q['M']}x{q['N']}x{q['K']}" for q in probs)
            print(f"{name:34s} x{count} [{shp}] ks {ks}  chosen bn {bn0:3d}: {pts[bn0]['us']:8.2f} us {pts[bn0]['tflops']:6.1f} TF/s "
                  f"({100 * pts[bn0]['peak_share']:4.1f} %)  best bn {best:3d}: {pts[best]['us']:8.2f} us ({pts[best]['us'] / pts[bn0]['us'] - 1:+.1%})",
                  flush=True)
        per_step[set_name] = round(total / 1e3, 4)
    print("sum of count x us at the chosen widths, ms:", per_step)
    merged = merged_comparison(sms, args.launches)
    plan = {}
    if not args.no_plan:
        plan = {"cfg2_fwd": plan_gemm_ms("cfg2", False), "cfg5_fwd": plan_gemm_ms("cfg5", False), "cfg2_train": plan_gemm_ms("cfg2", True)}
        print("plan GEMM time per step:", plan)
    res = dict(gpu=gpu_info(), lib=os.environ.get("UNIVTG_LIB", "default"), launches=args.launches, peak_tflops=PEAK_TFLOPS,
               groups=rows, modelled_ms=per_step, merged=merged, plan=plan)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
