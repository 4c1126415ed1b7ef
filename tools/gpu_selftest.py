#!/usr/bin/env python
"""Operator-level self test on a real H100: each case runs in its own subprocess under a timeout so a hung
kernel cannot take the whole run down.  Usage: python tools/gpu_selftest.py [case ...]  (writes results/selftest.json)"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _t16(x, fmt):
    import torch
    return x.to(torch.bfloat16 if fmt else torch.float16)


def case_gemm(M, N, K, a_mn, b_mn, fmt, bn, ksplit, act, use_bias, cluster=False):
    import torch
    from univtg_b200 import _lib
    lib = _lib.load_library()
    gemm_fn = lib.univtg_op_gemm_cluster if cluster else lib.univtg_op_gemm
    g = torch.Generator(device="cpu").manual_seed(1234 + M + N + K)
    A = torch.randn(M, K, generator=g).cuda()
    Bm = torch.randn(N, K, generator=g).cuda()
    bias = torch.randn(N, generator=g).cuda() if use_bias else None
    A16, B16 = _t16(A, fmt), _t16(Bm, fmt)
    ref = A16.float() @ B16.float().t()
    if bias is not None:
        ref = ref + bias
    if act == 1:
        ref = torch.relu(ref)
    elif act == 2:
        ref = torch.nn.functional.gelu(ref)
    ref = ref * 0.5
    a_in = A16.t().contiguous() if a_mn else A16.contiguous()
    b_in = B16.t().contiguous() if b_mn else B16.contiguous()
    out32 = torch.zeros(M, N, device="cuda")
    out16 = torch.zeros(M, N, device="cuda", dtype=A16.dtype) if ksplit == 1 else None
    rc = gemm_fn(_lib.ptr(a_in), _lib.ptr(b_in), M, N, K, a_mn, b_mn, fmt, bn, ksplit, _lib.ptr(bias), act, 0.5,
                 _lib.ptr(out32), _lib.ptr(out16), _lib.stream_ptr())
    _lib.check(rc, "op_gemm")
    torch.cuda.synchronize()
    err = (out32 - ref).abs().max().item()
    scale = ref.abs().max().item()
    res = {"max_abs_err": err, "ref_max": scale}
    if out16 is not None:
        res["err16"] = (out16.float() - ref).abs().max().item()
    res["ok"] = bool(err <= 2e-3 * max(scale, 1.0) * (1 if K <= 4096 else 4))
    if not res["ok"]:
        bad = ((out32 - ref).abs() > 1e-2 * max(scale, 1.0)).nonzero()
        res["n_bad"] = int(bad.shape[0])
        res["first_bad"] = bad[:8].tolist()
        res["sample"] = [out32[0, :4].tolist(), ref[0, :4].tolist()]
    return res


def case_gemm_timeline(M, N, K, act, want32, want16, bn, cluster=False, a_mn=0, b_mn=0):
    """Per-CTA phase timeline (ns) of one GEMM launch: where does the time go?"""
    import torch
    from univtg_b200 import _lib
    lib = _lib.load_library()
    A = torch.randn(K, M, device="cuda").half() if a_mn else torch.randn(M, K, device="cuda").half()
    Bm = torch.randn(K, N, device="cuda").half() if b_mn else torch.randn(N, K, device="cuda").half()
    bias = torch.randn(N, device="cuda")
    out32 = torch.zeros(M, N, device="cuda") if want32 else None
    out16 = torch.zeros(M, N, device="cuda", dtype=torch.float16) if want16 else None
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    buf = torch.zeros(sms * 8, dtype=torch.int64, device="cuda")

    fn = lib.univtg_op_gemm_cluster if cluster else lib.univtg_op_gemm

    def run():
        _lib.check(fn(_lib.ptr(A), _lib.ptr(Bm), M, N, K, a_mn, b_mn, 0, bn, 1, _lib.ptr(bias), act, 1.0, _lib.ptr(out32),
                      _lib.ptr(out16), _lib.stream_ptr()), "op_gemm")
    return _timeline(run, sms, buf)


def _timeline(run, sms, buf):
    """Warm up, then record the per-CTA %globaltimer stamps of one launch (stamps of a CTA's last tile) and its event time."""
    import torch
    from univtg_b200 import _lib
    lib = _lib.load_library()
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    lib.univtg_debug_gemm_timeline(_lib.ptr(buf))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run()
    e1.record()
    torch.cuda.synchronize()
    lib.univtg_debug_gemm_timeline(None)
    t = buf.view(sms, 8).cpu()
    used = t[:, 0] > 0
    t = t[used]
    rel = (t - int(t[:, 0].min())).float() / 1000.0  # us
    names = ["entry", "setup", "tma_issued", "first_stage", "last_mma", "unused", "epi_done", "exit"]
    res = {"event_us": e0.elapsed_time(e1) * 1e3, "ctas": int(used.sum()), "ok": True}
    for i, n in enumerate(names):
        col = rel[:, i][t[:, i] > 0]  # CTA-pair mode: only the leader CTA stamps the MMA-side events
        res[n] = [round(float(col.min()), 2), round(float(col.median()), 2), round(float(col.max()), 2)] if col.numel() else None
    both = (t[:, 4] > 0) & (t[:, 6] > 0)
    res["epi_us"] = round(float(((t[both, 6] - t[both, 4]).float() / 1000.0).median()), 2)  # stamp 4 -> 6, median over CTAs
    # the same launch without the timeline buffer: mean of 50 back-to-back launches
    e0.record()
    for _ in range(50):
        run()
    e1.record()
    torch.cuda.synchronize()
    res["mean_us"] = round(e0.elapsed_time(e1) * 1e3 / 50, 2)
    return res


def case_group_timeline(kind, bn):
    """Phase timeline of one launch of the train step's backward, with the plan's epilogue options (train.cu, cfg2 sizes):
    ffn2_dgrad: 16-bit out * saved GELU' (mask16) + column sums;  ffn1_dgrad / qkv_dgrad: fp32 out + fp32 residual;
    out_dgrad: 16-bit out;  qkv_wgrad: [2d | d] x d weight gradients, both operands MN-major, split-K 4 into fp32."""
    import torch
    from univtg_b200 import _lib
    lib = _lib.load_library()
    M, d = 3424, 1024
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    buf = torch.zeros(sms * 8, dtype=torch.int64, device="cuda")
    keep = []

    def h(*shape):
        x = (torch.randn(*shape, device="cuda") * 0.1).half()
        keep.append(x)
        return x

    def f(*shape):
        x = torch.randn(*shape, device="cuda")
        keep.append(x)
        return x

    def dgrad(K):
        p = _lib.GemmProblem()
        a, b = h(M, K), h(K, d)
        p.a, p.lda, p.a_mn, p.b, p.ldb, p.b_mn = _lib.ptr(a), K, 0, _lib.ptr(b), d, 1
        p.M, p.N, p.K, p.ksplit, p.a_fmt, p.b_fmt, p.out_fmt, p.alpha = M, d, K, 1, -1, -1, -1, 1.0
        return p

    if kind == "qkv_wgrad":
        probs = []
        dq = h(M, 3 * d)
        for N, off in ((2 * d, 0), (d, 2 * d)):
            p = _lib.GemmProblem()
            x = h(M, d)
            out = f(N, d)
            p.a, p.lda, p.a_mn, p.b, p.ldb, p.b_mn = dq.data_ptr() + 2 * off, 3 * d, 1, x.data_ptr(), d, 1  # columns [off, off + N)
            p.M, p.N, p.K, p.ksplit, p.a_fmt, p.b_fmt, p.out_fmt, p.alpha = N, d, M, 4, -1, -1, -1, 1.0 / 1024
            p.out32, p.ld32 = _lib.ptr(out), d
            probs.append(p)
    else:
        p = dgrad(3 * d if kind == "qkv_dgrad" else d)
        if kind.startswith("ffn2_dgrad"):  # _nomask / _nocolsum: the same launch without one of its two extra options
            if kind != "ffn2_dgrad_nomask":
                p.mask16, p.ld_mask, p.mask_mul = _lib.ptr(h(M, d)), d, 1
            p.out16, p.ld16 = _lib.ptr(h(M, d)), d
            if kind != "ffn2_dgrad_nocolsum":
                p.colsum, p.colsum_scale = _lib.ptr(f(d)), 1.0 / 1024
        elif kind in ("ffn1_dgrad", "qkv_dgrad"):
            p.resid, p.ld_resid = _lib.ptr(f(M, d)), d
            p.out32, p.ld32 = _lib.ptr(f(M, d)), d
        else:
            p.out16, p.ld16 = _lib.ptr(h(M, d)), d
        probs = [p]
    arr = (_lib.GemmProblem * len(probs))(*probs)

    def run():
        _lib.check(lib.univtg_op_gemm_group(arr, len(probs), 0, bn, 1, None, _lib.stream_ptr()), "op_gemm_group")
    return _timeline(run, sms, buf)


def case_layernorm(rows, d, ld16, fmt):
    import torch
    from univtg_b200 import _lib
    lib = _lib.load_library()
    g = torch.Generator(device="cpu").manual_seed(7)
    x = (torch.randn(rows, d, generator=g) * 2 + 0.5).cuda()
    w = torch.randn(d, generator=g).cuda()
    b = torch.randn(d, generator=g).cuda()
    out32 = torch.empty(rows, d, device="cuda")
    out16 = torch.full((rows, ld16), 7.0, device="cuda", dtype=torch.bfloat16 if fmt else torch.float16)
    rc = lib.univtg_op_layernorm(_lib.ptr(x), rows, d, _lib.ptr(w), _lib.ptr(b), 1e-5, fmt, _lib.ptr(out32), _lib.ptr(out16), ld16,
                                 _lib.stream_ptr())
    _lib.check(rc, "op_layernorm")
    torch.cuda.synchronize()
    ref = torch.nn.functional.layer_norm(x, (d,), w, b, 1e-5)
    e32 = (out32 - ref).abs().max().item()
    e16 = (out16[:, :d].float() - _t16(ref, fmt).float()).abs().max().item()
    pad = out16[:, d:].float().abs().max().item() if ld16 > d else 0.0
    return {"err32": e32, "err16": e16, "pad_max": pad, "ok": bool(e32 < 2e-5 and e16 < 2e-2 and pad == 0.0)}


def case_attention(B, L, H, dh, fmt, impl):
    import torch
    from univtg_b200 import _lib
    lib = _lib.load_library()
    d = H * dh
    g = torch.Generator(device="cpu").manual_seed(99)
    q = torch.randn(B, L, H, dh, generator=g).cuda()
    k = torch.randn(B, L, H, dh, generator=g).cuda()
    v = torch.randn(B, L, H, dh, generator=g).cuda()
    lens = torch.randint(max(1, L // 3), L + 1, (B,), generator=g)
    lens[0] = L
    mask = (torch.arange(L)[None, :] < lens[:, None]).float().cuda()
    q16, k16, v16 = _t16(q, fmt), _t16(k, fmt), _t16(v, fmt)
    qkv = torch.cat([q16.reshape(B * L, d), k16.reshape(B * L, d), v16.reshape(B * L, d)], dim=1).contiguous()
    out = torch.zeros(B * L, d, device="cuda", dtype=q16.dtype)
    lse = torch.zeros(B, H, L, device="cuda")
    rc = lib.univtg_op_attention(_lib.ptr(qkv), _lib.ptr(mask), _lib.ptr(out), _lib.ptr(lse), B, L, H, dh, fmt, impl,
                                 _lib.stream_ptr())
    _lib.check(rc, "op_attention")
    torch.cuda.synchronize()
    s = torch.einsum("bihc,bjhc->bhij", q16.float(), k16.float()) * (dh ** -0.5)
    s = s.masked_fill(mask[:, None, None, :] == 0, float("-inf"))
    p = torch.softmax(s, dim=-1)
    ref = torch.einsum("bhij,bjhc->bihc", p, v16.float()).reshape(B * L, d)
    ref_lse = torch.logsumexp(s, dim=-1)
    err = (out.float() - ref).abs().max().item()
    elz = (lse - ref_lse).abs().max().item()
    res = {"max_abs_err": err, "lse_err": elz, "ref_max": ref.abs().max().item(), "ok": bool(err < 2e-2 and elz < 1e-3)}
    if not res["ok"]:
        res["sample"] = [out[0, :4].float().tolist(), ref[0, :4].tolist()]
    return res


def case_attention_bwd(B, L, H, dh, fmt, impl):
    import torch
    from univtg_b200 import _lib
    lib = _lib.load_library()
    d = H * dh
    g = torch.Generator(device="cpu").manual_seed(321)
    q = torch.randn(B, L, H, dh, generator=g).cuda()
    k = torch.randn(B, L, H, dh, generator=g).cuda()
    v = torch.randn(B, L, H, dh, generator=g).cuda()
    dO = (torch.randn(B, L, H, dh, generator=g) * 1e-3).cuda()
    lens = torch.randint(max(1, L // 3), L + 1, (B,), generator=g)
    lens[0] = L
    mask = (torch.arange(L)[None, :] < lens[:, None]).float().cuda()
    q16, k16, v16 = _t16(q, fmt), _t16(k, fmt), _t16(v, fmt)
    dO16 = _t16(dO * 1024.0, fmt)  # loss-scaled gradient in the activations' format
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q16, k16, v16))
    s = torch.einsum("bihc,bjhc->bhij", qf, kf) * (dh ** -0.5)
    s = s.masked_fill(mask[:, None, None, :] == 0, float("-inf"))
    p = torch.softmax(s, dim=-1)
    o = torch.einsum("bhij,bjhc->bihc", p, vf)
    o.backward(dO16.float())
    lse = torch.logsumexp(s, dim=-1).detach().contiguous()
    qkv = torch.cat([q16.reshape(B * L, d), k16.reshape(B * L, d), v16.reshape(B * L, d)], dim=1).contiguous()
    O16 = _t16(o.detach(), fmt).reshape(B * L, d).contiguous()
    delta = torch.zeros(B, H, L, device="cuda")
    dqkv = torch.full((B * L, 3 * d), float("nan"), device="cuda")
    rc = lib.univtg_op_attention_bwd(_lib.ptr(qkv), _lib.ptr(dO16.reshape(B * L, d).contiguous()), _lib.ptr(O16), _lib.ptr(mask),
                                     _lib.ptr(lse), _lib.ptr(delta), _lib.ptr(dqkv), B, L, H, dh, fmt, impl, _lib.stream_ptr())
    _lib.check(rc, "op_attention_bwd")
    torch.cuda.synchronize()
    res = {"ok": True}
    dqkv = dqkv / 1024.0
    for name, ref, got in (("dq", qf.grad / 1024.0, dqkv[:, :d]), ("dk", kf.grad / 1024.0, dqkv[:, d:2 * d]),
                           ("dv", vf.grad / 1024.0, dqkv[:, 2 * d:])):
        ref = ref.reshape(B * L, d)
        rel = ((got - ref).norm() / ref.norm()).item()
        res[name + "_rel"] = rel
        res["ok"] = bool(res["ok"] and rel < 2e-2 and bool(torch.isfinite(got).all()))
    return res


CASES = {
    # name: (fn, args)
    "gemm_k_small_fp16_bn128": (case_gemm, (128, 128, 64, 0, 0, 0, 128, 1, 0, False)),
    "gemm_k_small_fp16_bn256": (case_gemm, (128, 256, 64, 0, 0, 0, 256, 1, 0, False)),
    "gemm_k_k256_fp16": (case_gemm, (128, 256, 256, 0, 0, 0, 256, 1, 0, True)),
    "gemm_k_ragged_fp16": (case_gemm, (300, 384, 200, 0, 0, 0, 128, 1, 1, True)),
    "gemm_k_ragged_bf16_bn256": (case_gemm, (300, 512, 200, 0, 0, 1, 256, 1, 2, True)),
    "gemm_k_big_fp16": (case_gemm, (3424, 1024, 1024, 0, 0, 0, 256, 1, 2, True)),
    "gemm_k_big_multi_wave": (case_gemm, (3424, 3072, 1024, 0, 0, 0, 256, 1, 0, True)),
    "gemm_k_ksplit": (case_gemm, (1024, 1024, 3424, 0, 0, 0, 256, 4, 0, False)),
    "gemm_bn208": (case_gemm, (3424, 1024, 1024, 0, 0, 0, 208, 1, 2, True)),
    "gemm_bn144_ragged": (case_gemm, (300, 400, 200, 0, 0, 0, 144, 1, 1, True)),
    "gemm_bn192_bmn": (case_gemm, (256, 384, 192, 0, 1, 0, 192, 1, 0, True)),
    "tl_ffn1_bn208": (case_gemm_timeline, (3424, 1024, 1024, 2, False, True, 208)),
    "tl_plain16_bn208": (case_gemm_timeline, (3424, 1024, 1024, 0, False, True, 208)),
    "tl_qkv_bn208": (case_gemm_timeline, (3424, 3072, 1024, 0, False, True, 208)),
    "gemmcl_small": (case_gemm, (256, 256, 128, 0, 0, 0, 256, 1, 0, True, True)),
    "gemmcl_ragged": (case_gemm, (300, 384, 200, 0, 0, 0, 128, 1, 1, True, True)),
    "gemmcl_big": (case_gemm, (3424, 1024, 1024, 0, 0, 0, 256, 1, 2, True, True)),
    "gemmcl_big3": (case_gemm, (3424, 3072, 1024, 0, 0, 0, 256, 1, 0, True, True)),
    "gemmcl_amn_ksplit": (case_gemm, (1024, 1024, 3424, 1, 0, 0, 256, 2, 0, False, True)),
    "tlcl_plain16": (case_gemm_timeline, (3424, 1024, 1024, 0, False, True, 256, True)),
    "tlcl_qkv": (case_gemm_timeline, (3424, 3072, 1024, 0, False, True, 256, True)),
    "tl_plain16": (case_gemm_timeline, (3424, 1024, 1024, 0, False, True, 256)),
    "tl_k3072_kmajor": (case_gemm_timeline, (3424, 1024, 3072, 0, True, False, 256, False, 0, 0)),
    "tl_k3072_bmn": (case_gemm_timeline, (3424, 1024, 3072, 0, True, False, 256, False, 0, 1)),
    "tl_k3072_abmn": (case_gemm_timeline, (3424, 1024, 3072, 0, True, False, 256, False, 1, 1)),
    "tl_k3072_amn": (case_gemm_timeline, (3424, 1024, 3072, 0, True, False, 256, False, 1, 0)),
    "tl_nostore": (case_gemm_timeline, (3424, 1024, 1024, 0, False, False, 256)),
    "tl_plain16_m1664": (case_gemm_timeline, (1664, 1024, 1024, 0, False, True, 256)),
    # steady-state mainloop probes: 148 (bn 256) / 296 (bn 128) tiles of 64 k-blocks, i.e. more than one wave on 132 SMs
    "tl_k4096_bn256": (case_gemm_timeline, (9472, 512, 4096, 0, False, True, 256)),
    "tlcl_k4096_bn256": (case_gemm_timeline, (9472, 512, 4096, 0, False, True, 256, True)),
    "tl_k4096_bn128": (case_gemm_timeline, (9472, 512, 4096, 0, False, True, 128)),
    "tlcl_k4096_bn128": (case_gemm_timeline, (9472, 512, 4096, 0, False, True, 128, True)),
    "tl_k4096_bn64": (case_gemm_timeline, (9472, 512, 4096, 0, False, True, 64)),
    "tlcl_k4096_bn64": (case_gemm_timeline, (9472, 512, 4096, 0, False, True, 64, True)),
    "gemm_amn": (case_gemm, (256, 256, 192, 1, 0, 0, 256, 1, 0, True)),
    "gemm_bmn": (case_gemm, (256, 256, 192, 0, 1, 0, 256, 1, 0, True)),
    "gemm_abmn_bn128": (case_gemm, (256, 384, 200, 1, 1, 0, 128, 1, 0, True)),
    "gemm_abmn_big_ksplit": (case_gemm, (1024, 1024, 3424, 1, 1, 0, 256, 4, 0, False)),
    "tl_ffn1": (case_gemm_timeline, (3424, 1024, 1024, 2, False, True, 256)),
    "tl_outproj": (case_gemm_timeline, (3424, 1024, 1024, 0, True, False, 256)),
    "tl_qkv_bn256": (case_gemm_timeline, (3424, 3072, 1024, 0, False, True, 256)),
    "tl_ffn1_bn128": (case_gemm_timeline, (3424, 1024, 1024, 2, False, True, 128)),
    "tl_ffn2_dgrad": (case_group_timeline, ("ffn2_dgrad", 256)),
    "tl_ffn2_dgrad_nomask": (case_group_timeline, ("ffn2_dgrad_nomask", 256)),
    "tl_ffn2_dgrad_nocolsum": (case_group_timeline, ("ffn2_dgrad_nocolsum", 256)),
    "tl_ffn1_dgrad": (case_group_timeline, ("ffn1_dgrad", 256)),
    "tl_out_dgrad": (case_group_timeline, ("out_dgrad", 256)),
    "tl_qkv_dgrad": (case_group_timeline, ("qkv_dgrad", 256)),
    "tl_qkv_wgrad": (case_group_timeline, ("qkv_wgrad", 256)),
    "ln_1024": (case_layernorm, (3424, 1024, 1024, 0)),
    "ln_256_bf16": (case_layernorm, (77, 256, 256, 1)),
    "ln_2818": (case_layernorm, (300, 2818, 2880, 0)),
    "ln_514": (case_layernorm, (33, 514, 576, 0)),
    "attn_simt_dh32": (case_attention, (2, 27, 8, 32, 0, 1)),
    "attn_simt_dh128": (case_attention, (2, 107, 2, 128, 0, 1)),
    "attn_tc_dh128_L107": (case_attention, (3, 107, 4, 128, 0, 0)),
    "attn_tc_dh128_L128": (case_attention, (2, 128, 2, 128, 0, 0)),
    "attn_tc_dh128_L300": (case_attention, (2, 300, 2, 128, 0, 0)),
    "attn_tc_dh64_L182_bf16": (case_attention, (2, 182, 4, 64, 1, 0)),
    "attn_tc_dh128_L1277": (case_attention, (1, 1277, 8, 128, 0, 0)),
    "attnbwd_simt_dh32": (case_attention_bwd, (2, 27, 4, 32, 0, 1)),
    "attnbwd_simt_dh128": (case_attention_bwd, (2, 107, 2, 128, 0, 1)),
    "attnbwd_tc_dh128_L107": (case_attention_bwd, (3, 107, 4, 128, 0, 0)),
    "attnbwd_tc_dh128_L182": (case_attention_bwd, (2, 182, 2, 128, 0, 0)),
    "attnbwd_tc_dh64_L300_bf16": (case_attention_bwd, (2, 300, 4, 64, 1, 0)),
}


def main():
    if len(sys.argv) >= 3 and sys.argv[1] == "--one":
        name = sys.argv[2]
        fn, args = CASES[name]
        print("RESULT " + json.dumps(fn(*args)))
        return
    names = sys.argv[1:] or list(CASES)
    results = {}
    for name in names:
        try:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", name], capture_output=True, text=True,
                               timeout=60)
            line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            if line:
                results[name] = json.loads(line[-1][7:])
            else:
                results[name] = {"ok": False, "rc": p.returncode, "stderr": p.stderr[-600:], "stdout": p.stdout[-300:]}
        except subprocess.TimeoutExpired:
            results[name] = {"ok": False, "timeout": True}
        print(name, json.dumps(results[name]), flush=True)
    os.makedirs(os.path.join(ROOT, "results"), exist_ok=True)
    with open(os.path.join(ROOT, "results", "selftest.json"), "w") as f:
        json.dump(results, f, indent=1)
    n_ok = sum(1 for r in results.values() if r.get("ok"))
    print(f"SELFTEST {n_ok}/{len(results)} ok")


if __name__ == "__main__":
    main()
