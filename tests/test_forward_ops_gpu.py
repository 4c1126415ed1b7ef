"""Operator-level fp64 parity of the forward kernels (csrc/rowops.cu, csrc/attention.cu, the head conv GEMMs of csrc/gemm.cu),
each driven on its own through the univtg_op_* entry points, plus forward parity of whole models at hidden widths and feature
dimensions the golden fixtures do not use.

Method and tolerances as in tests/bounds.py: fp64 references from exactly the 16-bit and fp32 inputs the kernel was given, bounds
c(K) 2^-24 S plus half an ulp for 16-bit results, exact zeros where the bound is zero, NaN where nothing may be written.  Where a
kernel's input is a single IEEE fp32 operation of given values (the residual sum x + branch, the text-position sum xt + table) the
reference starts from that fp32 value, which the kernel must reproduce bit for bit where it stores it.  Every case asserts which
instantiation the routing reached; the module prints the coverage at the end (pytest -s).
"""
import ctypes
import math

import pytest
import torch

from tests.attn_bwd_ref import attn_reference, key_mask_gap, val16
from tests.bounds import U, all_nan, cfac, check, report_fixture, ulp16
from tests.test_backward_ops_gpu import DT, P, conv_buf, epilogue, gen, lib, nan, problem, randn, rnd16, run_group, check_rows
from univtg_b200 import _lib

pytestmark = pytest.mark.gpu

_SEEN = {"ln_kernel": set(), "attn_kernel": set()}
_RUNS = {"ln": 0, "attn": 0}  # cases that ran: the coverage test needs the whole module
_report = report_fixture(_SEEN)


def hilo(x32):
    """fp16x3 pair of fp32 values: hi = fp16(x), lo = fp16(x - hi)."""
    hi = x32.half()
    return hi, (x32 - hi.float()).half()


def check16(fam, name, hi, lo, ref, S, K, fmt):
    """A 16-bit result (fmt 0/1) or an fp16x3 pair (lo given): the pair is fp32(v) split into hi and lo, so it may differ from the
    fp32 value by half an ulp of lo."""
    if lo is None:
        check(fam, name, hi, ref, S, K, fmt=fmt)
        return
    b = cfac(K) * U * S.double()
    got = val16(hi, lo)
    check(fam, name, got, ref, S, K, extra=0.5 * ulp16((ref.double() - hi.double()).abs() + b, 0) + U * ref.double().abs())


class Arena:
    """16-bit buffers carved from one allocation whose second half holds their fp16x3 lo planes (`lo` elements after each hi)."""

    def __init__(self, dtype, sizes):
        offs, n = [], 0
        for s in sizes:
            offs.append(n)
            n += (s + 63) // 64 * 64
        self.lo = n
        self.flat = torch.full((2 * n,), float("nan"), dtype=dtype, device="cuda")
        self.offs = offs

    def hi(self, i, shape):
        n = math.prod(shape)
        return self.flat[self.offs[i]:self.offs[i] + n].view(shape)

    def lo_(self, i, shape):
        n = math.prod(shape)
        return self.flat[self.lo + self.offs[i]:self.lo + self.offs[i] + n].view(shape)


def ln_stats(v64, d):
    """fp64 mean / rstd of the rows the kernel normalises and the S terms of their bounds (tests/bounds.py)."""
    mean = v64.mean(1, keepdim=True)
    dx = v64 - mean
    var = (dx * dx).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + 1e-5)
    am = v64.abs().mean(1, keepdim=True)
    # var: c U mean(dx^2) from the squares and their sum, plus the square of the mean's error (sum_i (v_i - mean) = 0, so the
    # mean's error enters the variance only to second order); rstd then carries half of var's relative error plus rsqrtf's.
    R = 0.5 * ((dx * dx).mean(1, keepdim=True) + cfac(d) * U * am * am) / (var + 1e-5) + 1.0
    return mean, rstd, dx, am, R


def layer_norm_ref(v64, gamma, beta):
    """fp64 LayerNorm (eps 1e-5) of the rows v64 with its statistics and the S of its bound; returns (y, S_y, mean, rstd, S_mean,
    S_rstd)."""
    d = v64.shape[1]
    mean, rstd, dx, am, R = ln_stats(v64, d)
    gm, bt = gamma.double(), beta.double()
    y = dx * rstd * gm + bt
    Sy = gm.abs() * rstd * (am + dx.abs() * (1.0 + R)) + bt.abs()
    return y, Sy, mean[:, 0], rstd[:, 0], am[:, 0], (rstd * R)[:, 0]


def sine_ref(vid_mask, dim_t):
    """Sine table [B*Lv, d] in fp64 of the fp32 angle the kernel forms, emulated exactly in fp32 (each step one IEEE operation):
    fl(fl(c / fl(c_last + 1e-6)) * fl32(2 pi)) / dim_t."""
    vm, dt = vid_mask.float().cpu(), dim_t.float().cpu()
    B, Lv = vm.shape
    c = torch.cumsum(vm, 1)  # small integers: exact
    denom = c[:, -1:] + torch.tensor(1e-6, dtype=torch.float32)
    e = (c / denom) * torch.tensor(2 * math.pi, dtype=torch.float32)
    arg = (e[:, :, None] / dt[0::2]).double()  # [B, Lv, d/2]
    return torch.stack([torch.sin(arg), torch.cos(arg)], -1).reshape(B * Lv, dt.numel())


def pool_ref(xt, w, txt_mask):
    """WeightedPool in fp64 from the fp32 inputs: (logits, alpha, pooled) and the S of their bounds.  A masked logit is
    fp32(s - 1e30) = fp32(-1e30), as the kernel forms it."""
    X, W = xt.double(), w.double()
    s = X @ W
    Ss = X.abs() @ W.abs()
    masked = txt_mask.to(X.device) == 0
    lg = torch.where(masked, torch.full_like(s, float(torch.tensor(-1e30, dtype=torch.float32))), s)
    al = torch.softmax(lg, 1)
    # alpha's relative error: the logits' errors (two of them after the max shift) plus expf and the division
    es = torch.where(masked, 0.0, Ss)
    Sal = al * (es + (al * es).sum(1, keepdim=True) + 2.0)
    pooled = torch.einsum("bl,bld->bd", al, X)
    Sp = torch.einsum("bl,bld->bd", al + Sal, X.abs())
    return lg, es, al, Sal, pooled, Sp


def saliency_ref(xv, pooled, vid_mask):
    """cos(x_vid, pooled) (norms clamped at 1e-8) + log(fp32(1e-45)) on padded clips, fp64, and the S of its bound."""
    V, Pd = xv.double(), pooled.double()
    dot = torch.einsum("bld,bd->bl", V, Pd)
    Sdot = torch.einsum("bld,bd->bl", V.abs(), Pd.abs())
    nvp = V.norm(dim=2).clamp_min(1e-8) * Pd.norm(dim=1, keepdim=True).clamp_min(1e-8)
    off = (vid_mask.to(V.device) == 0).double() * math.log(float(torch.tensor(1e-45, dtype=torch.float32)))
    return dot / nvp + off, (Sdot + dot.abs()) / nvp, off


def conv_k3_ref(Xbuf, Wp, rows_out):
    """k=3 Conv1d over the conv-head layout: Y[m] = sum_t Xbuf[m + t] Wp[:, t*C:(t+1)*C]^T (buffer row m + t is logical row
    m + t - 1) for the logical rows m of `rows_out`, fp64, and the same over absolute values."""
    X, C = Xbuf.double(), Xbuf.shape[1]
    acc = sum(X[rows_out + t] @ Wp[:, t * C:(t + 1) * C].double().t() for t in range(3))
    S = sum(X[rows_out + t].abs() @ Wp[:, t * C:(t + 1) * C].double().abs().t() for t in range(3))
    return acc, S


# ================================================= LayerNorm forward =================================================
# role: proj (projector input: shard / fp32 input, K padding, dropout, statistics), ln1 (x + branch -> sum_out, out32, out16),
# ln2 (ln1 + out16p with the sine table on video rows and pos_txt on text rows, outc on the last layer)
def _ln(name, role, d, B, Lv, Lt, kexp, fmt=0, **o):
    return pytest.param(dict(role=role, d=d, B=B, Lv=Lv, Lt=Lt, kexp=kexp, fmt=fmt, **o), id=name)


LN_CASES = [
    _ln("proj_1024_in16_drop", "proj", 1024, 32, 107, 0, 0, in16=0, drop=1),
    _ln("proj_2818_in16_drop", "proj", 2818, 32, 107, 0, 10, in16=0, ld16=2880, drop=1),
    _ln("proj_2050_mul_bf16", "proj", 2050, 1, 7, 0, 10, fmt=1, ld16=2112, mul=1),
    _ln("proj_2818_fp16x3", "proj", 2818, 3, 11, 0, 22, fmt=2, ld16=2880),
    _ln("proj_4098_drop", "proj", 4098, 3, 11, 0, 11, ld16=4160, drop=1),
    _ln("proj_4098_fp16x3", "proj", 4098, 1, 7, 0, 23, fmt=2, ld16=4160),
    _ln("proj_3073_odd", "proj", 3073, 1, 7, 0, 11, ld_in=3080, ld16=3136, mul=1),
    _ln("proj_515_odd_mul", "proj", 515, 3, 11, 0, 6, ld16=576, mul=1),
    _ln("proj_194_in16_bf16_drop", "proj", 194, 3, 11, 0, 6, in16=1, fmt=1, ld16=256, drop=1),
    _ln("proj_768", "proj", 768, 1, 1, 0, 6),
    _ln("ln1_256", "ln1", 256, 3, 8, 3, 2),
    _ln("ln1_512_bf16", "ln1", 512, 1, 4, 3, 1, fmt=1),
    _ln("ln1_1024_one_row", "ln1", 1024, 1, 1, 0, 0),
    _ln("ln1_768", "ln1", 768, 3, 8, 3, 6),
    _ln("ln1_1536", "ln1", 1536, 3, 8, 3, 7),
    _ln("ln1_3072", "ln1", 3072, 1, 4, 3, 7, fmt=1),
    _ln("ln1_1024_fp16x3", "ln1", 1024, 3, 8, 3, 12, fmt=2),
    _ln("ln1_512_fp16x3", "ln1", 512, 1, 4, 3, 13, fmt=2),
    _ln("ln1_256_fp16x3", "ln1", 256, 32, 75, 32, 14, fmt=2),
    _ln("ln1_768_fp16x3", "ln1", 768, 1, 4, 3, 18, fmt=2),
    _ln("ln1_1536_fp16x3", "ln1", 1536, 1, 4, 3, 19, fmt=2),
    _ln("ln2_256_outc", "ln2", 256, 32, 75, 32, 2, outc=1),
    _ln("ln2_768_outc", "ln2", 768, 3, 8, 3, 6, outc=1),
    _ln("ln2_txt_1024", "ln2", 1024, 3, 8, 3, 3, txt=1, outc=1),
    _ln("ln2_txt_512_bf16", "ln2", 512, 1, 4, 3, 4, txt=1, fmt=1),
    _ln("ln2_txt_256", "ln2", 256, 32, 75, 32, 5, txt=1, outc=1),
    _ln("ln2_txt_768", "ln2", 768, 3, 8, 3, 8, txt=1, outc=1),
    _ln("ln2_txt_192_text_row_only", "ln2", 192, 1, 0, 1, 8, txt=1),
    _ln("ln2_txt_1536", "ln2", 1536, 3, 8, 3, 9, txt=1, outc=1),
    _ln("ln2_txt_2816_bf16", "ln2", 2816, 1, 4, 3, 9, txt=1, fmt=1),
    _ln("ln2_txt_1024_fp16x3", "ln2", 1024, 1, 4, 3, 15, txt=1, fmt=2, outc=1),
    _ln("ln2_txt_512_fp16x3", "ln2", 512, 3, 8, 3, 16, txt=1, fmt=2),
    _ln("ln2_txt_256_fp16x3", "ln2", 256, 1, 4, 3, 17, txt=1, fmt=2, outc=1),
    _ln("ln2_txt_768_fp16x3", "ln2", 768, 3, 8, 3, 20, txt=1, fmt=2, outc=1),
    _ln("ln2_txt_1536_fp16x3", "ln2", 1536, 1, 4, 3, 21, txt=1, fmt=2, outc=1),
]


@pytest.mark.parametrize("c", LN_CASES)
def test_layernorm_fwd(c, request):
    cid = request.node.callspec.id
    role, d, B, Lv, Lt, fmt = c["role"], c["d"], c["B"], c["Lv"], c["Lt"], c["fmt"]
    L = Lv + Lt
    split = fmt == 2
    f16 = 0 if split else fmt
    rows = B * Lv if role == "proj" else B * L
    g = gen(1000 + d + rows + 7 * fmt)
    ld_in, ld16 = c.get("ld_in", d), c.get("ld16", d)
    # ---- inputs ----
    x_buf, in16 = None, None
    if "in16" in c:
        in16 = torch.full((rows, ld_in), float("nan"), dtype=DT[c["in16"]], device="cuda")
        in16[:, :d] = rnd16((rows, d), c["in16"], g, 2.0) + 0.5
        if rows > 1:
            in16[0, :d] = 0.375  # constant row: var = 0, rstd = eps^-1/2
        x32 = in16[:, :d].float()
    else:
        x_buf = nan((rows, ld_in))
        x = randn((rows, d), g, 2.0) + 0.5
        x[0] = 0.375
        if rows > 1:
            x[1] = 1000.0 + 1e-2 * randn((d,), g)  # large mean, small variance
        x_buf[:, :d] = x
        x32 = x
    gamma, beta = randn((d,), g, 0.5) + 1.0, randn((d,), g, 0.5)
    outc_rows = B * (Lv + 1) + 2
    sizes = [rows * d, rows * ld16, rows * ld16, outc_rows * d]
    ar = Arena(torch.float16 if split else DT[f16], sizes)
    add16 = add_lo = out16 = out16_lo = out16p = out16p_lo = outc = outc_lo = None
    v32 = x32
    if role != "proj":
        br = randn((rows, d), g)
        br[0] = 0.0
        if rows > 1:
            br[1] = 0.0
        add16 = ar.hi(0, (rows, d))
        if split:
            h, l_ = hilo(br)
            add16.copy_(h)
            add_lo = ar.lo_(0, (rows, d))
            add_lo.copy_(l_)
            v32 = x32 + (h.float() + l_.float())  # the kernel's fp32 sum: x + ld16x3(hi, lo)
        else:
            add16.copy_(br.to(DT[f16]))
            v32 = x32 + add16.float()
    out16 = ar.hi(1, (rows, ld16))
    out16_lo = ar.lo_(1, (rows, ld16)) if split else None
    sum_out = out32 = pos = pos_txt = None
    if role != "proj":
        sum_out, out32 = nan((rows, d)), nan((rows, d))
    if role == "ln2":
        out16p = ar.hi(2, (rows, ld16))
        out16p_lo = ar.lo_(2, (rows, ld16)) if split else None
        pos = randn((B * Lv, d), g)
        if c.get("txt"):
            pos_txt = randn((B * Lt, d), g)
        if c.get("outc"):
            outc = ar.hi(3, (outc_rows, d))
            outc_lo = ar.lo_(3, (outc_rows, d)) if split else None
    mean_out, rstd_out = nan((rows,)), nan((rows,))
    mul32, rng, midx, mul = None, None, -1, None
    if c.get("mul"):
        mul32 = ((torch.rand((rows, d), generator=g) > 0.3).float() / 0.7).cuda()
        mul = mul32
    if c.get("drop"):
        rng, midx = _lib.Rng(77 + d, 0.3, 0.0), 3
        mul = nan((rows, d))
        _lib.check(lib().univtg_dropout_mask(ctypes.byref(rng), midx, rows, d, P(mul), None), "dropout_mask")
    a = _lib.LnFwd()
    a.in_, a.in16, a.in_fmt, a.ld_in = P(x_buf), P(in16), c.get("in16", 0), ld_in
    a.add16, a.ld_add16, a.sum_out = P(add16), d, P(sum_out)
    a.rows, a.d, a.gamma, a.beta, a.eps, a.fmt, a.lo = rows, d, P(gamma), P(beta), 1e-5, fmt, ar.lo if split else 0
    a.L, a.Lv = (L, Lv) if role == "ln2" else (0, 0)
    a.out32, a.out16, a.out16p, a.ld16 = P(out32), P(out16), P(out16p), ld16
    a.pos, a.pos_txt, a.outc, a.mul32 = P(pos), P(pos_txt), P(outc), P(mul32)
    a.mean_out, a.rstd_out = P(mean_out), P(rstd_out)
    used = ctypes.c_int32(-9)
    _lib.check(lib().univtg_op_layernorm_fwd(ctypes.byref(a), ctypes.byref(rng) if rng else None, midx, ctypes.byref(used), None),
               "op_layernorm_fwd")
    torch.cuda.synchronize()
    _SEEN["ln_kernel"].add(used.value)
    _RUNS["ln"] += 1
    assert used.value == c["kexp"], f"routing reached kernel {used.value}, expected {c['kexp']}"

    # ---- fp64 reference from the fp32 rows the kernel normalises ----
    fam = "layernorm_fwd"
    if sum_out is not None:
        assert torch.equal(sum_out, v32), "sum_out must be the fp32 sum x + branch, bit for bit"
    y, Sy, mean, rstd, Sm, Sr = layer_norm_ref(v32.double(), gamma, beta)
    check(fam, f"{cid}/mean_out", mean_out, mean, Sm, d)
    check(fam, f"{cid}/rstd_out", rstd_out, rstd, Sr, d)
    if out32 is not None:
        check(fam, f"{cid}/out32", out32, y, Sy, d)
    m = mul.double() if mul is not None else torch.ones_like(y)
    yd, Syd = y * m, Sy * m.abs()
    check16(fam, f"{cid}/out16", out16[:, :d], None if out16_lo is None else out16_lo[:, :d], yd, Syd, d, f16)
    if ld16 > d:
        assert (out16[:, d:].float() == 0).all(), "out16 padding columns [d, ld16) must be zero"
        if split:
            assert (out16_lo[:, d:].float() == 0).all(), "out16 lo-plane padding columns must be zero"
    if out16p is not None:
        r = torch.arange(rows, device="cuda")
        b_, l_ = r // L, r % L
        vid = l_ < Lv
        add = torch.zeros_like(yd)
        add[vid] = pos.double()[(b_ * Lv + l_)[vid]]
        if pos_txt is not None:
            add[~vid] = pos_txt.double()[(b_ * Lt + l_ - Lv)[~vid]]
        check16(fam, f"{cid}/out16p", out16p, out16p_lo, yd + add, Syd + add.abs(), d, f16)
    if outc is not None:
        r = torch.arange(rows, device="cuda")
        b_, l_ = r // L, r % L
        vid = l_ < Lv
        crow = 1 + b_[vid] * (Lv + 1) + l_[vid]
        assert torch.equal(outc[crow].view(torch.int16), out16[vid, :d].view(torch.int16)), "outc must hold out16's video rows"
        others = torch.ones(outc_rows, dtype=torch.bool, device="cuda")
        others[crow] = False
        all_nan(outc[others], "outc rows 0, separators, tail")
        if split:
            assert torch.equal(outc_lo[crow].view(torch.int16), out16_lo[vid, :d].view(torch.int16)), "outc lo plane"
            all_nan(outc_lo[others], "outc lo plane rows 0, separators, tail")
    if role != "ln2":
        all_nan(ar.hi(2, (rows, ld16)), "out16p (not requested)")


def test_layernorm_fwd_rejects_bad_arguments():
    l_ = lib()
    x = torch.zeros((64, 1024), device="cuda")
    h = torch.zeros((64, 1024), dtype=torch.float16, device="cuda")
    v = torch.zeros(1024, device="cuda")
    n0 = l_.univtg_launch_count()

    def call(**kw):
        a = _lib.LnFwd()
        a.in_, a.ld_in, a.rows, a.d, a.gamma, a.beta, a.eps, a.out16, a.ld16 = P(x), 1024, 64, 1024, P(v), P(v), 1e-5, P(h), 1024
        for k, val in kw.items():
            setattr(a, k, val)
        assert l_.univtg_op_layernorm_fwd(ctypes.byref(a), None, 0, None, None) != 0
        return _lib.last_error()

    assert "gamma" in call(gamma=None)
    assert "ld_add16" in call(add16=P(h), ld_add16=1022)
    assert "16-byte" in call(gamma=P(v) + 4)
    assert "8-byte" in call(out16=P(h) + 2)
    assert "ld16" in call(ld16=1000)
    assert "lo" in call(fmt=2, lo=0)
    assert "L" in call(pos=P(x), out16p=P(h))
    assert l_.univtg_launch_count() == n0


def test_layernorm_rejects_fused_add_beyond_3072():
    """The generic kernel cannot add the residual branch: d > 3072 with add16 is refused by the routing, nothing launches."""
    l_ = lib()
    d, rows = 3136, 4
    x, h = torch.zeros((rows, d), device="cuda"), torch.zeros((rows, d), dtype=torch.float16, device="cuda")
    v = torch.zeros(d, device="cuda")
    a = _lib.LnFwd()
    a.in_, a.ld_in, a.rows, a.d, a.gamma, a.beta, a.eps, a.out16, a.ld16, a.add16, a.ld_add16 = P(x), d, rows, d, P(v), P(v), 1e-5, P(h), d, \
        P(h), d
    n0 = l_.univtg_launch_count()
    assert l_.univtg_op_layernorm_fwd(ctypes.byref(a), None, 0, None, None) != 0 and "3072" in _lib.last_error()
    assert l_.univtg_launch_count() == n0


# ================================================= text positions =================================================
@pytest.mark.parametrize("d", [64, 256, 768, 1024])
@pytest.mark.parametrize("Lt", [1, 7, 32])
@pytest.mark.parametrize("mode", ["none", "mul", "drop", "fp16x3"])
def test_txt_pos_fwd(d, Lt, mode):
    g = gen(2000 + d + Lt)
    B, Lv, max_q_l = 3, 5, 32
    L = Lv + Lt
    fmt = 2 if mode == "fp16x3" else (1 if mode == "mul" else 0)
    xt, table = randn((B * Lt, d), g), randn((max_q_l, d), g, 0.5)
    xt[0], table[0] = 0.125, 0.25  # constant row 0: xt + table = 0.375, var = 0
    gamma, beta = randn((d,), g, 0.5) + 1.0, randn((d,), g, 0.5)
    mul32, rng, midx, mul = None, None, -1, None
    if mode == "mul":
        mul32 = ((torch.rand((B * Lt, d), generator=g) > 0.1).float() / 0.9).cuda()
        mul = mul32
    elif mode == "drop":
        rng, midx = _lib.Rng(31 + d, 0.1, 0.0), 4
        mul = nan((B * Lt, d))
        _lib.check(lib().univtg_dropout_mask(ctypes.byref(rng), midx, B * Lt, d, P(mul), None), "dropout_mask")
    pos, mean_out, rstd_out = nan((B * Lt, d)), nan((B * Lt,)), nan((B * Lt,))
    xp = torch.full((2, B * L, d), float("nan"), dtype=DT[0 if fmt == 2 else fmt], device="cuda")
    a = _lib.TxtPosFwd(P(xt), P(table), P(gamma), P(beta), P(mul32), P(pos), P(mean_out), P(rstd_out), P(xp), B, Lt, L, Lv, d, fmt,
                       B * L * d if fmt == 2 else 0)
    _lib.check(lib().univtg_op_txt_pos(ctypes.byref(a), ctypes.byref(rng) if rng else None, midx, None), "op_txt_pos")
    torch.cuda.synchronize()
    lidx = torch.arange(B * Lt, device="cuda") % Lt
    u32 = xt + table[lidx]  # the kernel's fp32 sum
    y, Sy, mean, rstd, Sm, Sr = layer_norm_ref(u32.double(), gamma, beta)
    tag, fam = f"d{d}_Lt{Lt}_{mode}", "txt_pos_fwd"
    check(fam, f"{tag}/mean", mean_out, mean, Sm, d)
    check(fam, f"{tag}/rstd", rstd_out, rstd, Sr, d)
    m = mul.double() if mul is not None else 1.0
    check(fam, f"{tag}/pos", pos, y * m, Sy * (m.abs() if mul is not None else 1.0), d)
    trow = (torch.arange(B, device="cuda")[:, None] * L + Lv + torch.arange(Lt, device="cuda")[None, :]).flatten()
    s32 = xt + pos  # what the kernel rounds: fp32(xt + pos) with the pos it stored
    if fmt == 2:
        h, l_ = hilo(s32)
        assert torch.equal(xp[0, trow].view(torch.int16), h.view(torch.int16)), "xpos16 text rows (hi)"
        assert torch.equal(xp[1, trow].view(torch.int16), l_.view(torch.int16)), "xpos16 text rows (lo)"
    else:
        assert torch.equal(xp[0, trow].view(torch.int16), s32.to(DT[fmt]).view(torch.int16)), "xpos16 text rows = 16-bit(xt + pos)"
    others = torch.ones(B * L, dtype=torch.bool, device="cuda")
    others[trow] = False
    all_nan(xp[0, others], "xpos16 video rows")
    if fmt != 2:
        all_nan(xp[1], "xpos16 lo plane (not fp16x3)")


# ================================================= sine position table =================================================
@pytest.mark.parametrize("Lv", [1, 75, 256, 257, 1277])
@pytest.mark.parametrize("pattern", ["zero", "prefix", "holey"])
def test_sine_pos(Lv, pattern):
    g = gen(3000 + Lv)
    B, Lt, d = 3, 9, 256
    vm = torch.zeros((B, Lv))
    if pattern == "prefix":
        for b, n in enumerate((Lv, max(1, Lv // 2), max(1, Lv - 3))):
            vm[b, :n] = 1
    elif pattern == "holey":
        vm = (torch.rand((B, Lv), generator=g) > 0.35).float()
        vm[:, 0] = 1
    tm = (torch.rand((B, Lt), generator=g) > 0.3).float()
    dim_t = (10000.0 ** (2 * (torch.arange(d, dtype=torch.float32) // 2) / d)).float()
    n_sites = 4
    rng = _lib.Rng(555 + Lv, 0.0, 0.2)
    pos, km, dp = nan((B * Lv, d)), nan((B, Lv + Lt)), nan((n_sites, B))
    vmc, tmc, dtc = vm.cuda(), tm.cuda(), dim_t.cuda()
    _lib.check(lib().univtg_op_sine_pos(P(vmc), P(tmc), P(dtc), P(pos), P(km), B, Lv, Lt, d, ctypes.byref(rng), n_sites, P(dp), None),
               "op_sine_pos")
    ref_dp = nan((n_sites, B))
    _lib.check(lib().univtg_droppath_scales(ctypes.byref(rng), n_sites, B, P(ref_dp), None), "droppath_scales")
    torch.cuda.synchronize()
    assert torch.equal(km.cpu(), torch.cat([vm, tm], 1)), "key_mask = cat(vid_mask, txt_mask)"
    assert torch.equal(dp, ref_dp), "DropPath scales differ from univtg_droppath_scales"
    ref = sine_ref(vm, dim_t)
    err = (pos.double().cpu() - ref).abs().max().item()
    bound = 2 * 2.0 ** -23
    assert err <= bound, f"sine table: max |got - ref| {err:.3g} > 2 fp32 ulp of 1"
    print(f"  sine_pos/Lv{Lv}_{pattern}: worst |got-ref|/bound = {err / bound:.3f}")


# ================================================= pool + cosine saliency =================================================
@pytest.mark.parametrize("Lt", [1, 32, 33, 77, 300])
@pytest.mark.parametrize("d", [256, 320, 1024])
def test_pool_saliency(Lt, d):
    g = gen(4000 + Lt + d)
    B, Lv = 3, 37
    xt, xv = randn((B, Lt, d), g), randn((B, Lv, d), g)
    w = randn((d,), g, 1.0 / math.sqrt(d))
    tm = torch.ones((B, Lt))
    tm[1, :] = 0  # all-masked text row: uniform alpha
    if Lt > 2:
        tm[2, Lt // 2:] = 0
    if Lt > 32:  # one token beyond the first 32 dominates (logit ~ 120): the softmax max must see every token
        xt[0, Lt - 1] = w * (120.0 / float((w.double() ** 2).sum()))
    vm = torch.ones((B, Lv))
    vm[1, Lv // 3:] = 0  # padded clips: + log(1e-45)
    xv[2, 5] = 0.0  # all-zero clip: the 1e-8 norm clamp
    tmc, vmc = tm.cuda(), vm.cuda()
    pooled, sal, alpha, logits = nan((B, d)), nan((B, Lv)), nan((B, Lt)), nan((B, Lt))
    _lib.check(lib().univtg_op_pool_saliency(P(xt), P(xv), P(tmc), P(vmc), P(w), P(pooled), P(sal), P(alpha), P(logits), B, Lt, Lv, d,
                                             None), "op_pool_saliency")
    torch.cuda.synchronize()
    fam, tag = "pool_saliency", f"Lt{Lt}_d{d}"
    lg, Slg, al, Sal, ref, Sp = pool_ref(xt, w, tmc)
    check(fam, f"{tag}/logits", logits, lg, Slg, d)  # masked logits are exact
    K = d * max(Lt, 2)
    check(fam, f"{tag}/alpha", alpha, al, Sal, K, extra=2.0 ** -149)  # expf underflows to 0 below the smallest denormal
    check(fam, f"{tag}/pooled", pooled, ref, Sp, K)
    ref_s, Ssal, off = saliency_ref(xv, pooled, vmc)  # from the pooled vector the kernel stored (its input)
    check(fam, f"{tag}/saliency", sal, ref_s, Ssal + 3 * off.abs() / cfac(d), d)  # logf(1e-45f) and the sum: within 3 U |offset|


# ================================================= final conv head =================================================
@pytest.mark.parametrize("B,Lv", [(1, 1), (5, 75), (1, 300), (5, 1)])
@pytest.mark.parametrize("d", [256, 320, 1024])
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_conv_head_final(B, Lv, d, fmt):
    g = gen(5000 + B + Lv + d + fmt)
    Mh = B * (Lv + 1)
    split = fmt == 2
    h = []
    for _ in range(2):
        x32 = randn((Mh + 2, d), g).abs()  # ReLU outputs
        x32[0] = 0
        x32[Mh + 1] = 0
        x32[1 + Lv::Lv + 1][:B] = 0
        if split:
            hi, lo = hilo(x32)
            buf = torch.cat([hi.flatten(), lo.flatten()])
        else:
            buf = x32.to(DT[fmt]).flatten()
        h.append(buf)
    w_cls, w_span = randn((3, d), g, 2.0 / math.sqrt(d)), randn((2, 3, d), g, 2.0 / math.sqrt(d))
    b_cls, b_span = randn((1,), g, 0.5), randn((2,), g, 0.5)
    pl, ps = nan((B * Lv,)), nan((B * Lv, 2))
    _lib.check(lib().univtg_op_conv_head_final(P(h[0]), P(h[1]), P(w_cls), P(w_span), P(b_cls), P(b_span), P(pl), P(ps), B, Lv, d, fmt,
                                               None), "op_conv_head_final")
    torch.cuda.synchronize()
    n = (Mh + 2) * d
    Hs = [(val16(t[:n], t[n:]) if split else t.double()).view(Mh + 2, d) for t in h]
    rows = (torch.arange(B, device="cuda")[:, None] * (Lv + 1) + torch.arange(Lv, device="cuda")[None, :] + 1).flatten()
    fam, tag = "conv_head_final", f"B{B}_Lv{Lv}_d{d}_f{fmt}"
    for nm, Hm, w, b, got, sign in (("cls", Hs[0], w_cls, b_cls[0], pl, 1.0), ("span0", Hs[1], w_span[0], b_span[0], ps[:, 0], -1.0),
                                    ("span1", Hs[1], w_span[1], b_span[1], ps[:, 1], 1.0)):
        z = sum(Hm[rows + t - 1] @ w[t].double() for t in range(3)) + b.double()
        Sz = sum(Hm[rows + t - 1].abs() @ w[t].double().abs() for t in range(3)) + b.double().abs()
        sg = torch.sigmoid(z)
        # pre-sigmoid bound through sigma' = sigma (1 - sigma), plus a few ulp for expf and the division
        check(fam, f"{tag}/{nm}", got, sign * sg, sg * (1 - sg) * Sz, 3 * d, extra=8 * U * sg)


# ================================================= forward conv GEMM (conv = 3) =================================================
@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("Lv", [1, 75])
def test_gemm_conv_forward_heads(fmt, Lv):
    """The k=3 head convs as the forward launches them (conv_fwd_problem): conv1 d -> 2d alone, then the conv-2 pair reading the two
    column halves of conv1's output (lda = 2d) in one launch; bias + ReLU, separator rows exact zeros although bias + ReLU would
    make them positive, buffer rows 0 and Mh+1 untouched."""
    g = gen(6000 + Lv + fmt)
    B, d, bn = 3, 256, 128
    Mh = B * (Lv + 1)
    X = conv_buf(B, Lv, d, fmt, g)
    W1 = rnd16((2 * d, 3 * d), fmt, g, 0.05)
    b1 = randn((2 * d,), g).abs() + 1.0  # positive: ReLU(acc + bias) > 0 on the zero separator rows unless zero_sep stores 0
    h1 = nan((Mh + 2, 2 * d), DT[fmt])
    p = problem(a=X, lda=d, b=W1, ldb=3 * d, M=Mh, N=2 * d, K=3 * d, conv=3, bias=b1, act=1, rps_in=Lv + 1, rps_out=Lv + 1, row_off=1,
                zero_sep=1, out16=h1, ld16=2 * d)
    run_group([p], fmt, bn)

    def ref(A, Wp, bias):
        acc, S = conv_k3_ref(A, Wp, torch.arange(Mh, device="cuda"))
        return epilogue(acc, S, fmt, bias=bias, act=1, rps_in=Lv + 1, rps_out=Lv + 1, row_off=1, zero_sep=1)

    e = ref(X, W1, b1)
    check_rows("gemm_conv_fwd", f"conv1_f{fmt}_Lv{Lv}", h1, e, 3 * d, fmt=fmt)
    assert (h1[1 + Lv:Mh + 1:Lv + 1].float() == 0).all(), "conv1 separator rows must be exact zeros"
    # conv-2 pair over the two halves of h1 (rows 0 and Mh+1 of its input must be zero, as univtg_prepare_workspace leaves them)
    h1[0] = 0
    h1[Mh + 1] = 0
    W2 = [rnd16((d, 3 * d), fmt, g, 0.05) for _ in range(2)]
    b2 = [randn((d,), g).abs() + 1.0 for _ in range(2)]
    outs = [nan((Mh + 2, d), DT[fmt]) for _ in range(2)]
    probs = [problem(a=h1[:, s * d:], lda=2 * d, b=W2[s], ldb=3 * d, M=Mh, N=d, K=3 * d, conv=3, bias=b2[s], act=1, rps_in=Lv + 1,
                     rps_out=Lv + 1, row_off=1, zero_sep=1, out16=outs[s], ld16=d) for s in range(2)]
    run_group(probs, fmt, bn)
    for s in range(2):
        e = ref(h1[:, s * d:(s + 1) * d], W2[s], b2[s])
        check_rows("gemm_conv_fwd", f"conv2.{s}_f{fmt}_Lv{Lv}", outs[s], e, 3 * d, fmt=fmt)
        assert (outs[s][1 + Lv:Mh + 1:Lv + 1].float() == 0).all(), "conv2 separator rows must be exact zeros"


# ================================================= attention forward =================================================
def run_attention(B, L, H, dh, fmt, impl, causal=0, km=None, p=0.0, seed=0):
    d = H * dh
    g = gen(seed)
    split = fmt == 2
    x32 = randn((B * L, 3 * d), g)
    if split:
        hi, lo = hilo(x32)
        qkv = torch.cat([hi.flatten(), lo.flatten()])
        out = torch.full((2 * B * L * d,), float("nan"), dtype=torch.float16, device="cuda")
    else:
        qkv = x32.to(DT[fmt]).flatten()
        out = torch.full((B * L * d,), float("nan"), dtype=DT[fmt], device="cuda")
    kmc = (km if km is not None else torch.ones((B, L))).cuda()
    lse = nan((B, H, L))
    rng = _lib.Rng(4242 + L, 0.0, 0.0) if p > 0 else None
    layer = 1
    a = _lib.AttnFwd(P(qkv), P(kmc), P(out), P(lse), B, L, H, dh, fmt, impl, causal)
    used = ctypes.c_int32(-9)
    _lib.check(lib().univtg_op_attention_fwd(ctypes.byref(a), ctypes.byref(rng) if rng else None, p, layer, ctypes.byref(used), None),
               "op_attention_fwd")
    mul = None
    if p > 0:
        mul = nan((B, H, L, L))
        _lib.check(lib().univtg_attention_dropout_mask(ctypes.byref(rng), p, layer, B, H, L, P(mul), None), "attention_dropout_mask")
        mul = mul.double()
    torch.cuda.synchronize()
    _SEEN["attn_kernel"].add(used.value)
    _RUNS["attn"] += 1
    n = B * L * 3 * d
    ref, bo, rlse, Slse = attn_reference(qkv[:n].view(B * L, 3 * d), qkv[n:].view(B * L, 3 * d) if split else None, kmc, B, L, H, dh, fmt,
                                         bool(causal), mul)
    m = B * L * d
    hi_o = out[:m].view(B * L, d)
    lo_o = out[m:].view(B * L, d) if split else None
    return used.value, hi_o, lo_o, ref, bo, lse, rlse, Slse


def check_attention(tag, res, fmt, K):
    used, hi_o, lo_o, ref, bo, lse, rlse, Slse = res
    fam = "attention_fwd"
    # the output bound is absolute (bo); pass it through `extra` with S = 0 so that check() adds the 16-bit rounding on top
    if lo_o is None:
        got = hi_o.double()
        ex = bo + 0.5 * ulp16(ref.abs() + bo, fmt)
    else:
        got = val16(hi_o, lo_o)
        ex = bo + 0.5 * ulp16((ref - hi_o.double()).abs() + bo, 0) + U * ref.abs()
    check(fam, f"{tag}/out", got, ref, torch.zeros_like(ref), K, extra=ex)
    check(fam, f"{tag}/lse", lse, rlse, Slse, K)


ATT_L = [1, 63, 64, 65, 127, 128, 129, 300, 1277]
N_ATTN_CASES = len(ATT_L) * 4 * 3 + 6 * 2 + 2 * 4 * 2


@pytest.mark.parametrize("L", ATT_L)
@pytest.mark.parametrize("dh,impl", [(64, 0), (128, 0), (32, 1), (96, 1)])
@pytest.mark.parametrize("fmt", [0, 1, 2])
def test_attention_fwd(L, dh, impl, fmt):
    B, H = 2, 2
    km = key_mask_gap(B, L, None)
    res = run_attention(B, L, H, dh, fmt, impl, km=km, seed=7000 + L + dh + fmt)
    if impl == 1:
        kexp = 14 if fmt == 2 else 12
    elif fmt == 2:
        kexp = 11 if dh == 128 else 10
    else:
        kexp = (4 if dh == 128 else 0) + 2 * fmt
    assert res[0] == kexp, f"routing reached attention kernel {res[0]}, expected {kexp}"
    check_attention(f"L{L}_dh{dh}_i{impl}_f{fmt}", res, fmt, L * dh)


@pytest.mark.parametrize("dh,impl,fmt,kexp", [(64, 0, 0, 1), (64, 0, 1, 3), (128, 0, 0, 5), (128, 0, 1, 7), (32, 1, 0, 13), (96, 1, 1, 13)])
@pytest.mark.parametrize("L", [65, 300])
def test_attention_fwd_dropout(dh, impl, fmt, kexp, L):
    B, H = 2, 2
    res = run_attention(B, L, H, dh, fmt, impl, km=key_mask_gap(B, L, None), p=0.25, seed=8000 + L + dh + fmt)
    assert res[0] == kexp, f"routing reached attention kernel {res[0]}, expected {kexp}"
    check_attention(f"drop_L{L}_dh{dh}_i{impl}_f{fmt}", res, fmt, L * dh)


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("L", [1, 77, 129, 300])
@pytest.mark.parametrize("pad", [False, True])
def test_attention_fwd_causal(fmt, L, pad):
    B, H = 2, 3
    km = torch.ones((B, L))
    if pad and L > 4:
        km[0, L - 3:] = 0  # padded text tokens at the end of the sequence
        km[1, L // 2:] = 0
    res = run_attention(B, L, H, 64, fmt, 0, causal=1, km=km, seed=9000 + L + fmt)
    assert res[0] == 8 + fmt, f"routing reached attention kernel {res[0]}, expected {8 + fmt}"
    check_attention(f"causal_L{L}_f{fmt}_pad{int(pad)}", res, fmt, L * 64)


def test_forward_ops_cover_every_instantiation():
    """Runs last in the module: together the cases above reached all 24 LayerNorm and all 15 attention instantiations."""
    if _RUNS["ln"] < len(LN_CASES) or _RUNS["attn"] < N_ATTN_CASES:
        pytest.skip("needs every LayerNorm and attention case of the module to have run")
    assert _SEEN["ln_kernel"] == set(range(24)), sorted(set(range(24)) - _SEEN["ln_kernel"])
    assert _SEEN["attn_kernel"] == set(range(15)), sorted(set(range(15)) - _SEEN["attn_kernel"])


# ================================================= whole-model forward at further widths =================================================
WIDTH_CFGS = [
    pytest.param(dict(hidden_dim=768, nheads=12, dim_feedforward=1024, v_feat_dim=194, t_feat_dim=128), True, id="d768_h12_txtpos"),
    pytest.param(dict(hidden_dim=1536, nheads=12, dim_feedforward=1024, v_feat_dim=194, t_feat_dim=128), False, id="d1536_h12"),
    pytest.param(dict(hidden_dim=320, nheads=5, dim_feedforward=512, v_feat_dim=194, t_feat_dim=128), False, id="d320_h5"),
    pytest.param(dict(hidden_dim=256, nheads=2, dim_feedforward=256, v_feat_dim=4098, t_feat_dim=128), False, id="vfeat4098"),
    pytest.param(dict(hidden_dim=256, nheads=2, dim_feedforward=256, v_feat_dim=515, t_feat_dim=128), False, id="vfeat515"),
]


@pytest.mark.parametrize("over,txt_pos", WIDTH_CFGS)
def test_forward_parity_at_further_widths(over, txt_pos):
    """Model.forward (eval) against the fp16-emulating oracle, at the bars of test_forward_matches_fp16_emulating_oracle: checks the
    routing and wiring of the operators at widths the golden fixtures do not use."""
    from oracle import univtg_oracle as O
    from univtg_b200 import build_model, synth

    from tests import txt_pos_oracle as TO

    cfg = dict(synth.CONFIGS["tiny"], **over)
    model, _ = build_model(synth.reference_args(cfg, device="cuda", use_txt_pos=txt_pos))
    sd = synth.make_state_dict(cfg, seed=21)
    model.load_state_dict(sd, strict=True)
    model.to("cuda").eval()
    inp = synth.make_inputs(cfg, seed=23, ragged=True)
    with torch.no_grad():
        out = model(**{k: v.cuda() for k, v in inp.items()})
    torch.cuda.synchronize()
    emu = TO.forward(sd, cfg, **inp, opq=O.round_fp16, use_txt_pos=True) if txt_pos else O.forward(sd, cfg, **inp, opq=O.round_fp16)
    for k in ("pred_logits", "pred_spans", "saliency_scores"):
        torch.testing.assert_close(out[k].double().cpu(), emu[k], rtol=2e-4, atol=5e-5, msg=lambda m: f"{k}: {m}")
    for k in ("vid_mem_proj", "txt_mem_proj"):
        torch.testing.assert_close(out[k].double().cpu(), emu[k], rtol=5e-4, atol=5e-4, msg=lambda m: f"{k}: {m}")
