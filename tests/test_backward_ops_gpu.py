"""Operator-level fp64 parity of the backward kernels (csrc/backward.cu) and of the GEMM epilogue options the backward and the
training forward use (csrc/gemm.cu), each driven on its own through the univtg_op_* entry points.

Method: the 16-bit inputs are drawn once and the reference is computed in fp64 from exactly those values (and from the given
fp32 statistics where a kernel consumes the forward's mean / rstd / alpha).  Outputs are filled with NaN before the call and
accumulated outputs with known non-zero values, so "overwritten", "added to" and "left alone" are each checked.

Tolerances come from the arithmetic (tests/bounds.py): c(K) * 2^-24 * S with S the same formula over absolute values, plus half
an ulp for 16-bit results; zero-bound entries must be exact and regions the kernel must not write must still hold NaN.  The
worst |got - ref| / bound of every case is printed (pytest -s) and summarised per kernel family at the end of the module.
"""
import ctypes
import math

import pytest
import torch

from tests.bounds import all_nan, check, offset_view, report_fixture
from univtg_b200 import _lib

pytestmark = pytest.mark.gpu

DT = {0: torch.float16, 1: torch.bfloat16}
_SEEN = {"lnb_kernel": set(), "vec_ok": set(), "full": set()}
_report = report_fixture(_SEEN)


def lib():
    return _lib.load_library()


def P(t):
    return None if t is None else t.data_ptr()


def gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def randn(shape, g, scale=1.0):
    return (torch.randn(shape, generator=g, dtype=torch.float64) * scale).float().cuda()


def nan(shape, dtype=torch.float32):
    return torch.full(shape, float("nan"), dtype=dtype, device="cuda")


def rnd16(shape, fmt, g, scale=1.0):
    return (torch.randn(shape, generator=g) * scale).to(DT[fmt]).cuda()


def pos16(t):
    return t.view(torch.int16) > 0  # sign bit clear and not +0 (the kernels' test for a positive 16-bit value)


# ================================================= LayerNorm backward =================================================
# (id, d, rows, options, kernel the routing must reach)
LN_CASES = [
    ("warp2_rowscale", 256, 3424, dict(dy32=1, dbr16=1, colsum=1, row_scale=1, L=107, ps=0.5), 1),
    ("warp4_relu_mul", 512, 33, dict(dy32=1, dbr16=1, relu=1, dout_mul=1, colsum=1), 2),
    ("warp8_drop_bf16", 1024, 7, dict(dbr16=1, drop=1, fmt16=1, colsum=1, row_scale=1, L=3), 3),
    ("warp8_one_row", 1024, 1, dict(dy32=1), 3),
    ("vec1_kpad", 384, 3424, dict(dy32=1, dbr16=1, ld_dout=448, ld_y=400, ld16=448, colsum=1, ps=0.25), 4),
    ("vec1_ld16", 256, 7, dict(dbr16=1, ld16=320, colsum=1), 4),
    ("vec2_drop_relu", 768, 33, dict(dbr16=1, dy32=1, drop=1, relu=1, row_scale=1, L=11), 5),
    ("row8_194", 194, 7, dict(dy32=1, dbr16=1, ld_dout=256, ld16=256, colsum=1, relu=1), 6),
    ("row8_514", 514, 1, dict(dbr16=1, dout_mul=1, ld16=520), 6),
    ("row24_1536", 1536, 33, dict(dbr16=1, dy32=1, drop=1, ld16=1600, fmt16=1, colsum=1), 7),
    ("row24_2818", 2818, 3424, dict(dbr16=1, ld_dout=2880, ld16=2880, relu=1, colsum=1, row_scale=1, L=107, ps=0.5), 7),
    ("params_fp32", 256, 1, dict(), 0),
    ("params_y16_fp16_drop", 2818, 3424, dict(y16=0, drop=1, ld_dout=2880), 0),
    ("params_y16_bf16_mul", 1024, 33, dict(y16=1, dout_mul=1), 0),
    ("params_768_ps", 768, 7, dict(ps=0.125), 0),
]


@pytest.mark.parametrize("cid,d,rows,o,kexp", LN_CASES, ids=[c[0] for c in LN_CASES])
def test_layernorm_bwd(cid, d, rows, o, kexp):
    g = gen(100 + d + rows)
    ld_dout, ld_y, ld16 = o.get("ld_dout", d), o.get("ld_y", d), o.get("ld16", d)
    fmt16, ps, L = o.get("fmt16", 0), o.get("ps", 1.0), o.get("L", 0)
    dout_buf = nan((rows, ld_dout))
    dout_buf[:, :d] = randn((rows, d), g)
    y16 = None
    if "y16" in o:
        y16 = torch.full((rows, ld_y), float("nan"), dtype=DT[o["y16"]], device="cuda")
        y16[:, :d] = rnd16((rows, d), o["y16"], g, 2.0) + 0.5
        yv = y16[:, :d].double()
        y_buf = None
    else:
        y_buf = nan((rows, ld_y))
        y = randn((rows, d), g, 2.0) + 0.5
        if o.get("relu"):  # the ReLU mask must treat 0, -0 and negative denormals as "not positive", positive denormals as positive
            y[:, 0::7] = 0.0
            y[:, 1::11] = -0.0
            y[:, 2::13] = 1e-40
            y[:, 3::17] = -1e-40
        y_buf[:, :d] = y
        yv = y.double()
    mean = yv.mean(1).float()
    rstd = (1.0 / torch.sqrt(yv.var(1, unbiased=False) + 1e-5)).float()
    gamma = randn((d,), g, 0.5) + 1.0
    mul, dout_mul, rng, midx = None, None, None, -1
    if o.get("dout_mul"):
        dout_mul = ((torch.rand((rows, d), generator=g) > 0.3).float() / 0.7).cuda()
        mul = dout_mul
    if o.get("drop"):
        rng = _lib.Rng(1234 + d, 0.25, 0.0)
        midx = 5
        mul = nan((rows, d))
        _lib.check(lib().univtg_dropout_mask(ctypes.byref(rng), midx, rows, d, P(mul), None), "dropout_mask")
    nsamp = (rows + max(L, 1) - 1) // max(L, 1)
    row_scale = None
    if o.get("row_scale"):
        row_scale = (torch.rand(nsamp, generator=g) * 1.5 + 0.25).cuda()
        row_scale[min(1, nsamp - 1)] = 0.0
    dy32 = nan((rows, d)) if o.get("dy32") else None
    dbr16 = torch.full((rows, ld16), float("nan"), dtype=DT[fmt16], device="cuda") if o.get("dbr16") else None
    init_g, init_b, init_c = randn((d,), g), randn((d,), g), randn((d,), g)
    dgamma, dbeta = init_g.clone(), init_b.clone()
    colsum = init_c.clone() if o.get("colsum") else None
    a = _lib.LnBwd(P(dout_buf), ld_dout, P(y_buf), ld_y, P(y16), o.get("y16", 0), P(mean), P(rstd), P(gamma), rows, d, P(row_scale), L,
                   1 if o.get("relu") else 0, P(dy32), P(dbr16), ld16, fmt16, P(dgamma), P(dbeta), P(colsum), ps, P(dout_mul))
    used = ctypes.c_int32(-9)
    _lib.check(lib().univtg_op_layernorm_bwd(ctypes.byref(a), ctypes.byref(rng) if rng else None, midx, ctypes.byref(used), None),
               "op_layernorm_bwd")
    torch.cuda.synchronize()
    _SEEN["lnb_kernel"].add(used.value)
    assert used.value == kexp, f"routing reached kernel {used.value}, expected {kexp}"

    # fp64 reference from the given inputs and statistics
    dout = dout_buf[:, :d].double() * (mul.double() if mul is not None else 1.0)
    mu, rs_ = mean.double()[:, None], rstd.double()[:, None]
    xh = (yv - mu) * rs_
    gg = dout * gamma.double()
    dy = rs_ * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    Sdy = rs_ * (gg.abs() + gg.abs().mean(1, keepdim=True) + xh.abs() * (gg * xh).abs().mean(1, keepdim=True))
    if o.get("relu"):
        keep = yv > 0
        dy, Sdy = torch.where(keep, dy, 0.0), torch.where(keep, Sdy, 0.0)
    rsr = row_scale.double()[torch.arange(rows, device="cuda") // L][:, None] if row_scale is not None else torch.ones_like(dy[:, :1])
    br, Sbr = dy * rsr, Sdy * rsr.abs()
    fam = "layernorm_bwd"
    check(fam, f"{cid}/dgamma", dgamma, init_g.double() + ps * (dout * xh).sum(0),
          init_g.double().abs() + abs(ps) * (dout * xh).abs().sum(0), rows)
    check(fam, f"{cid}/dbeta", dbeta, init_b.double() + ps * dout.sum(0), init_b.double().abs() + abs(ps) * dout.abs().sum(0), rows)
    if dy32 is not None:
        check(fam, f"{cid}/dy32", dy32, dy, Sdy, d)
    if dbr16 is not None:
        check(fam, f"{cid}/dbr16", dbr16[:, :d], br, Sbr, d, fmt=fmt16)
        assert (dbr16[:, d:].float() == 0).all(), "dbr16 padding columns [d, ld16) must be zero"
    if colsum is not None:  # column sums of the fp32 values before their 16-bit rounding
        check(fam, f"{cid}/colsum", colsum, init_c.double() + ps * br.sum(0), init_c.double().abs() + abs(ps) * Sbr.sum(0), rows * d)


def test_layernorm_bwd_rejects_bad_arguments():
    l_ = lib()
    x = torch.zeros(64, 256, device="cuda")
    v = torch.zeros(64, device="cuda")
    n0 = l_.univtg_launch_count()
    a = _lib.LnBwd(P(x), 256, P(x), 256, None, 0, P(v), P(v), None, 64, 256, None, 0, 0, P(x), None, 256, 0, None, None, None, 1.0, None)
    assert l_.univtg_op_layernorm_bwd(ctypes.byref(a), None, 0, None, None) != 0 and "gamma" in _lib.last_error()
    a.gamma, a.d = P(v), 4096
    assert l_.univtg_op_layernorm_bwd(ctypes.byref(a), None, 0, None, None) != 0 and "d 4096" in _lib.last_error()
    a.d, a.ld_dout = 256, 200
    assert l_.univtg_op_layernorm_bwd(ctypes.byref(a), None, 0, None, None) != 0 and "ld_dout" in _lib.last_error()
    assert l_.univtg_launch_count() == n0


# ================================================= GEMM epilogue =================================================
def problem(**kw):
    p = _lib.GemmProblem()
    p.ksplit, p.a_fmt, p.b_fmt, p.out_fmt, p.alpha, p.colsum_scale = 1, -1, -1, -1, 1.0, 1.0
    for k, v in kw.items():
        setattr(p, k, v.data_ptr() if torch.is_tensor(v) else v)
    return p


def run_group(probs, fmt, bn, cluster=1):
    arr = (_lib.GemmProblem * len(probs))(*probs)
    full = ctypes.c_int32(-1)
    _lib.check(lib().univtg_op_gemm_group(arr, len(probs), fmt, bn, cluster, ctypes.byref(full), None), "op_gemm_group")
    torch.cuda.synchronize()
    vec = [arr[i].vec_ok for i in range(len(probs))]
    _SEEN["vec_ok"].update(vec)
    _SEEN["full"].add(full.value)
    return full.value, vec


def mm(A, a_mn, B, b_mn):
    """acc[M, N] = sum_k A(m, k) B(n, k) and the same product of absolute values, fp64."""
    Am = A.double().t() if a_mn else A.double()
    Bm = B.double().t() if b_mn else B.double()
    return Am @ Bm.t(), Am.abs() @ Bm.abs().t()


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def dgelu(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def epilogue(acc, S, fmt, bias=None, act=0, alpha=1.0, row_scale=None, rps_in=0, rps_out=0, row_off=0, zero_sep=0, skip_sep=0,
             resid=None, mask=None, mask_mul=0):
    """Reference of epi_step: returns v, S_v [M, N] (fp64), the out row of every m and which rows are stored."""
    M, N = acc.shape
    m = torch.arange(M, device="cuda")
    if rps_in:
        b, l_ = m // rps_in, m % rps_in
        orow, sep = b * rps_out + l_ + row_off, l_ == rps_in - 1
    else:
        b, orow, sep = torch.zeros_like(m), m + row_off, torch.zeros_like(m, dtype=torch.bool)
    pre, Sp = acc.clone(), S.clone()
    if bias is not None:
        pre, Sp = pre + bias.double(), Sp + bias.double().abs()
    dact, Sd = None, None
    if act == 1:
        v, Sv = pre.clamp_min(0.0), Sp
    elif act == 2:  # |GELU'| <= 1.13, |GELU''| <= 0.8; erf itself is evaluated to ~1 ulp
        v, Sv = gelu(pre), 1.13 * Sp + pre.abs()
        dact, Sd = dgelu(pre), 0.8 * Sp + 1.0
    else:
        v, Sv = pre, Sp
    sc = torch.full((M,), float(alpha), dtype=torch.float64, device="cuda")
    if row_scale is not None:
        sc = sc * row_scale.double()[b]
    if zero_sep:
        sc = torch.where(sep, 0.0, sc)
    v, Sv = v * sc[:, None], Sv * sc.abs()[:, None]
    if resid is not None:
        r = resid[orow].double()
        v, Sv = v + r, Sv + r.abs()
    if mask is not None:
        mk = mask[orow]
        if mask_mul:
            mv = mk.double()
            v, Sv = v * mv, Sv * mv.abs()
        else:
            keep = pos16(mk)
            v, Sv = torch.where(keep, v, 0.0), torch.where(keep, Sv, 0.0)
    valid = ~(sep & bool(skip_sep))
    return dict(v=v, S=Sv, orow=orow, valid=valid, dact=dact, Sd=Sd)


def check_rows(fam, name, out, e, K, fmt=None, key="v", Skey="S", init=None):
    """Stored rows equal the reference (init + v when accumulating); every other row of `out` still holds its prefill."""
    rows = e["orow"][e["valid"]]
    ref, S = e[key][e["valid"]], e[Skey][e["valid"]]
    N = ref.shape[1]
    if init is not None:
        ref, S = init[rows, :N].double() + ref, init[rows, :N].double().abs() + S
    check(fam, name, out[rows, :N], ref, S, K, fmt=fmt)
    others = torch.ones(out.shape[0], dtype=torch.bool, device="cuda")
    others[rows] = False
    if init is None:
        all_nan(out[others], f"{name}: rows outside the stored set")
        all_nan(out[:, N:], f"{name}: columns [N, ld)")
    else:
        assert torch.equal(out[others], init[others]), f"{name}: rows outside the stored set changed"


def check_colsum(fam, name, colsum, init, scale, e, K):
    v = torch.where(e["valid"][:, None], e["v"], 0.0)
    S = torch.where(e["valid"][:, None], e["S"], 0.0)
    check(fam, name, colsum, init.double() + scale * v.sum(0), init.double().abs() + abs(scale) * S.sum(0), K * v.shape[0])


def conv_buf(B, Lv, C, fmt, g, ld=None, scale=1.0, zero_sep=True):
    """16-bit activation / gradient in the conv-head layout [B*(Lv+1)+2, C]: rows 0 and Mh+1 zero, separators zero."""
    Mh = B * (Lv + 1)
    x = rnd16((Mh + 2, ld or C), fmt, g, scale)
    x[0] = 0
    x[Mh + 1] = 0
    if zero_sep:
        x[1 + Lv::Lv + 1][:B] = 0
    return x


@pytest.mark.parametrize("fmt", [0, 1])
def test_gemm_ffn2_dgrad_mask_mul_out16_colsum(fmt):
    """d(hpre) = (dF W2) * GELU'(hpre) as a 16-bit operand + linear1.bias column sums.  bf16: the operand / output formats come
    from the per-problem overrides (group format fp16) and the output is a 16- but not 32-byte aligned view (128-bit path)."""
    g = gen(7 + fmt)
    M, d, ff, bn = 300, 256, 1008, 128
    gfmt = fmt if fmt == 0 else 0
    A = rnd16((M, d), fmt, g)
    W2 = rnd16((d, ff), fmt, g, 0.05)
    dg = (torch.rand((M, ff), generator=g) * 1.3 - 0.2).to(DT[gfmt]).cuda()  # GELU' in (-0.2, 1.1), in the group format
    if fmt == 0:
        out, vexp = nan((M, ff), DT[fmt]), 2
    else:
        out, vexp = offset_view(M, ff + 8, DT[fmt], 16), 1
    ci = randn((ff,), g)
    cs = ci.clone()
    p = problem(a=A, lda=d, b=W2, ldb=ff, b_mn=1, M=M, N=ff, K=d, a_fmt=fmt, b_fmt=fmt, out_fmt=fmt, mask16=dg, ld_mask=ff, mask_mul=1,
                out16=out, ld16=out.shape[1], colsum=cs, colsum_scale=0.5)
    full, vec = run_group([p], gfmt, bn)
    assert full == 1 and vec == [vexp]
    acc, S = mm(A, 0, W2, 1)
    e = epilogue(acc, S, fmt, mask=dg, mask_mul=1)
    check_rows("gemm_epilogue", f"ffn2_dgrad{fmt}/out16", out, e, d, fmt=fmt)
    check_colsum("gemm_epilogue", f"ffn2_dgrad{fmt}/colsum", cs, ci, 0.5, e, d)


@pytest.mark.parametrize("fmt", [0, 1])
def test_gemm_conv2_dgrad_rowmap_zero_sep_relu_mask(fmt):
    """Conv layer-2 data gradient of both heads in one launch: conv taps, rows remapped into the conv layout (row_off 1),
    separator rows stored as zeros, ReLU mask of h1, 16-bit output into interleaved column halves, bias column sums."""
    g = gen(11 + fmt)
    B, Lv, d, bn = 3, 75, 256, 192
    Mh = B * (Lv + 1)
    dY = [conv_buf(B, Lv, d, fmt, g) for _ in range(2)]
    Wp = [rnd16((d, 3 * d), fmt, g, 0.05) for _ in range(2)]
    h1 = conv_buf(B, Lv, 2 * d, fmt, g, zero_sep=False)  # positive separator entries: only zero_sep may zero those rows
    h1[1 + Lv::Lv + 1][:B] = h1[1 + Lv::Lv + 1][:B].abs()
    dh1 = nan((Mh + 2, 2 * d), DT[fmt])
    ci = [randn((d,), g) for _ in range(2)]
    cs = [c.clone() for c in ci]
    probs = [problem(a=dY[s], lda=d, b=Wp[s], ldb=3 * d, b_mn=1, M=Mh, N=d, K=d, conv=1, rps_in=Lv + 1, rps_out=Lv + 1, row_off=1,
                     zero_sep=1, mask16=h1[:, s * d:], ld_mask=2 * d, out16=dh1[:, s * d:], ld16=2 * d, out_fmt=fmt, colsum=cs[s],
                     colsum_scale=0.25) for s in range(2)]
    full, vec = run_group(probs, fmt, bn)
    assert full == 1 and vec == [2, 2]
    for s in range(2):
        Y = dY[s].double()
        acc = sum(Y[2 - t:2 - t + Mh] @ Wp[s][:, t * d:(t + 1) * d].double() for t in range(3))  # dX[m] = sum_t dY[m - t + 1] W[:, :, t]
        S = sum(Y[2 - t:2 - t + Mh].abs() @ Wp[s][:, t * d:(t + 1) * d].double().abs() for t in range(3))
        e = epilogue(acc, S, fmt, rps_in=Lv + 1, rps_out=Lv + 1, row_off=1, zero_sep=1, mask=h1[:, s * d:(s + 1) * d])
        sub = dh1[:, s * d:(s + 1) * d]
        check("gemm_epilogue", f"conv2_dgrad{fmt}.{s}/out16", sub[1:Mh + 1], e["v"], e["S"], 3 * d, fmt=fmt)
        assert (sub[1 + Lv:Mh + 1:Lv + 1].float() == 0).all(), "separator rows must be exact zeros"
        all_nan(sub[0], "conv buffer row 0")
        all_nan(sub[Mh + 1], "conv buffer row Mh+1")
        check_colsum("gemm_epilogue", f"conv2_dgrad{fmt}.{s}/colsum", cs[s], ci[s], 0.25, e, 3 * d)


def test_gemm_conv1_dgrad_skip_sep_into_stream_rows():
    """Conv layer-1 data gradient (fused 2d input channels) written into the video rows of the [B*L, d] stream gradient:
    separator rows are not stored, text rows are left alone.  Lean epilogue variant."""
    g = gen(13)
    B, Lv, Lt, d, bn, fmt = 3, 75, 33, 256, 192, 0
    L, Mh = Lv + Lt, B * (Lv + 1)
    dh1 = conv_buf(B, Lv, 2 * d, fmt, g)
    W1p = rnd16((2 * d, 3 * d), fmt, g, 0.05)
    dx = nan((B * L, d))
    p = problem(a=dh1, lda=2 * d, b=W1p, ldb=3 * d, b_mn=1, M=Mh, N=d, K=2 * d, conv=1, rps_in=Lv + 1, rps_out=L, skip_sep=1, out32=dx,
                ld32=d)
    full, vec = run_group([p], fmt, bn)
    assert full == 0 and vec == [2]
    Y = dh1.double()
    acc = sum(Y[2 - t:2 - t + Mh] @ W1p[:, t * d:(t + 1) * d].double() for t in range(3))
    S = sum(Y[2 - t:2 - t + Mh].abs() @ W1p[:, t * d:(t + 1) * d].double().abs() for t in range(3))
    e = epilogue(acc, S, fmt, rps_in=Lv + 1, rps_out=L, skip_sep=1)
    check_rows("gemm_epilogue", "conv1_dgrad/out32", dx, e, 6 * d)


@pytest.mark.parametrize("ksplit", [1, 2, 4])
def test_gemm_conv_wgrad_taps_split_k(ksplit):
    """Conv weight gradient, one problem per tap (dW[n, c, t] = sum_m dY[m, n] X[m + t - 1, c]); split-K adds into planes that
    already hold values, ksplit 1 overwrites NaN planes whose padding columns [N, ld32) must stay NaN."""
    g = gen(17 + ksplit)
    B, Lv, d, bn, fmt = 3, 75, 256, 192, 1
    Mh = B * (Lv + 1)
    dY = conv_buf(B, Lv, d, fmt, g)
    h1 = conv_buf(B, Lv, 2 * d, fmt, g)
    ld32 = d + 16 if ksplit == 1 else d
    planes = nan((3, d, ld32)) if ksplit == 1 else randn((3, d, ld32), g)
    init = None if ksplit == 1 else planes.clone()
    probs = [problem(a=dY, lda=d, a_mn=1, b=h1, ldb=2 * d, b_mn=1, M=d, N=d, K=Mh, conv=2, tap=t, out32=planes[t], ld32=ld32, alpha=0.5,
                     ksplit=ksplit) for t in range(3)]
    full, vec = run_group(probs, fmt, bn)
    assert full == (0 if ksplit == 1 else 1) and vec == [2, 2, 2]
    Y, X = dY.double(), h1[:, :d].double()
    for t in range(3):
        acc, S = Y[1:Mh + 1].t() @ X[t:t + Mh], Y[1:Mh + 1].abs().t() @ X[t:t + Mh].abs()
        e = epilogue(acc, S, fmt, alpha=0.5)
        check_rows("gemm_epilogue", f"conv_wgrad_ks{ksplit}/tap{t}", planes[t], e, Mh, init=None if init is None else init[t])


@pytest.mark.parametrize("fmt", [0, 1])
def test_gemm_qkv_dgrad_resid_and_text_positions(fmt):
    """dx = dy + [dq|dk|dv] W_in, and in the same launch d(pos_t) += [dq|dk] [Wq; Wk] over the text rows (resid == out32, in
    place).  fp16: both problems allow 256-bit accesses (lean variant); bf16: d(pos_t) is a 16- but not 32-byte aligned view,
    so the 128-bit path and the FULL variant run beside a lean-capable problem."""
    g = gen(19 + fmt)
    B, Lv, Lt, d, bn = 3, 75, 33, 256, 192
    M, Mt = B * (Lv + Lt), B * Lt
    dqkv = rnd16((M, 3 * d), fmt, g)
    Win = rnd16((3 * d, d), fmt, g, 0.05)
    dqk = rnd16((Mt, 2 * d), fmt, g)
    dy = randn((M, d), g)
    dx = nan((M, d))
    if fmt == 0:
        dpos = randn((Mt, d), g)
    else:
        dpos = offset_view(Mt, d, torch.float32, 16)
        dpos.copy_(randn((Mt, d), g))
    dpos0 = dpos.clone()
    p0 = problem(a=dqkv, lda=3 * d, b=Win, ldb=d, b_mn=1, M=M, N=d, K=3 * d, resid=dy, ld_resid=d, out32=dx, ld32=d)
    p1 = problem(a=dqk, lda=2 * d, b=Win, ldb=d, b_mn=1, M=Mt, N=d, K=2 * d, resid=dpos, ld_resid=d, out32=dpos, ld32=d)
    full, vec = run_group([p0, p1], fmt, bn)
    assert (full, vec) == ((0, [2, 2]) if fmt == 0 else (1, [2, 1]))
    acc, S = mm(dqkv, 0, Win, 1)
    check_rows("gemm_epilogue", f"qkv_dgrad{fmt}/dx", dx, epilogue(acc, S, fmt, resid=dy), 3 * d)
    acc, S = mm(dqk, 0, Win[:2 * d], 1)
    check("gemm_epilogue", f"qkv_dgrad{fmt}/dpos", dpos, dpos0.double() + acc, dpos0.double().abs() + S, 2 * d)


@pytest.mark.parametrize("fmt,cluster", [(0, 1), (1, 1), (0, 2)])
def test_gemm_projector_forward_rowmap_out32_id_addtab(fmt, cluster):
    """Last projector layer of the training forward: video and text rows scattered into the [B*L, d] stream (rps / row_off),
    fp32 identity-row copies (out32_id), 16-bit x and x + pos (addtab, video only), per-sample row scale with a zero."""
    g = gen(23 + fmt + 3 * cluster)
    B, Lv, Lt, d, K, bn = 3, 75, 33, 256, 384, 96
    L, Mv, Mt = Lv + Lt, B * Lv, B * Lt
    Av, At = rnd16((Mv, K), fmt, g), rnd16((Mt, K), fmt, g)
    Wv, Wt = rnd16((d, K), fmt, g, 0.05), rnd16((d, K), fmt, g, 0.05)
    bv, bt = randn((d,), g), randn((d,), g)
    rs = torch.tensor([1.25, 0.0, 0.5], device="cuda")
    pos = randn((Mv, d), g)
    x32, x16, xp16 = nan((B * L, d)), nan((B * L, d), DT[fmt]), nan((B * L, d), DT[fmt])
    vid, txt = nan((Mv, d)), nan((Mt, d))
    pv = problem(a=Av, lda=K, b=Wv, ldb=K, M=Mv, N=d, K=K, bias=bv, row_scale=rs, rps_in=Lv, rps_out=L, out32=x32, ld32=d, out16=x16,
                 out16p=xp16, ld16=d, addtab=pos, ld_addtab=d, out32_id=vid, ld32_id=d)
    pt = problem(a=At, lda=K, b=Wt, ldb=K, M=Mt, N=d, K=K, bias=bt, row_scale=rs, rps_in=Lt, rps_out=L, row_off=Lv, out32=x32, ld32=d,
                 out16=x16, out16p=xp16, ld16=d, out32_id=txt, ld32_id=d)
    full, vec = run_group([pv, pt], fmt, bn, cluster)
    assert full == 1 and vec == [2, 2]
    fam, tag = "gemm_epilogue", f"proj_fwd{fmt}c{cluster}"
    for nm, A, W, b, rps, off, ident, add in (("vid", Av, Wv, bv, Lv, 0, vid, pos), ("txt", At, Wt, bt, Lt, Lv, txt, None)):
        acc, S = mm(A, 0, W, 0)
        e = epilogue(acc, S, fmt, bias=b, row_scale=rs, rps_in=rps, rps_out=L, row_off=off)
        r = e["orow"]
        check(fam, f"{tag}/{nm}/out32", x32[r], e["v"], e["S"], K)
        check(fam, f"{tag}/{nm}/out16", x16[r], e["v"], e["S"], K, fmt=fmt)
        check(fam, f"{tag}/{nm}/out32_id", ident, e["v"], e["S"], K)
        pv_ = e["v"] + (add.double() if add is not None else 0.0)
        Sp = e["S"] + (add.double().abs() if add is not None else 0.0)
        check(fam, f"{tag}/{nm}/out16p", xp16[r], pv_, Sp, K, fmt=fmt)


@pytest.mark.parametrize("fmt,cluster", [(0, 1), (1, 1), (1, 2)])
def test_gemm_ffn1_forward_dact16_beside_lean_problem(fmt, cluster):
    """FFN1 of the training forward (GELU + its saved 16-bit derivative, FULL variant) grouped with an out-projection problem
    (per-sample row scale, 16-bit branch output) that alone runs the lean variant."""
    g = gen(29 + fmt + 3 * cluster)
    B, L, d, ff, bn = 3, 108, 256, 1008, 96
    M = B * L
    X, Wa = rnd16((M, d), fmt, g), rnd16((ff, d), fmt, g, 0.08)
    b1 = randn((ff,), g, 0.5)
    At, Wo = rnd16((M, d), fmt, g), rnd16((d, d), fmt, g, 0.05)
    bo = randn((d,), g)
    rs = torch.tensor([1.25, 0.0, 2.0], device="cuda")
    h16, dg16, br16 = nan((M, ff), DT[fmt]), nan((M, ff), DT[fmt]), nan((M, d), DT[fmt])
    p0 = problem(a=X, lda=d, b=Wa, ldb=d, M=M, N=ff, K=d, bias=b1, act=2, out16=h16, ld16=ff, dact16=dg16, ld_dact=ff)
    p1 = problem(a=At, lda=d, b=Wo, ldb=d, M=M, N=d, K=d, bias=bo, rps_in=L, rps_out=L, row_scale=rs, out16=br16, ld16=d)
    full, vec = run_group([p0, p1], fmt, bn, cluster)
    assert full == 1 and vec == [2, 2]
    tag = f"ffn1_fwd{fmt}c{cluster}"
    acc, S = mm(X, 0, Wa, 0)
    e = epilogue(acc, S, fmt, bias=b1, act=2)
    check("gemm_epilogue", f"{tag}/h16", h16, e["v"], e["S"], d, fmt=fmt)
    check("gemm_epilogue", f"{tag}/dact16", dg16, e["dact"], e["Sd"], d, fmt=fmt)
    acc, S = mm(At, 0, Wo, 0)
    e1 = epilogue(acc, S, fmt, bias=bo, rps_in=L, rps_out=L, row_scale=rs)
    check("gemm_epilogue", f"{tag}/br16", br16, e1["v"], e1["S"], d, fmt=fmt)
    br16.fill_(float("nan"))
    full, vec = run_group([p1], fmt, bn, cluster)
    assert full == 0 and vec == [2]
    check("gemm_epilogue", f"{tag}/br16_lean", br16, e1["v"], e1["S"], d, fmt=fmt)


@pytest.mark.parametrize("ksplit", [1, 2])
def test_gemm_projector_wgrad_scalar_path(ksplit):
    """Video projector weight gradient dW = dOut^T a with N = 2818 (no vector access possible: scalar epilogue stores).  A bias
    rides along: with split-K only the first split may add it."""
    g = gen(31 + ksplit)
    Mv, d, din, kpad, bn, fmt = 225, 256, 2818, 2880, 128, 1
    dout = rnd16((Mv, d), fmt, g)
    a = torch.full((Mv, kpad), float("nan"), dtype=DT[fmt], device="cuda")  # columns >= din are never read (operand extent N)
    a[:, :din] = rnd16((Mv, din), fmt, g)
    out = nan((d, din)) if ksplit == 1 else randn((d, din), g)
    init = None if ksplit == 1 else out.clone()
    bias = randn((din,), g)
    p = problem(a=dout, lda=d, a_mn=1, b=a, ldb=kpad, b_mn=1, M=d, N=din, K=Mv, bias=bias, out32=out, ld32=din, alpha=0.5, ksplit=ksplit)
    full, vec = run_group([p], fmt, bn)
    assert full == 1 and vec == [0]
    acc, S = mm(dout, 1, a[:, :din], 1)
    check_rows("gemm_epilogue", f"proj_wgrad_ks{ksplit}/out32", out, epilogue(acc, S, fmt, bias=bias, alpha=0.5), Mv, init=init)


def test_gemm_group_rejects_split_epilogues_that_are_not_additive():
    """ksplit > 1 or accumulate with an option that each split would apply to its partial sum is an error naming the option;
    nothing is launched."""
    l_ = lib()
    M, N, K = 128, 128, 256
    A, Bw = torch.zeros((M, K), dtype=torch.float16, device="cuda"), torch.zeros((N, K), dtype=torch.float16, device="cuda")
    o32, o16 = torch.zeros((M, N), device="cuda"), torch.zeros((M, N), dtype=torch.float16, device="cuda")
    n0 = l_.univtg_launch_count()
    for split in (dict(ksplit=2), dict(accumulate=1)):
        for opt, kw in (("act", dict(act=1)), ("resid", dict(resid=o32, ld_resid=N)), ("out16", dict(out16=o16, ld16=N)),
                        ("out16p", dict(out16p=o16, ld16=N)), ("out32_id", dict(out32_id=o32, ld32_id=N)),
                        ("dact16", dict(act=2, dact16=o16, ld_dact=N))):
            p = problem(a=A, lda=K, b=Bw, ldb=K, M=M, N=N, K=K, out32=o32, ld32=N, **split, **kw)
            arr = (_lib.GemmProblem * 1)(p)
            assert l_.univtg_op_gemm_group(arr, 1, 0, 128, 1, None, None) != 0, (split, opt)
            msg = _lib.last_error()
            assert opt in msg and ("ksplit" in msg or "accumulate" in msg), msg
    assert l_.univtg_launch_count() == n0
    # the additive options stay legal with split-K: bias (split 0 only), alpha, mask16, colsum
    p = problem(a=A, lda=K, b=Bw, ldb=K, M=M, N=N, K=K, out32=o32, ld32=N, ksplit=2, bias=o32[0], alpha=0.5)
    run_group([p], 0, 128)


# ================================================= head_final_bwd =================================================
@pytest.mark.parametrize("B,Lv,d,fa,fg", [(1, 1, 256, 0, 0), (5, 31, 512, 0, 1), (5, 75, 2048, 1, 1), (1, 75, 1024, 0, 1)])
def test_head_final_bwd(B, Lv, d, fa, fg):
    g = gen(37 + B + Lv + d)
    Mh = B * (Lv + 1)
    hc, hs = conv_buf(B, Lv, d, fa, g).abs(), conv_buf(B, Lv, d, fa, g)
    hc[:, ::5] = 0  # exact zeros: ReLU' = 0 there
    hc[1:Mh + 1] *= torch.where(torch.rand((Mh, d), generator=g) > 0.5, 1.0, -1.0).to(DT[fa]).cuda()
    w_cls, w_span = randn((3, d), g, 0.1), randn((2, 3, d), g, 0.1)
    pl = (torch.rand((B, Lv), generator=g) * 0.98 + 0.01).cuda()
    ps_ = (torch.rand((B, Lv, 2), generator=g) * 0.98 + 0.01).cuda()
    ps_[..., 0] = -ps_[..., 0]
    gl, gsp = randn((B, Lv), g), randn((B, Lv, 2), g)
    dz = nan((Mh + 2, 4))
    dhc, dhs = nan((Mh + 2, d), DT[fg]), nan((Mh + 2, d), DT[fg])
    i_gwc, i_gbc, i_gws, i_gbs = randn((1, d, 3), g), randn((1,), g), randn((2, d, 3), g), randn((2,), g)
    i_csc, i_css = randn((d,), g), randn((d,), g)
    gwc, gbc, gws, gbs, csc, css = (t.clone() for t in (i_gwc, i_gbc, i_gws, i_gbs, i_csc, i_css))
    insc, pgs = 4.0, 0.25
    a = _lib.HeadFinalBwd(P(gl), P(gsp), P(pl), P(ps_), P(hc), P(hs), P(w_cls), P(w_span), P(dz), P(dhc), P(dhs), P(gwc), P(gbc),
                          P(gws), P(gbs), P(csc), P(css), insc, pgs, B, Lv, d, fa, fg)
    _lib.check(lib().univtg_op_head_final_bwd(ctypes.byref(a), None), "op_head_final_bwd")
    torch.cuda.synchronize()
    fam, tag = "head_final_bwd", f"B{B}_Lv{Lv}_d{d}"
    # dz (logical rows m; separators zero), buffer row m + 1
    ref = torch.zeros((Mh + 2, 4), dtype=torch.float64, device="cuda")
    pc, s0, s1 = pl.double(), -ps_[..., 0].double(), ps_[..., 1].double()
    zz = torch.stack([insc * gl.double() * pc * (1 - pc), -insc * gsp[..., 0].double() * s0 * (1 - s0),
                      insc * gsp[..., 1].double() * s1 * (1 - s1)], -1)  # [B, Lv, 3]
    rows = (torch.arange(B, device="cuda")[:, None] * (Lv + 1) + torch.arange(Lv, device="cuda")[None, :] + 1).flatten()
    ref[rows, :3] = zz.reshape(-1, 3)
    check(fam, f"{tag}/dz", dz, ref, ref.abs(), 4)
    dzl = ref[1:Mh + 1]  # logical rows
    dzb = ref  # buffer rows: dz_logical[j] = dzb[j + 1]
    # dh[m] = relu'(h[m]) * sum_t dz[m - t + 1] w[:, t]  (logical), stored at buffer row m + 1
    for nm, h, dh, ws in (("cls", hc, dhc, [(0, w_cls)]), ("span", hs, dhs, [(1, w_span[0]), (2, w_span[1])])):
        acc = torch.zeros((Mh, d), dtype=torch.float64, device="cuda")
        S = torch.zeros_like(acc)
        for col, w in ws:
            for t in range(3):
                z = dzb[2 - t:2 - t + Mh, col:col + 1]
                acc += z * w[t].double()
                S += z.abs() * w[t].double().abs()
        keep = pos16(h[1:Mh + 1])
        acc, S = torch.where(keep, acc, 0.0), torch.where(keep, S, 0.0)
        check(fam, f"{tag}/dh_{nm}", dh[1:Mh + 1], acc, S, 6, fmt=fg)
        assert (dh[1 + Lv:Mh + 1:Lv + 1].float() == 0).all(), "dh separator rows must be zero"
        all_nan(dh[0], "dh row 0")
        all_nan(dh[Mh + 1], "dh row Mh+1")
    # weight / bias gradients: gw[o, c, t] = sum_m dz_o[m] h[m + t - 1, c]  (h_logical[j] = hbuf[j + 1])
    for nm, h, gw, i_gw, cols in (("cls", hc, gwc, i_gwc, [0]), ("span", hs, gws, i_gws, [1, 2])):
        H = h.double()
        ref = torch.stack([torch.stack([dzl[:, c] @ H[t:t + Mh] for t in range(3)], -1) for c in cols])
        S = torch.stack([torch.stack([dzl[:, c].abs() @ H[t:t + Mh].abs() for t in range(3)], -1) for c in cols])
        check(fam, f"{tag}/gw_{nm}", gw, i_gw.double() + pgs * ref, i_gw.double().abs() + pgs * S, Mh)
    check(fam, f"{tag}/gb_cls", gbc, i_gbc.double() + pgs * dzl[:, 0].sum(), i_gbc.double().abs() + pgs * dzl[:, 0].abs().sum(), Mh)
    check(fam, f"{tag}/gb_span", gbs, i_gbs.double() + pgs * dzl[:, 1:3].sum(0), i_gbs.double().abs() + pgs * dzl[:, 1:3].abs().sum(0), Mh)
    # column sums of the STORED 16-bit dh values
    for nm, dh, cs, ics in (("cls", dhc, csc, i_csc), ("span", dhs, css, i_css)):
        v = dh[1:Mh + 1].double()
        check(fam, f"{tag}/cs_{nm}", cs, ics.double() + pgs * v.sum(0), ics.double().abs() + pgs * v.abs().sum(0), Mh)


# ================================================= colsum16 / cvt16_colsum =================================================
# (rows, text copy (L, Lv) or None)
CS_CASES = [(1, None), (15, None), (17, None), (33, (11, 4)), (3424, (107, 75))]


@pytest.mark.parametrize("rows,txt", CS_CASES)
@pytest.mark.parametrize("fmt", [0, 1])
def test_colsum16(rows, txt, fmt):
    """colsum += scale * column sums of the STORED 16-bit values; optional text-row copy of the first 2d of 3d columns."""
    g = gen(41 + rows + fmt)
    d = 256
    cols, ld = 3 * d, 3 * d + 8
    x = torch.full((rows, ld), float("nan"), dtype=DT[fmt], device="cuda")
    x[:, :cols] = rnd16((rows, cols), fmt, g)
    ci = randn((cols,), g)
    cs = ci.clone()
    L, Lv = txt if txt else (0, 0)
    t16 = nan((rows // L * (L - Lv), 2 * d), DT[fmt]) if txt else None
    _lib.check(lib().univtg_op_colsum16(P(x), ld, rows, cols, fmt, P(cs), 0.5, P(t16), L, Lv, 2 * d, None), "op_colsum16")
    torch.cuda.synchronize()
    v = x[:, :cols].double()
    check("colsum16", f"r{rows}_f{fmt}", cs, ci.double() + 0.5 * v.sum(0), ci.double().abs() + 0.5 * v.abs().sum(0), rows)
    if txt:
        sel = (torch.arange(rows, device="cuda") % L) >= Lv
        assert torch.equal(t16.view(torch.int16), x[sel, :2 * d].view(torch.int16)), "text-row copy differs"


@pytest.mark.parametrize("rows,txt", CS_CASES)
@pytest.mark.parametrize("fmt", [0, 1])
def test_cvt16_colsum(rows, txt, fmt):
    """out16 = RN(in32) and colsum += scale * column sums of the fp32 values (before their rounding); text-row copy."""
    g = gen(43 + rows + fmt)
    d = 256
    cols, ld_in, ld_out = 3 * d, 3 * d + 4, 3 * d + 4
    x = nan((rows, ld_in))
    x[:, :cols] = randn((rows, cols), g)
    out = nan((rows, ld_out), DT[fmt])
    ci = randn((cols,), g)
    cs = ci.clone()
    L, Lv = txt if txt else (0, 0)
    t16 = nan((rows // L * (L - Lv), 2 * d), DT[fmt]) if txt else None
    _lib.check(lib().univtg_op_cvt16_colsum(P(x), ld_in, P(out), ld_out, rows, cols, fmt, P(cs), 0.25, P(t16), L, Lv, 2 * d, None),
               "op_cvt16_colsum")
    torch.cuda.synchronize()
    assert torch.equal(out[:, :cols].view(torch.int16), x[:, :cols].to(DT[fmt]).view(torch.int16)), "16-bit conversion is not RN"
    all_nan(out[:, cols:], "out16 columns [cols, ld_out)")
    v = x[:, :cols].double()
    check("cvt16_colsum", f"r{rows}_f{fmt}", cs, ci.double() + 0.25 * v.sum(0), ci.double().abs() + 0.25 * v.abs().sum(0), rows)
    if txt:
        sel = (torch.arange(rows, device="cuda") % L) >= Lv
        assert torch.equal(t16.view(torch.int16), out[sel, :2 * d].view(torch.int16)), "text-row copy differs"


def test_column_sum_ops_reject_bad_arguments():
    l_ = lib()
    x = torch.zeros((32, 256), dtype=torch.float16, device="cuda")
    x32 = torch.zeros((32, 256), device="cuda")
    cs = torch.zeros(256, device="cuda")
    n0 = l_.univtg_launch_count()
    assert l_.univtg_op_colsum16(P(x), 256, 32, 252, 0, P(cs), 1.0, None, 0, 0, 0, None) != 0 and "multiples of 8" in _lib.last_error()
    assert l_.univtg_op_colsum16(P(x), 256, 32, 256, 0, P(cs), 1.0, P(x), 7, 3, 128, None) != 0 and "rows % L" in _lib.last_error()
    assert l_.univtg_op_cvt16_colsum(x32.data_ptr() + 4, 256, P(x), 256, 8, 128, 0, None, 1.0, None, 0, 0, 0, None) != 0
    assert "16-byte" in _lib.last_error()
    assert l_.univtg_op_stream_gather(P(x32), 8, 4, None, 1.0, P(x), None, 1.0, 2, 6, 256, 0, None) != 0 and "off + Ls" in _lib.last_error()
    assert l_.univtg_launch_count() == n0


# ================================================= stream_gather =================================================
@pytest.mark.parametrize("off_vid,extra_scale,d", [(True, 4.0, 256), (False, None, 256), (False, 1.0, 1024)])
def test_stream_gather(off_vid, extra_scale, d):
    g = gen(47 + d + int(off_vid))
    B, Lv, Lt, fmt = 3, 75, 33, 1
    L = Lv + Lt
    off, Ls = (0, Lv) if off_vid else (Lv, Lt)
    dx = randn((B * L, d), g)
    extra = randn((B * Ls, d), g) if extra_scale is not None else None
    out = nan((B * Ls, d), DT[fmt])
    ci = randn((d,), g)
    cs = ci.clone()
    es = extra_scale if extra_scale is not None else 1.0
    _lib.check(lib().univtg_op_stream_gather(P(dx), L, off, P(extra), es, P(out), P(cs), 0.5, B, Ls, d, fmt, None), "op_stream_gather")
    torch.cuda.synchronize()
    rows = (torch.arange(B, device="cuda")[:, None] * L + off + torch.arange(Ls, device="cuda")[None, :]).flatten()
    v, S = dx[rows].double(), dx[rows].double().abs()
    if extra is not None:
        v, S = v + es * extra.double(), S + abs(es) * extra.double().abs()
    tag = f"off{off}_d{d}_x{extra_scale}"
    check("stream_gather", f"{tag}/out16", out, v, S, 2, fmt=fmt)
    check("stream_gather", f"{tag}/colsum", cs, ci.double() + 0.5 * v.sum(0), ci.double().abs() + 0.5 * S.sum(0), 2 * B * Ls)


# ================================================= pool_bwd =================================================
@pytest.mark.parametrize("Lt,d", [(1, 256), (32, 1024), (300, 256)])
def test_pool_bwd(Lt, d):
    g = gen(53 + Lt + d)
    B, osc = 3, 4.0
    x = randn((B, Lt, d), g)
    w = randn((d,), g, 0.1)
    logits = torch.randn((B, Lt), generator=g, dtype=torch.float64)
    valid = torch.ones((B, Lt), dtype=torch.bool)
    if Lt > 1:
        valid[1, Lt // 2:] = False  # padded text tokens: alpha = 0
        valid[2, -1] = False
    alpha = torch.softmax(logits.masked_fill(~valid, float("-inf")), -1).float().cuda()
    gp = randn((B, d), g)
    dxt = nan((B, Lt, d))
    i_gw = randn((d,), g)
    gw = i_gw.clone()
    _lib.check(lib().univtg_op_pool_bwd(P(x), P(alpha), P(w), P(gp), P(dxt), P(gw), osc, B, Lt, d, None), "op_pool_bwd")
    torch.cuda.synchronize()
    X, al, G, W = x.double(), alpha.double(), gp.double(), w.double()
    da = torch.einsum("bld,bd->bl", X, G)
    Sda = torch.einsum("bld,bd->bl", X.abs(), G.abs())
    dot = (al * da).sum(1, keepdim=True)
    Sdot = (al * Sda).sum(1, keepdim=True)
    dl, Sdl = al * (da - dot), al * (Sda + Sdot)
    ref = (al[..., None] * G[:, None, :] + dl[..., None] * W) * osc
    S = (al[..., None] * G[:, None, :].abs() + Sdl[..., None] * W.abs()) * osc
    check("pool_bwd", f"Lt{Lt}_d{d}/dx", dxt, ref, S, d * Lt)
    check("pool_bwd", f"Lt{Lt}_d{d}/gw", gw, i_gw.double() + torch.einsum("bl,bld->d", dl, X),
          i_gw.double().abs() + torch.einsum("bl,bld->d", Sdl, X.abs()), B * Lt * d)


# ================================================= txt_pos_bwd =================================================
@pytest.mark.parametrize("B,Lt,d,mode", [(1, 32, 256, "none"), (32, 7, 1024, "drop"), (32, 32, 256, "mul"), (1, 5, 1024, "drop")])
def test_txt_pos_bwd(B, Lt, d, mode):
    g = gen(59 + B + Lt + d)
    Lv, max_q_l, ps = 75, 32, 0.5
    L = Lv + Lt
    dpos, xt = randn((B * Lt, d), g), randn((B * Lt, d), g)
    table = randn((max_q_l, d), g, 0.5)
    gamma = randn((d,), g, 0.5) + 1.0
    lidx = torch.arange(B * Lt, device="cuda") % Lt
    u = xt.double() + table.double()[lidx]
    mean = u.mean(1).float()
    rstd = (1.0 / torch.sqrt(u.var(1, unbiased=False) + 1e-12)).float()
    mul32, rng, midx, mul = None, None, -1, None
    if mode == "mul":
        mul32 = ((torch.rand((B * Lt, d), generator=g) > 0.1).float() / 0.9).cuda()
        mul = mul32
    elif mode == "drop":
        rng, midx = _lib.Rng(99 + B, 0.1, 0.0), 4
        mul = nan((B * Lt, d))
        _lib.check(lib().univtg_dropout_mask(ctypes.byref(rng), midx, B * Lt, d, P(mul), None), "dropout_mask")
    dx = nan((B * L, d))
    trow = (torch.arange(B, device="cuda")[:, None] * L + Lv + torch.arange(Lt, device="cuda")[None, :]).flatten()
    dx[trow] = randn((B * Lt, d), g)
    dx0 = dx.clone()
    dtable = nan((max_q_l, d))
    i_g, i_b = randn((d,), g), randn((d,), g)
    dgam, dbet = i_g.clone(), i_b.clone()
    a = _lib.TxtPosBwd(P(dpos), P(xt), P(table), P(gamma), P(mean), P(rstd), P(mul32), P(dx), P(dtable), P(dgam), P(dbet), ps, B, Lt, L,
                       Lv, d)
    _lib.check(lib().univtg_op_txt_pos_bwd(ctypes.byref(a), ctypes.byref(rng) if rng else None, midx, None), "op_txt_pos_bwd")
    torch.cuda.synchronize()
    g0 = dpos.double() * (mul.double() if mul is not None else 1.0)
    mu, rs_ = mean.double()[:, None], rstd.double()[:, None]
    xh = (u - mu) * rs_
    Sxh = (u.abs() + mu.abs()) * rs_
    gg = g0 * gamma.double()
    du = rs_ * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    Sdu = rs_ * (gg.abs() + gg.abs().mean(1, keepdim=True) + Sxh * (gg.abs() * Sxh).mean(1, keepdim=True))
    tag = f"B{B}_Lt{Lt}_d{d}_{mode}"
    check("txt_pos_bwd", f"{tag}/dx", dx[trow], dx0[trow].double() + du, dx0[trow].double().abs() + Sdu, d)
    others = torch.ones(B * L, dtype=torch.bool, device="cuda")
    others[trow] = False
    all_nan(dx[others], "dx video rows")
    check("txt_pos_bwd", f"{tag}/dtable", dtable[:Lt], ps * du.view(B, Lt, d).sum(0), ps * Sdu.view(B, Lt, d).sum(0), B * d)
    all_nan(dtable[Lt:], "dtable rows >= Lt")
    check("txt_pos_bwd", f"{tag}/dgamma", dgam, i_g.double() + ps * (g0 * xh).sum(0), i_g.double().abs() + ps * (g0.abs() * Sxh).sum(0),
          B * Lt)
    check("txt_pos_bwd", f"{tag}/dbeta", dbet, i_b.double() + ps * g0.sum(0), i_b.double().abs() + ps * g0.abs().sum(0), B * Lt)
