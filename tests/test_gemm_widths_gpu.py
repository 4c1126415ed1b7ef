"""Every tile width the GEMM accepts, against an fp64 reference.

The kernel compiles one mainloop, accumulator array and epilogue read-out per tile width and picks it at launch, so each width
is its own code path.  This module runs all of them: multiples of 16 in [32, 256] with a K-major B, multiples of 64 with an
MN-major B, both A layouts, fp16 and bf16, the lean and the FULL epilogue variant (asserted through univtg_op_gemm_group's
report), single CTAs and 2-CTA clusters (multiples of 32, K-major B), and the fp16x3 split variant at a few widths.

M is ragged (not a multiple of the 128-row tile, an odd tile count for the cluster pairs) and N = 2 bn - 16 leaves a partial
last column tile.  Outputs are pre-filled with NaN; columns [N, ld) must still hold NaN.  Bound: |got - ref| <= c 2^-24 S with
S = |A| |B|^T + |bias| and c = 4 (ceil(log2 K) + 1), plus half an ulp for 16-bit results.
"""
import ctypes
import itertools
import math

import pytest
import torch

from univtg_b200 import _lib

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DT = {0: torch.float16, 1: torch.bfloat16}
M, K = 333, 320
WIDTHS = list(range(32, 257, 16))
SPLIT_WIDTHS = [48, 176, 240, 256]


def lib():
    return _lib.load_library()


def cfac(k):
    return 4 * (math.ceil(math.log2(k)) + 1)


def ulp16(x, fmt):
    p, emin = (10, -14) if fmt == 0 else (7, -126)
    _, e = torch.frexp(x)
    return torch.pow(2.0, torch.clamp(e.to(torch.float64) - 1, min=emin) - p)


def check(name, got, ref, S, fmt=None):
    got, ref = got.double(), ref.double()
    assert torch.isfinite(got).all(), f"{name}: {int((~torch.isfinite(got)).sum())} entries not written"
    b = cfac(K) * U * S
    if fmt is not None:
        b = b + 0.5 * ulp16(ref.abs() + b, fmt)
    err = (got - ref).abs()
    assert (err <= b).all(), f"{name}: {int((err > b).sum())} entries out of bound, worst ratio {float((err / b).max()):.3g}"


def run_case(bn, fmt, a_mn, b_mn, full, cluster, seed):
    g = torch.Generator().manual_seed(seed)
    N = 2 * bn - 16
    dt = DT[fmt]
    a = (torch.randn(M, K, generator=g)).to(dt)
    b = (torch.randn(N, K, generator=g) * 0.1).to(dt)
    lda = (M + 7) // 8 * 8
    a_buf = torch.zeros(K, lda, dtype=dt) if a_mn else a
    if a_mn:
        a_buf[:, :M] = a.t()
    b_buf = b.t().contiguous() if b_mn else b
    a_buf, b_buf = a_buf.cuda(), b_buf.cuda()
    bias = torch.randn(N, generator=g).cuda()
    # the FULL variant is reached through a 16- but not 32-byte aligned out32 pitch (128-bit rather than 256-bit stores)
    ld32 = N + 4 if full else N
    out32 = torch.full((M, ld32), float("nan"), device="cuda")
    out16 = torch.full((M, N), float("nan"), dtype=dt, device="cuda")
    p = _lib.GemmProblem()
    p.ksplit, p.a_fmt, p.b_fmt, p.out_fmt, p.alpha, p.colsum_scale = 1, -1, -1, -1, 1.0, 1.0
    p.a, p.lda, p.a_mn = a_buf.data_ptr(), lda if a_mn else K, a_mn
    p.b, p.ldb, p.b_mn = b_buf.data_ptr(), N if b_mn else K, b_mn
    p.M, p.N, p.K = M, N, K
    p.bias, p.out32, p.ld32, p.out16, p.ld16 = bias.data_ptr(), out32.data_ptr(), ld32, out16.data_ptr(), N
    arr = (_lib.GemmProblem * 1)(p)
    used = ctypes.c_int32(-1)
    _lib.check(lib().univtg_op_gemm_group(arr, 1, fmt, bn, cluster, ctypes.byref(used), None), "op_gemm_group")
    torch.cuda.synchronize()
    name = f"bn{bn}/fmt{fmt}/a_mn{a_mn}/b_mn{b_mn}/{'full' if full else 'lean'}/cl{cluster}"
    assert used.value == int(full), f"{name}: ran the {'FULL' if used.value else 'lean'} variant"
    ad, bd = a.double().cuda(), b.double().cuda()
    ref = ad @ bd.t() + bias.double()
    S = ad.abs() @ bd.abs().t() + bias.double().abs()
    check(name + "/out32", out32[:, :N], ref, S)
    check(name + "/out16", out16, ref, S, fmt=fmt)
    if ld32 > N:
        assert torch.isnan(out32[:, N:]).all(), f"{name}: columns [N, ld32) were written"


@pytest.mark.parametrize("bn", WIDTHS)
def test_gemm_width(bn):
    n = 0
    for fmt in (0, 1):
        for b_mn in ((0, 1) if bn % 64 == 0 else (0,)):
            for a_mn in (0, 1):
                for full in (False, True):
                    for cluster in ((1, 2) if bn % 32 == 0 and not b_mn else (1,)):
                        run_case(bn, fmt, a_mn, b_mn, full, cluster, seed=1000 * bn + n)
                        n += 1


def pair(x):
    hi = x.half()
    lo = (x - hi.float()).half()
    return torch.stack([hi, lo])


@pytest.mark.parametrize("bn", SPLIT_WIDTHS)
def test_gemm_width_fp16x3(bn):
    g = torch.Generator().manual_seed(bn)
    N = 2 * bn - 16
    A, B = pair(torch.randn(M, K, generator=g)).cuda(), pair(torch.randn(N, K, generator=g) * 0.05).cuda()
    bias = torch.randn(N, generator=g).cuda()
    out32 = torch.full((M, N), float("nan"), device="cuda")
    out16 = torch.full((2, M, N), float("nan"), device="cuda", dtype=torch.float16)
    _lib.check(lib().univtg_op_gemm(_lib.ptr(A), _lib.ptr(B), M, N, K, 0, 0, 2, bn, 1, _lib.ptr(bias), 0, 1.0, _lib.ptr(out32),
                                    _lib.ptr(out16), _lib.stream_ptr()), "op_gemm fp16x3")
    torch.cuda.synchronize()
    av, bv = A[0].double() + A[1].double(), B[0].double() + B[1].double()
    ref = av @ bv.t() + bias.double()
    bound = (3 * 2.0 ** -22 + cfac(K) * U) * (av.abs() @ bv.abs().t()) + U * bias.double().abs()
    err = (out32.double() - ref).abs()
    assert torch.isfinite(out32).all() and (err <= bound).all(), f"bn {bn}: worst err / bound {float((err / bound).max()):.3g}"
    assert not torch.isnan(out16).any()
    assert torch.equal(out16[0], out32.half())


OP_CASES = [c for c in itertools.product((0, 1), (0, 1), (0, 1), (1, 2), (1, 2)) if not (c[4] == 2 and c[2])]  # clusters: K-major B


@pytest.mark.parametrize("fmt,a_mn,b_mn,ksplit,cluster", OP_CASES)
def test_op_gemm_matches_group(fmt, a_mn, b_mn, ksplit, cluster):
    """univtg_op_gemm (cluster 1) and univtg_op_gemm_cluster (cluster 2) run the kernel with the same parameters as
    univtg_op_gemm_group on the equivalent problem, so their outputs agree bit for bit.  With ksplit 2 the two partial sums are
    added with atomics: within one fp32 ulp of the magnitude.  An MN-major operand's pitch is its M / N: both multiples of 8."""
    bn, Mo = 192, 336
    N = 2 * bn - 16
    g = torch.Generator().manual_seed(16 * fmt + 8 * a_mn + 4 * b_mn + 2 * ksplit + cluster)
    dt = DT[fmt]
    a = torch.randn(Mo, K, generator=g).to(dt)
    b = (torch.randn(N, K, generator=g) * 0.1).to(dt)
    a_buf = (a.t() if a_mn else a).contiguous().cuda()
    b_buf = (b.t() if b_mn else b).contiguous().cuda()
    bias = torch.randn(N, generator=g).cuda()
    alpha = 0.5

    def outputs():  # split-K accumulates into a zeroed out32 and cannot store out16
        if ksplit > 1:
            return torch.zeros(Mo, N, device="cuda"), None
        return torch.full((Mo, N), float("nan"), device="cuda"), torch.full((Mo, N), float("nan"), dtype=dt, device="cuda")

    o32, o16 = outputs()
    fn = lib().univtg_op_gemm_cluster if cluster == 2 else lib().univtg_op_gemm
    _lib.check(fn(_lib.ptr(a_buf), _lib.ptr(b_buf), Mo, N, K, a_mn, b_mn, fmt, bn, ksplit, _lib.ptr(bias), 0, alpha, _lib.ptr(o32),
                  _lib.ptr(o16), _lib.stream_ptr()), "op_gemm")
    r32, r16 = outputs()
    p = _lib.GemmProblem()
    p.ksplit, p.a_fmt, p.b_fmt, p.out_fmt, p.alpha, p.colsum_scale = ksplit, -1, -1, -1, alpha, 1.0
    p.a, p.lda, p.a_mn = a_buf.data_ptr(), Mo if a_mn else K, a_mn
    p.b, p.ldb, p.b_mn = b_buf.data_ptr(), N if b_mn else K, b_mn
    p.M, p.N, p.K = Mo, N, K
    p.bias, p.out32, p.ld32, p.out16, p.ld16 = bias.data_ptr(), r32.data_ptr(), N, r16.data_ptr() if r16 is not None else None, N
    _lib.check(lib().univtg_op_gemm_group((_lib.GemmProblem * 1)(p), 1, fmt, bn, cluster, None, _lib.stream_ptr()), "op_gemm_group")
    torch.cuda.synchronize()
    name = f"fmt{fmt}/a_mn{a_mn}/b_mn{b_mn}/ksplit{ksplit}/cl{cluster}"
    assert torch.isfinite(o32).all() and torch.isfinite(r32).all(), f"{name}: out32 not fully written"
    if ksplit == 1:
        assert torch.equal(o32, r32), f"{name}: out32 differs from univtg_op_gemm_group"
        assert torch.isfinite(o16).all() and torch.equal(o16, r16), f"{name}: out16 differs from univtg_op_gemm_group"
    else:
        ad, bd = a.double().cuda(), b.double().cuda()
        S = alpha * (ad.abs() @ bd.abs().t()) + bias.double().abs()
        err = (o32.double() - r32.double()).abs()
        assert (err <= 2 * U * S).all(), f"{name}: worst difference / (2^-23 S) {float((err / (2 * U * S)).max()):.3g}"
