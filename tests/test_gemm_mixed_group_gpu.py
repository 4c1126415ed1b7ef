"""A data gradient and split-K weight gradients in one GEMM launch, as the backward runs them, against separate launches.

The merged launch deals its units longest first over the persistent CTAs (the problems are launched in that order, not the
caller's), and each problem keeps its own split-K factor.  Neither may change what a problem computes: the ksplit-1 problem
(K-major A, MN-major B, fp32 output plus a residual) equals its own launch bit for bit; the split-K problems (both operands
MN-major, fp32 partial sums added into a zeroed output) agree with their own launches within one fp32 ulp per partial sum.
"""
import ctypes

import pytest
import torch

from univtg_b200 import _lib

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DT = {0: torch.float16, 1: torch.bfloat16}


def lib():
    return _lib.load_library()


def make(shapes, fmt, seed):
    """shapes: (M, N, K, a_mn, ksplit) -> problems with their operands and a fresh output each time they are launched"""
    g = torch.Generator().manual_seed(seed)
    dt = DT[fmt]
    out = []
    for M, N, K, a_mn, ks in shapes:
        a = torch.randn(M, K, generator=g).to(dt)
        b = (torch.randn(N, K, generator=g) * 0.1).to(dt)
        q = dict(M=M, N=N, K=K, a_mn=a_mn, ks=ks, a=a, b=b,
                 a_buf=(a.t() if a_mn else a).contiguous().cuda(), b_buf=b.t().contiguous().cuda(),  # B always MN-major
                 bias=torch.randn(N, generator=g).cuda(),
                 resid=None if ks > 1 else torch.randn(M, N, generator=g).cuda())
        out.append(q)
    return out


def launch(probs, idx, fmt, bn):
    """launch problems probs[i] for i in idx as one group; returns their fp32 outputs"""
    arr = (_lib.GemmProblem * len(idx))()
    outs = []
    for j, i in enumerate(idx):
        q, p = probs[i], arr[j]
        M, N, K = q["M"], q["N"], q["K"]
        o32 = torch.zeros(M, N, device="cuda") if q["ks"] > 1 else torch.full((M, N), float("nan"), device="cuda")
        p.ksplit, p.a_fmt, p.b_fmt, p.out_fmt, p.alpha, p.colsum_scale = q["ks"], -1, -1, -1, 0.5, 1.0
        p.a, p.lda, p.a_mn = q["a_buf"].data_ptr(), M if q["a_mn"] else K, q["a_mn"]
        p.b, p.ldb, p.b_mn = q["b_buf"].data_ptr(), N, 1
        p.M, p.N, p.K = M, N, K
        p.bias, p.out32, p.ld32 = q["bias"].data_ptr(), o32.data_ptr(), N
        if q["resid"] is not None:
            p.resid, p.ld_resid = q["resid"].data_ptr(), N
        outs.append(o32)
    full = ctypes.c_int32(-1)
    _lib.check(lib().univtg_op_gemm_group(arr, len(idx), fmt, bn, 1, ctypes.byref(full), _lib.stream_ptr()), "op_gemm_group")
    torch.cuda.synchronize()
    return outs, full.value


# (M, N, K, a_mn, ksplit): problem 0 is the data gradient; the split problems have longer units, so the launch runs them first
CASES = {
    "one_split": [(336, 240, 320, 0, 1), (256, 192, 1024, 1, 2)],
    "two_splits": [(336, 240, 320, 0, 1), (256, 192, 1024, 1, 2), (200, 128, 1024, 1, 4)],
}


@pytest.mark.parametrize("fmt", [0, 1])
@pytest.mark.parametrize("case", sorted(CASES))
def test_mixed_group_matches_separate_launches(case, fmt):
    bn = 128
    probs = make(CASES[case], fmt, seed=len(CASES[case]) * 10 + fmt)
    merged, full = launch(probs, list(range(len(probs))), fmt, bn)
    assert full == 1  # split-K problems run the FULL epilogue; the data gradient sharing their launch runs it too
    for i, q in enumerate(probs):
        alone, _ = launch(probs, [i], fmt, bn)
        got, ref = merged[i], alone[0]
        name = f"{case}/fmt{fmt}/problem{i}/ksplit{q['ks']}"
        assert torch.isfinite(got).all() and torch.isfinite(ref).all(), f"{name}: output not fully written"
        if q["ks"] == 1:
            assert torch.equal(got, ref), f"{name}: differs from its own launch"
        else:
            ad, bd = q["a"].double().cuda(), q["b"].double().cuda()
            S = 0.5 * (ad.abs() @ bd.abs().t()) + q["bias"].double().abs()
            err = (got.double() - ref.double()).abs()
            bound = q["ks"] * 2 * U * S
            assert (err <= bound).all(), f"{name}: worst difference / bound {float((err / bound).max()):.3g}"
        # and both are the product: fp64 reference with the epilogue
        ad, bd = q["a"].double().cuda(), q["b"].double().cuda()
        ref64 = 0.5 * (ad @ bd.t() + q["bias"].double()) + (q["resid"].double() if q["resid"] is not None else 0)
        S = 0.5 * (ad.abs() @ bd.abs().t() + q["bias"].double().abs()) + (q["resid"].double().abs() if q["resid"] is not None else 0)
        assert ((got.double() - ref64).abs() <= 64 * U * S + 1e-30).all(), f"{name}: off the fp64 product"
