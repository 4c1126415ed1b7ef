"""fp64 references of the attention kernels and their error bounds, shared by tests/test_forward_ops_gpu.py (attention forward),
tests/test_attention_bwd_gpu.py (attention backward, attn_delta) and tests/test_attention_bwd_cpu.py.

Backward.  Notation per (b, h): S = Q K^T from the exact 16-bit operands, sigma = fp32(1 / sqrt(dh)), lse and delta as the kernels
are given them (fp32), M the explicit dropout multipliers (univtg_attention_dropout_mask; all 1 without dropout), valid = the key
mask.  Then
    P = exp(sigma S - lse) on valid keys, 0 elsewhere        dP = dO V^T          dS = P o (M o dP - delta) sigma
    dV = (P o M)^T dO        dK = dS^T Q        dQ = dS K        delta = rowsum(dO o O) per head.

Bounds (U = 2^-24, c(K) = tests/bounds.py cfac):
  * score: the fp32 products over dh, c(dh) U |Q||K|^T sigma, plus 4 U (|sigma S| + |lse|) for the rounded sigma log2(e) product,
    lse log2(e) and the subtraction (the wgmma kernel forms exp2f(S sigma log2e - lse log2e), the SIMT kernel expf(S sigma - lse)).
    P then carries the relative error expm1(e_x) + 4 U (exp2f / expf within 2 ulp), and at most 2^-126 absolute where fp32
    underflows (scores far below the row maximum give P = 0).
  * dP: c(dh) U |dO||V|^T.
  * dS: sigma (e_P |M dP - delta| + P M e_dP) + 4 U sigma P (M |dP| + |delta|) for the four fp32 operations; P o M picks up 2 U P M
    for the product with the fp32 multiplier.
  * wgmma only: P o M and dS are rounded to the 16-bit operand format before the dV, dK and dQ products: relative u16 = 2^-11
    (fp16) or 2^-8 (bf16), and for fp16 an absolute 2^-25 (half the smallest subnormal) on valid keys.  The SIMT kernel keeps P and
    dS in fp32, so its bound has no such term.
  * dV, dK, dQ: the propagated elementwise errors above, summed against |dO|, |Q|, |K| (extra), plus c(L) U times the sum of the
    absolute products (S, K = L) for the fp32 accumulation over queries or keys (fp32 atomics across key tiles included).
  * The fused 16-bit output (dqkv16) adds half an ulp of its format (tests/bounds.py check with fmt).
Masked keys have P = dS = 0 exactly, so their dK and dV rows have bound 0 and must be exact zeros.

delta: c(dh) U sum_c |dO||O| per (b, h, i).
"""
import math

import torch

from tests.bounds import U, cfac


def val16(hi, lo=None):
    """fp64 value of a 16-bit operand (hi + lo for an fp16x3 pair)."""
    return hi.double() if lo is None else hi.double() + lo.double()


def fp32_scale(dh):
    """The kernels' softmax scale fp32(1 / sqrt(dh)), as a Python float."""
    return float(torch.tensor(1.0 / math.sqrt(dh), dtype=torch.float32))


def key_mask_gap(B, L, g):
    """The product's key mask cat(vid_mask, txt_mask): valid clips, padded clips, valid text, padded text (per sample)."""
    km = torch.ones((B, L))
    if L < 8:
        return km
    for b in range(B):
        lv = L * 2 // 3
        nv = max(1, lv - 5 * b - 3)
        km[b, nv:lv] = 0
        nt = max(1, (L - lv) - 2 * b)
        km[b, lv + nt:] = 0
    return km


def attn_reference(qkv, lo, km, B, L, H, dh, fmt, causal=False, mul=None):
    """fp64 attention from the exact operands, with the bounds of the output and of lse."""
    d = H * dh
    Qkv = val16(qkv, lo).view(B, L, 3, H, dh)
    q, k, v = (Qkv[:, :, i].permute(0, 2, 1, 3) for i in range(3))  # [B, H, L, dh]
    dev = q.device
    scale = fp32_scale(dh)
    s = torch.einsum("bhid,bhjd->bhij", q, k) * scale
    Ss = torch.einsum("bhid,bhjd->bhij", q.abs(), k.abs()) * scale
    valid = (km.to(dev) != 0)[:, None, None, :].expand(B, H, L, L)
    if causal:
        valid = valid & torch.ones((L, L), dtype=torch.bool, device=dev).tril()
    s = torch.where(valid, s, float("-inf"))
    m = s.max(-1, keepdim=True).values
    p = torch.exp(s - m)
    l = p.sum(-1, keepdim=True)
    lse = (m + torch.log(l))[..., 0]
    pm = p * mul if mul is not None else p
    o = torch.einsum("bhij,bhjd->bhid", pm, v) / l
    split = fmt == 2
    u16 = 2.0 ** -21 if split else (2.0 ** -11 if fmt == 0 else 2.0 ** -8)
    floor = 0.0 if fmt == 1 else 2.0 ** -25
    # score error: fp32 products over dh (+ the lo x lo term fp16x3 drops) and the rounded exponent scale
    es = torch.where(valid, cfac(dh) * U * Ss + 4 * U * s.abs().nan_to_num(0.0, 0.0, 0.0) + (2.0 ** -22 * Ss if split else 0.0), 0.0)
    c = cfac(L)
    pa = pm.abs()
    num = torch.einsum("bhij,bhjd->bhid", (c * U + u16) * pa + 2 * pa * es + floor * valid, v.abs())
    den = ((2 * p * es).sum(-1, keepdim=True) + c * U * l)
    bo = (num + o.abs() * den) / l
    Slse = es.max(-1).values / (cfac(L * dh) * U) + lse.abs() + 1.0
    return o.permute(0, 2, 1, 3).reshape(B * L, d), bo.permute(0, 2, 1, 3).reshape(B * L, d), lse, Slse


def delta_reference(dO, O, B, L, H, dh):
    """delta [B, H, L] = rowsum per head of dO o O in fp64, and the sum of |dO o O| (S of its bound, K = dh)."""
    prod = dO.double().view(B, L, H, dh) * O.double().view(B, L, H, dh)
    return prod.sum(-1).permute(0, 2, 1), prod.abs().sum(-1).permute(0, 2, 1)


def _rows(t, B, L, d):
    """[B, H, L, dh] -> [B*L, H*dh] (the token-major layout of qkv and dqkv)."""
    return t.permute(0, 2, 1, 3).reshape(B * L, d)


def attn_bwd_reference(qkv, dO, km, lse, delta, B, L, H, dh, fmt, tc, mul=None):
    """fp64 gradients of the attention core from the exact operands qkv [B*L, 3d], dO [B*L, d] (any dtype) and the given lse and
    delta [B, H, L].  tc: bound of the wgmma kernel (16-bit P o M and dS), else of the SIMT kernel.  Returns {"dq", "dk", "dv"}:
    (ref, S, extra) as [B*L, d] each, for tests/bounds.py check(..., S, K=L, extra=extra)."""
    d = H * dh
    X = qkv.double().view(B, L, 3, H, dh)
    q, k, v = (X[:, :, i].permute(0, 2, 1, 3) for i in range(3))  # [B, H, L, dh]
    g = dO.double().view(B, L, H, dh).permute(0, 2, 1, 3)
    dev = q.device
    sc = fp32_scale(dh)
    S = q @ k.transpose(-1, -2)
    Ss = q.abs() @ k.abs().transpose(-1, -2)
    valid = (km.to(dev) != 0)[:, None, None, :].expand(B, H, L, L)
    ls = lse.double().to(dev)[..., None]
    dl = delta.double().to(dev)[..., None]
    P = torch.where(valid, torch.exp(sc * S - ls), 0.0)
    dP = g @ v.transpose(-1, -2)
    SdP = g.abs() @ v.abs().transpose(-1, -2)
    M = mul.double().to(dev) if mul is not None else torch.ones_like(P)
    A = M * dP - dl
    dS = P * A * sc
    PM = P * M
    # elementwise errors of P, P o M and dS (module docstring)
    ex = cfac(dh) * U * sc * Ss + 4 * U * ((sc * S).abs() + ls.abs())
    eP = torch.where(valid, P * (torch.expm1(ex) + 4 * U) + 2.0 ** -126, 0.0)
    ePM = M * eP + 2 * U * PM
    edS = sc * (eP * A.abs() + P * M * cfac(dh) * U * SdP) + 4 * U * sc * P * (M * dP.abs() + dl.abs())
    if tc:
        u16 = 2.0 ** -11 if fmt == 0 else 2.0 ** -8
        floor = 2.0 ** -25 if fmt == 0 else 0.0
        # rounding of the fp32 values the kernel holds, which already carry the errors above
        ePM = ePM + torch.where(valid & (M != 0), u16 * (PM + ePM) + floor, 0.0)
        edS = edS + torch.where(valid, u16 * (dS.abs() + edS) + floor, 0.0)
    PMt, dSt = PM.transpose(-1, -2), dS.transpose(-1, -2)
    out = {
        "dv": (PMt @ g, PMt.abs() @ g.abs(), ePM.transpose(-1, -2) @ g.abs()),
        "dk": (dSt @ q, dSt.abs() @ q.abs(), edS.transpose(-1, -2) @ q.abs()),
        "dq": (dS @ k, dS.abs() @ k.abs(), edS @ k.abs()),
    }
    return {n: tuple(_rows(t, B, L, d) for t in ts) for n, ts in out.items()}
