"""CPU checks that go with tests/test_attention_bwd_gpu.py.

* The fp64 backward reference (tests/attn_bwd_ref.py), which works from lse and delta, equals torch.autograd in fp64 of masked-softmax
  attention with explicit dropout multipliers, in the formulation of tests/attn_dropout_oracle.py (normaliser = the un-dropped row
  sum), and its bounds have the shape the GPU tests rely on.
* univtg_op_attention_bwd_full and univtg_op_attn_delta refuse, before touching any pointer, what their kernels cannot handle and
  name the argument; training refuses a sequence the SIMT attention backward cannot stage.  The pointers passed here are fake: a
  refusal launches nothing.
"""
import ctypes

import pytest
import torch

from tests.attn_bwd_ref import attn_bwd_reference, delta_reference, fp32_scale, key_mask_gap
from univtg_b200 import _lib


def _autograd(qkv, dO, km, B, L, H, dh, mul):
    """Gradients of O = softmax-with-dropout attention (tests/attn_dropout_oracle.py's core) by torch.autograd, plus O and lse."""
    d = H * dh
    X = qkv.view(B, L, 3, H, dh)
    q, k, v = (X[:, :, i].permute(0, 2, 1, 3).detach().clone().requires_grad_(True) for i in range(3))
    s = (q @ k.transpose(-1, -2)) * fp32_scale(dh)
    s = s.masked_fill(~(km != 0)[:, None, None, :], float("-inf"))
    lse = torch.logsumexp(s, -1).detach()
    s = s - s.amax(dim=-1, keepdim=True)
    p = torch.exp(s)
    denom = p.sum(dim=-1, keepdim=True)
    if mul is not None:
        p = p * mul
    o = (p @ v) / denom
    g = dO.view(B, L, H, dh).permute(0, 2, 1, 3)
    o.backward(g)
    rows = lambda t: t.permute(0, 2, 1, 3).reshape(B * L, d)  # noqa: E731
    return rows(q.grad), rows(k.grad), rows(v.grad), rows(o.detach()), lse


@pytest.mark.parametrize("p", [0.0, 0.25])
@pytest.mark.parametrize("L", [1, 37, 130])
def test_reference_matches_autograd(p, L):
    B, H, dh = 2, 3, 16
    d = H * dh
    g = torch.Generator().manual_seed(10 + L)
    qkv = torch.randn((B * L, 3 * d), generator=g, dtype=torch.float64)
    dO = torch.randn((B * L, d), generator=g, dtype=torch.float64)
    km = key_mask_gap(B, L, None)
    mul = None
    if p > 0:
        mul = (torch.rand((B, H, L, L), generator=g) >= p).double() / (1 - p)
    gq, gk, gv, O, lse = _autograd(qkv, dO, km, B, L, H, dh, mul)
    delta, _ = delta_reference(dO, O, B, L, H, dh)
    for tc in (True, False):
        ref = attn_bwd_reference(qkv, dO, km, lse, delta, B, L, H, dh, 0, tc, mul)
        for n, want in (("dq", gq), ("dk", gk), ("dv", gv)):
            r, S, E = ref[n]
            torch.testing.assert_close(r, want, rtol=1e-12, atol=1e-12, msg=lambda m: f"{n}: {m}")
            assert (S >= r.abs() * (1 - 1e-12)).all() and (E >= 0).all()
            if n != "dq":  # masked keys: exact zeros with a zero bound
                mk = (km == 0).flatten()
                assert (r[mk] == 0).all() and (S[mk] == 0).all() and (E[mk] == 0).all()
    # the SIMT bound (fp32 P and dS) is nowhere looser than the wgmma bound (16-bit P o M and dS), and much tighter for dV, whose
    # propagated error the rounding of P o M dominates (dK and dQ may be dominated by the cancellation in M dP - delta instead)
    e_tc = attn_bwd_reference(qkv, dO, km, lse, delta, B, L, H, dh, 0, True, mul)
    e_simt = attn_bwd_reference(qkv, dO, km, lse, delta, B, L, H, dh, 0, False, mul)
    for n in ("dq", "dk", "dv"):
        assert (e_simt[n][2] <= e_tc[n][2]).all(), n
    assert float(e_simt["dv"][2].sum()) < 0.05 * float(e_tc["dv"][2].sum())


# ---- host checks: every refusal happens before a pointer is read, so fake device addresses are enough ----
def _fake(off=0):
    return 0x7F0000000000 + off


def _bwd_full(**kw):
    lib = _lib.load_library()
    f = _fake
    a = _lib.AttnBwd(f(), f(0x1000), f(0x2000), f(0x3000), f(0x4000), f(0x5000), None, 2, 107, 2, 64, 0, 0)
    rng = _lib.Rng(1, 0.0, 0.0)
    p, layer, use_rng, args = kw.pop("p", 0.0), kw.pop("layer", 0), kw.pop("rng", True), kw.pop("args", True)
    for k, v in kw.items():
        setattr(a, k, v)
    n0 = lib.univtg_launch_count()
    rc = lib.univtg_op_attention_bwd_full(ctypes.byref(a) if args else None, ctypes.byref(rng) if use_rng else None, p, layer, None,
                                          None, None)
    assert rc != 0, kw
    assert lib.univtg_launch_count() == n0
    return _lib.last_error()


def test_attention_bwd_full_refusals():
    assert "null args" in _bwd_full(args=False)
    for n in ("qkv", "dO", "key_mask", "lse", "delta", "dqkv32"):
        assert n in _bwd_full(**{n: None})
    assert "B 0" in _bwd_full(B=0)
    assert "dh 0" in _bwd_full(dh=0)
    assert "fmt 2" in _bwd_full(fmt=2)
    assert "impl 2" in _bwd_full(impl=2)
    assert "dh 64 or 128" in _bwd_full(dh=96)
    assert "dqkv16" in _bwd_full(dqkv16=_fake(0x6000), impl=1)
    assert "dqkv16" in _bwd_full(dqkv16=_fake(0x6000), L=129)
    assert "16-byte" in _bwd_full(qkv=_fake(8))
    assert "16-byte" in _bwd_full(dO=_fake(0x1002))
    assert "8-byte" in _bwd_full(dqkv32=_fake(0x5004))
    assert "p 1" in _bwd_full(p=1.0)
    assert "p -0.1" in _bwd_full(p=-0.1)
    assert "rng" in _bwd_full(p=0.1, rng=False)
    assert "layer" in _bwd_full(p=0.1, layer=-1)
    msg = _bwd_full(impl=1, dh=40, L=7265)
    assert "L 7265" in msg and "7264" in msg and "SIMT" in msg, msg


def _delta(dO=True, fmt_do=0, O=True, fmt_o=0, delta=True, B=2, L=107, H=2, dh=64):
    lib = _lib.load_library()
    n0 = lib.univtg_launch_count()
    rc = lib.univtg_op_attn_delta(_fake() if dO else None, fmt_do, _fake(0x1000) if O else None, fmt_o,
                                  _fake(0x2000) if delta else None, B, L, H, dh, None, None)
    assert rc != 0
    assert lib.univtg_launch_count() == n0
    return _lib.last_error()


def test_attn_delta_refusals():
    assert "dO" in _delta(dO=False)
    assert "O" in _delta(O=False)
    assert "delta" in _delta(delta=False)
    assert "fmt_do 2" in _delta(fmt_do=2)
    assert "fmt_o -1" in _delta(fmt_o=-1)
    assert "B 0" in _delta(B=0)
    assert "L 0" in _delta(L=0)
    assert "H 0" in _delta(H=0)
    assert "dh 0" in _delta(dh=0)


def test_training_refuses_sequence_the_simt_backward_cannot_stage():
    """Head sizes other than 64 and 128 train on the SIMT attention backward, which holds 32 L bytes of shared memory per block:
    on an H100 (227 KB opt-in) L = l_vid + l_txt may be at most 7264.  Longer sequences are refused when the training workspace is
    sized, naming L and the limit, instead of failing in the middle of the first backward."""
    lib = _lib.load_library()
    cfg = _lib.Config(256, 8, 256, 2, 2, 512, 512, 0)  # dh 32
    for Lv, Lt, ok in ((7232, 32, True), (7233, 32, False), (9000, 32, False)):
        got = lib.univtg_train_workspace_bytes(ctypes.byref(cfg), ctypes.byref(_lib.Shape(1, Lv, Lt, 1)))
        assert (got > 0) == ok, (Lv, Lt, got)
        if not ok:
            msg = _lib.last_error()
            assert f"L = l_vid + l_txt = {Lv + Lt}" in msg and "7264" in msg and "SIMT" in msg, msg
    cfg_tc = _lib.Config(512, 8, 256, 2, 2, 512, 512, 0)  # dh 64: the tensor-core backward has no such limit
    assert lib.univtg_train_workspace_bytes(ctypes.byref(cfg_tc), ctypes.byref(_lib.Shape(1, 8000, 32, 1))) > 0
