"""CPU checks that go with tests/test_forward_ops_gpu.py: its fp64 references agree with the oracle pinned to the upstream code
(oracle/univtg_oracle.py), and configurations whose first encoder LayerNorm could not run are refused up front."""
import ctypes

import torch

from oracle import univtg_oracle as O
from tests.test_forward_ops_gpu import conv_k3_ref, layer_norm_ref, pool_ref, saliency_ref, sine_ref
from univtg_b200 import _lib


def _g(seed):
    return torch.Generator().manual_seed(seed)


def test_layer_norm_reference_matches_oracle():
    g = _g(1)
    for d in (194, 515, 1024, 4098):
        v = torch.randn((7, d), generator=g, dtype=torch.float64) * 2 + 0.5
        v[0] = 0.375
        v[1] = 1000.0 + 1e-2 * torch.randn(d, generator=g, dtype=torch.float64)
        gm, bt = torch.randn(d, generator=g, dtype=torch.float64) + 1, torch.randn(d, generator=g, dtype=torch.float64)
        y, Sy, mean, rstd, _, _ = layer_norm_ref(v, gm, bt)
        torch.testing.assert_close(y, O.layer_norm(v, gm, bt), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(rstd, 1.0 / torch.sqrt(v.var(1, unbiased=False) + 1e-5), rtol=1e-10, atol=0)
        assert float(rstd[0]) == 1e-5 ** -0.5 and (Sy >= y.abs() - 1e-9).all()


def test_sine_reference_matches_oracle():
    g = _g(2)
    d = 256
    dim_t = (10000.0 ** (2 * (torch.arange(d, dtype=torch.float32) // 2) / d)).float()
    for Lv in (1, 75, 257):
        vm = (torch.rand((3, Lv), generator=g) > 0.3).float()
        vm[0] = 0
        ref = sine_ref(vm, dim_t).view(3, Lv, d)
        # the oracle forms the angle in fp64; the test's reference rounds it to fp32 as the kernel does
        torch.testing.assert_close(ref, O.sine_position(vm, d, torch.float64), rtol=0, atol=2e-6)


def test_pool_and_saliency_references_match_oracle():
    g = _g(3)
    B, Lt, Lv, d = 3, 33, 11, 320
    xt = torch.randn((B, Lt, d), generator=g)
    xv = torch.randn((B, Lv, d), generator=g)
    xv[2, 5] = 0
    w = torch.randn(d, generator=g) / d ** 0.5
    tm = torch.ones((B, Lt))
    tm[1] = 0
    tm[2, Lt // 2:] = 0
    vm = torch.ones((B, Lv))
    vm[1, 4:] = 0
    _, _, al, _, pooled, _ = pool_ref(xt, w, tm)
    op, oal = O.weighted_pool(xt.double(), tm.double(), w.double())
    torch.testing.assert_close(al, oal, rtol=1e-12, atol=1e-300)
    torch.testing.assert_close(pooled, op, rtol=1e-12, atol=1e-12)
    assert torch.equal(al[1], torch.full((Lt,), 1.0 / Lt, dtype=torch.float64)), "all-masked text row: uniform alpha"
    sal, _, off = saliency_ref(xv, pooled, vm)
    osal = O.cosine(xv.double(), pooled[:, None, :]) + torch.log(vm.double() + 2.0 ** -149)
    torch.testing.assert_close(sal, osal, rtol=1e-12, atol=1e-12)
    assert abs(float(off[1, 5]) + 103.27892990343184) < 1e-12 and float(sal[2, 5]) == 0.0


def test_conv_reference_matches_oracle():
    g = _g(4)
    B, Lv, C, N = 3, 7, 64, 24
    x = torch.randn((B, Lv, C), generator=g, dtype=torch.float64)
    w = torch.randn((N, C, 3), generator=g, dtype=torch.float64)
    b = torch.zeros(N, dtype=torch.float64)
    Mh = B * (Lv + 1)
    buf = torch.zeros((Mh + 2, C), dtype=torch.float64)  # conv-head layout: row 1 + b*(Lv+1) + l, zero rows between samples
    rows = (torch.arange(B)[:, None] * (Lv + 1) + torch.arange(Lv)[None, :]).flatten()
    buf[rows + 1] = x.reshape(-1, C)
    w2 = w.permute(0, 2, 1).reshape(N, 3 * C)  # w2[n, t*C + c] = w[n, c, t], the packed layout
    acc, _ = conv_k3_ref(buf, w2, rows)
    torch.testing.assert_close(acc.view(B, Lv, N), O.conv1d_k3(x, w, b, O._ident, O._ident), rtol=1e-12, atol=1e-12)


def test_hidden_dim_beyond_layernorm_limit_is_rejected():
    """hidden_dim > 3072 would pass every other check and fail at the first encoder LayerNorm (the fused residual add stops at
    3072): the config is refused with a message naming the limit."""
    lib = _lib.load_library()
    for d, ok in ((3072, True), (3136, False), (4096, False)):
        cfg = _lib.Config(d, 8, 1024, 2, 2, 2818, 512, 0)
        got = lib.univtg_packed_bytes(ctypes.byref(cfg))
        assert (got > 0) == ok, (d, got)
        if not ok:
            msg = _lib.last_error()
            assert "hidden_dim" in msg and "3072" in msg and "LayerNorm" in msg, msg
