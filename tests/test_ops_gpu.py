"""Operator-level parity of the CUDA kernels against plain PyTorch fp32 references of the same op (the correctness cases of
tools/gpu_selftest.py, run in-process): wgmma GEMM (K-/MN-major operands, ragged shapes, split-K, 2-CTA clusters, epilogues),
LayerNorm rows, attention forward and backward (wgmma and SIMT paths; L = 107, 128, 182, 300, 1277)."""
import importlib.util
import os

import pytest

pytestmark = pytest.mark.gpu

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_spec = importlib.util.spec_from_file_location("gpu_selftest", os.path.join(_ROOT, "tools", "gpu_selftest.py"))
selftest = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(selftest)

_CORRECTNESS = {selftest.case_gemm, selftest.case_layernorm, selftest.case_attention, selftest.case_attention_bwd}
_CASES = sorted(name for name, (fn, _) in selftest.CASES.items() if fn in _CORRECTNESS)


@pytest.mark.parametrize("name", _CASES)
def test_operator_matches_torch_reference(name):
    fn, args = selftest.CASES[name]
    res = fn(*args)
    assert res.get("ok"), (name, res)


def test_delta_and_column_sum_helpers_match_torch():
    """attn_delta (rowsum(dO * O) per head) for dh in {32, 64, 128} and the 16-bit column sums behind in_proj_bias gradients."""
    import torch

    from univtg_b200 import _lib

    lib = _lib.load_library()
    g = torch.Generator(device="cpu").manual_seed(5)
    for (B, L, H, dh) in ((2, 107, 8, 128), (3, 33, 4, 64), (2, 27, 6, 32), (1, 182, 3, 64)):
        d = H * dh
        q = torch.randn(B, L, H, dh, generator=g).cuda().half()
        k = torch.randn(B, L, H, dh, generator=g).cuda().half()
        v = torch.randn(B, L, H, dh, generator=g).cuda().half()
        dO = torch.randn(B, L, H, dh, generator=g).cuda().half()
        mask = torch.ones(B, L, device="cuda")
        qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
        s = torch.einsum("bihc,bjhc->bhij", qf, kf) * (dh ** -0.5)
        o = torch.einsum("bhij,bjhc->bihc", torch.softmax(s, dim=-1), vf)
        lse = torch.logsumexp(s, dim=-1).detach().contiguous()
        O16 = o.detach().half().reshape(B * L, d).contiguous()
        qkv = torch.cat([q.reshape(B * L, d), k.reshape(B * L, d), v.reshape(B * L, d)], dim=1).contiguous()
        delta = torch.full((B, H, L), float("nan"), device="cuda")
        dqkv = torch.zeros(B * L, 3 * d, device="cuda")
        impl = 0 if dh in (64, 128) else 1
        _lib.check(lib.univtg_op_attention_bwd(_lib.ptr(qkv), _lib.ptr(dO.reshape(B * L, d).contiguous()), _lib.ptr(O16), _lib.ptr(mask),
                                               _lib.ptr(lse), _lib.ptr(delta), _lib.ptr(dqkv), B, L, H, dh, 0, impl, _lib.stream_ptr()),
                   "op_attention_bwd")
        torch.cuda.synchronize()
        ref = (dO.float() * O16.reshape(B, L, H, dh).float()).sum(-1).permute(0, 2, 1)
        torch.testing.assert_close(delta, ref, rtol=1e-4, atol=1e-3)
