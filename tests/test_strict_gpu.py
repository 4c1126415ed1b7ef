"""operand_format="fp16x3": the strict inference mode (fp16 hi / lo operand pairs, three MMA products per product) against the fp32
reference goldens, the fp64 oracle and the fp16x3-emulating oracle, its kernel paths one by one, its behaviour, its training
refusals, and its single operators against fp64."""
import ctypes
import math

import pytest
import torch

from oracle import univtg_oracle as O
from tests import txt_pos_oracle as TO
from tests.helpers import GOLDEN_CASES, OUT_KEYS, load_golden
from tests.strict_oracle import round_fp16x3
from tests.test_strict_cpu import HEAD_TOL, PROJ_TOL, check_against_reference
from univtg_b200 import _lib, build_model, synth

pytestmark = pytest.mark.gpu

# The projector outputs sum K = 2818 (x 3 products) terms in fp32 on the tensor cores.  On cfg2_full the worst vid_mem_proj element
# is 1.1e-5 from the reference (value -0.0123); the reference there is within 1.8e-6 of fp64 and the fp64-accumulating fp16x3
# oracle within 6.1e-6, so the rest is fp32 accumulation - far inside the GEMM round-off bound (3 * 2^-22 + 52 * 2^-24) * sum|a||b|
# (~8e-5 here).  The GPU bar for those two outputs is therefore atol 2e-5; every other bar is the CPU test's.
PROJ_TOL_GPU = dict(PROJ_TOL, atol=2e-5)


def _model(cfg, sd, fmt="fp16x3", **over):
    model, _ = build_model(synth.reference_args(cfg, device="cuda:0", operand_format=fmt, **over))
    model.load_state_dict(sd, strict=True)
    return model.to("cuda:0").eval()


def _run(model, inp):
    with torch.no_grad():
        out = model(**{k: v.cuda() for k, v in inp.items()})
    torch.cuda.synchronize()
    return {k: v for k, v in out.items() if torch.is_tensor(v) and k != "src_vid_mask"}


def _close(out, ref, name, head=HEAD_TOL, proj=PROJ_TOL_GPU):
    for k in OUT_KEYS:
        tol = proj if k.endswith("mem_proj") else head
        torch.testing.assert_close(out[k].double().cpu(), ref[k].double(), **tol, msg=lambda m: f"{name}/{k}: {m}")



@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_strict_matches_reference_golden(name):
    cfg, sd, inp, _, z = load_golden(name)
    check_against_reference(_run(_model(cfg, sd), inp), z, name, proj=PROJ_TOL_GPU)


@pytest.mark.parametrize("name", ["tiny_ragged", "cfg1_demo", "cfg2_b4_ragged"])
def test_strict_error_is_twenty_times_smaller_than_fp16(name):
    cfg, sd, inp, _, _ = load_golden(name)
    exact = O.forward(sd, cfg, **inp)
    strict = _run(_model(cfg, sd), inp)
    half = _run(_model(cfg, sd, fmt="fp16"), inp)
    for k in OUT_KEYS:
        e3 = (strict[k].double().cpu() - exact[k]).abs().max().item()
        e1 = (half[k].double().cpu() - exact[k]).abs().max().item()
        assert e3 <= e1 / 20, f"{name}/{k}: fp16x3 error {e3:.3g} vs fp16 error {e1:.3g}"


@pytest.mark.parametrize("name", ["tiny_ragged", "cfg1_demo", "cfg2_b4_ragged"])
def test_strict_matches_fp16x3_emulating_oracle(name):
    """Only fp32 accumulation order, the dropped lo * lo terms and fp32 (not fp64) splitting differ: the golden bars hold."""
    cfg, sd, inp, _, _ = load_golden(name)
    _close(_run(_model(cfg, sd), inp), O.forward(sd, cfg, **inp, opq=round_fp16x3), name)


TINY = synth.CONFIGS["tiny"]
PATHS = {
    "dh128_one_key_tile": (TINY, dict(batch=4), {}),
    "dh64": (dict(TINY, nheads=4), dict(batch=4), {}),
    "simt_dh32": (synth.CONFIGS["cfg1"], dict(batch=3), {}),
    "multi_tile_cfg5": (synth.CONFIGS["cfg5"], dict(batch=1, ragged=True), {}),
    "txt_pos": (TINY, dict(batch=4), dict(use_txt_pos=True)),
    "fp16_features": (TINY, dict(batch=4), {}),
}


@pytest.mark.parametrize("path", list(PATHS))
def test_strict_kernel_paths_match_emulating_oracle(path):
    cfg, inp_kw, over = PATHS[path]
    sd = synth.make_state_dict(cfg, seed=71)
    inp = synth.make_inputs(cfg, seed=72, ragged=inp_kw.get("ragged", True), batch=inp_kw["batch"])
    if path == "fp16_features":
        inp = {k: (v.half() if k in ("src_txt", "src_vid") else v) for k, v in inp.items()}
    model = _model(cfg, sd, **over)
    out = _run(model, inp)
    raw = {k: v.double() for k, v in inp.items()}
    if over.get("use_txt_pos"):
        ref = TO.forward(sd, cfg, **raw, opq=round_fp16x3, use_txt_pos=True)
    else:
        ref = O.forward(sd, cfg, **raw, opq=round_fp16x3)
    _close(out, ref, path)


def test_graph_replay_and_repeat_are_bit_identical_and_launches_match():
    cfg = TINY
    sd = synth.make_state_dict(cfg, seed=81)
    inp = {k: v.cuda() for k, v in synth.make_inputs(cfg, seed=82, ragged=True, batch=4).items()}
    model = _model(cfg, sd)
    a, b = _run(model, inp), _run(model, inp)
    model.use_cuda_graphs = True
    g1, g2 = _run(model, inp), _run(model, inp)
    model.use_cuda_graphs = False
    for k in OUT_KEYS:
        assert torch.equal(a[k], b[k]), k
        assert torch.equal(a[k], g1[k]) and torch.equal(a[k], g2[k]), k
    half = _model(cfg, sd, fmt="fp16")
    assert model.num_forward_launches(4, 24, 6) == half.num_forward_launches(4, 24, 6)
    tp = _model(cfg, sd, use_txt_pos=True)
    tp16 = _model(cfg, sd, fmt="fp16", use_txt_pos=True)
    assert tp.num_forward_launches(4, 24, 6) == tp16.num_forward_launches(4, 24, 6)


def test_sample_alone_matches_sample_in_batch():
    cfg = synth.CONFIGS["cfg2"]
    sd = synth.make_state_dict(cfg, seed=91)
    inp = synth.make_inputs(cfg, seed=92, ragged=True, batch=6)
    model = _model(cfg, sd)
    full = _run(model, inp)
    one = _run(model, {k: v[2:3] for k, v in inp.items()})
    for k in OUT_KEYS:
        torch.testing.assert_close(one[k], full[k][2:3], rtol=1e-6, atol=1e-6, msg=lambda m: f"{k}: {m}")


# ------------------------------------------------------------------------------------------------------------------ refusals
def test_training_is_refused_without_launching():
    lib = _lib.load_library()
    cfg = TINY
    sd = synth.make_state_dict(cfg, seed=3)
    model = _model(cfg, sd)
    inp = {k: v.cuda() for k, v in synth.make_inputs(cfg, seed=4, batch=2).items()}
    _run(model, inp)  # plans, packed weights
    n0 = lib.univtg_launch_count()
    model.train()
    with pytest.raises(NotImplementedError, match="inference mode"):
        model(**inp)
    model.eval()
    from univtg_b200.optim import FlatAdamW

    with pytest.raises(NotImplementedError, match="inference mode"):
        FlatAdamW(model)
    assert lib.univtg_launch_count() == n0

    c = model._cfgs[2]
    shp = _lib.Shape(2, inp["src_vid"].shape[1], inp["src_txt"].shape[1], 1)
    assert lib.univtg_train_workspace_bytes(ctypes.byref(c), ctypes.byref(shp)) == 0
    assert "fp16x3" in _lib.last_error()
    plan = model._get_plan(2, inp["src_vid"].shape[1], inp["src_txt"].shape[1], False)
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    outs = [torch.empty(1 << 16, device="cuda") for _ in range(5)]
    p = [_lib.ptr(t) for t in outs]
    rc = lib.univtg_forward_train(plan.handle, _lib.ptr(buf), _lib.ptr(inp["src_txt"]), _lib.ptr(inp["src_txt_mask"]), _lib.ptr(inp["src_vid"]),
                                  _lib.ptr(inp["src_vid_mask"]), None, None, None, *p, _lib.stream_ptr())
    assert rc != 0 and "fp16x3" in _lib.last_error()
    grads = (ctypes.c_void_p * 1)(_lib.ptr(buf))
    rc = lib.univtg_backward(plan.handle, _lib.ptr(buf), _lib.ptr(inp["src_txt"]), _lib.ptr(inp["src_vid"]), None, None, None, None, None,
                             None, None, 1.0, grads, 1, _lib.stream_ptr())
    assert rc != 0 and "fp16x3" in _lib.last_error()
    f = torch.zeros(64, device="cuda")
    rc = lib.univtg_adamw_step(_lib.ptr(f), _lib.ptr(f), _lib.ptr(f), _lib.ptr(f), 64, 1e-4, 0.9, 0.999, 1e-8, 0.0, 1, 0.0, 0, _lib.ptr(f),
                               ctypes.byref(c), _lib.ptr(model._packed[2]), _lib.stream_ptr())
    assert rc != 0 and "fp16x3" in _lib.last_error()
    rc = lib.univtg_op_colsum16(_lib.ptr(buf), 64, 4, 64, 2, _lib.ptr(f), 1.0, None, 0, 0, 0, _lib.stream_ptr())
    assert rc != 0 and "fp16x3" in _lib.last_error()
    torch.cuda.synchronize()
    assert lib.univtg_launch_count() == n0


# --------------------------------------------------------------------------------------------------------- single operators
def _pair(x):
    """fp32 tensor -> [2, *shape] fp16 hi / lo planes as the kernels store them."""
    hi = x.half()
    return torch.stack([hi, (x - hi.float()).half()]).contiguous()


def _value(p):
    return p[0].double() + p[1].double()


def _check_pairs(p):
    """|lo| <= half an ulp of hi for every stored pair (fp16 ulp at hi's exponent, subnormal spacing 2^-24 at least)."""
    hi, lo = p[0].float(), p[1].float()
    e = torch.floor(torch.log2(hi.abs().clamp_min(2.0 ** -14)))
    ulp = torch.exp2(e - 10)
    assert (lo.abs() <= 0.5 * ulp + 2.0 ** -25).all()


def _c(K):
    return 4 * (math.ceil(math.log2(K)) + 1)


@pytest.mark.parametrize("M,N,K,bn", [(300, 208, 256, 64), (77, 1024, 2880, 128), (128, 64, 64, 64), (513, 96, 1024, 96)])
def test_op_gemm_fp16x3_against_fp64(M, N, K, bn):
    lib = _lib.load_library()
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g)
    b = torch.randn(N, K, generator=g) * 0.05
    if K == 2880:  # the 2818-wide projector, zero-padded to a multiple of 64
        a[:, 2818:] = 0
        b[:, 2818:] = 0
    A, B = _pair(a).cuda(), _pair(b).cuda()
    bias = torch.randn(N, generator=g).cuda()
    out32 = torch.full((M, N), float("nan"), device="cuda")
    out16 = torch.full((2, M, N), float("nan"), device="cuda", dtype=torch.float16)
    _lib.check(lib.univtg_op_gemm(_lib.ptr(A), _lib.ptr(B), M, N, K, 0, 0, 2, bn, 1, _lib.ptr(bias), 0, 1.0, _lib.ptr(out32),
                                  _lib.ptr(out16), _lib.stream_ptr()), "op_gemm fp16x3")
    torch.cuda.synchronize()
    av, bv = _value(A.cpu()), _value(B.cpu())
    ref = av @ bv.T + bias.double().cpu()
    bound = (3 * 2.0 ** -22 + _c(K) * 2.0 ** -24) * (av.abs() @ bv.abs().T) + 2.0 ** -24 * bias.double().abs().cpu()
    err = (out32.double().cpu() - ref).abs()
    assert (err <= bound).all(), f"worst err / bound {(err / bound).max().item():.3g}"
    o16 = out16.cpu()
    assert not torch.isnan(o16).any()
    _check_pairs(o16)
    assert torch.equal(o16[0], out32.cpu().half())


def test_op_gemm_fp16x3_rejects_mn_major():
    lib = _lib.load_library()
    x = torch.zeros(2, 128, 64, dtype=torch.float16, device="cuda")
    n0 = lib.univtg_launch_count()
    rc = lib.univtg_op_gemm(_lib.ptr(x), _lib.ptr(x), 128, 64, 64, 1, 0, 2, 64, 1, None, 0, 1.0, None, _lib.ptr(x), _lib.stream_ptr())
    assert rc != 0 and "fp16x3" in _lib.last_error()
    assert lib.univtg_launch_count() == n0


@pytest.mark.parametrize("rows,d,ld16", [(37, 256, 256), (9, 1024, 1024), (21, 2818, 2880), (13, 514, 576)])
def test_op_layernorm_fp16x3_against_fp64(rows, d, ld16):
    lib = _lib.load_library()
    g = torch.Generator().manual_seed(rows * d)
    x = (torch.randn(rows, d, generator=g) * 3 + 1).cuda()
    gam = (torch.rand(d, generator=g) + 0.5).cuda()
    bet = torch.randn(d, generator=g).cuda()
    out16 = torch.full((2, rows, ld16), float("nan"), device="cuda", dtype=torch.float16)
    _lib.check(lib.univtg_op_layernorm(_lib.ptr(x), rows, d, _lib.ptr(gam), _lib.ptr(bet), 1e-5, 2, None, _lib.ptr(out16), ld16,
                                       _lib.stream_ptr()), "op_layernorm fp16x3")
    torch.cuda.synchronize()
    xd = x.double().cpu()
    xc = xd - xd.mean(-1, keepdim=True)
    ref = xc * torch.rsqrt((xc * xc).mean(-1, keepdim=True) + 1e-5) * gam.double().cpu() + bet.double().cpu()
    o = out16.cpu()
    assert torch.equal(o[:, :, d:], torch.zeros_like(o[:, :, d:]))  # K padding: exact zeros in both planes
    _check_pairs(o[:, :, :d])
    got = _value(o[:, :, :d])
    bound = 2.0 ** -22 * ref.abs() + 2.0 ** -25 + _c(d) * 2.0 ** -24 * (ref.abs() + bet.double().abs().cpu() + 1)
    assert ((got - ref).abs() <= bound).all(), f"worst {((got - ref).abs() / bound).max().item():.3g}"


@pytest.mark.parametrize("B,L,H,dh,impl", [(2, 107, 8, 128, 0), (2, 300, 2, 128, 0), (3, 33, 4, 64, 0), (1, 182, 3, 64, 0),
                                           (2, 27, 6, 32, 1), (2, 107, 2, 128, 1)])
def test_op_attention_fp16x3_against_fp64(B, L, H, dh, impl):
    lib = _lib.load_library()
    d = H * dh
    g = torch.Generator().manual_seed(B * L * H + dh)
    qkv = torch.randn(B * L, 3 * d, generator=g)
    mask = torch.ones(B, L)
    mask[0, L - L // 4:] = 0
    QKV = _pair(qkv).cuda()
    out = torch.full((2, B * L, d), float("nan"), device="cuda", dtype=torch.float16)
    _lib.check(lib.univtg_op_attention(_lib.ptr(QKV), _lib.ptr(mask.cuda()), _lib.ptr(out), None, B, L, H, dh, 2, impl,
                                       _lib.stream_ptr()), "op_attention fp16x3")
    torch.cuda.synchronize()
    v = _value(QKV.cpu()).reshape(B, L, 3, H, dh)
    q, k, vv = v[:, :, 0], v[:, :, 1], v[:, :, 2]
    s = torch.einsum("bihc,bjhc->bhij", q, k) / math.sqrt(dh)
    s = s.masked_fill(mask[:, None, None, :] == 0, float("-inf"))
    p = torch.softmax(s, dim=-1)
    ref = torch.einsum("bhij,bjhc->bihc", p, vv).reshape(B * L, d)
    o = out.cpu()
    _check_pairs(o)
    got = _value(o)
    # scores: dh-term dot products of |q||k| ~ dh; softmax and P V: L-term sums of p |v|
    bound = 64 * 2.0 ** -22 * (1 + ref.abs()) * (1 + math.sqrt(dh))
    assert ((got - ref).abs() <= bound).all(), f"worst {((got - ref).abs() / bound).max().item():.3g}"
