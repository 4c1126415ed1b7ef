"""Operator-level fp64 parity of the attention backward (csrc/attention_bwd.cu: the eight wgmma instantiations; csrc/backward.cu:
attention_bwd_simt_kernel<0/1> and attn_delta_kernel), driven through univtg_op_attention_bwd_full and univtg_op_attn_delta.

Inputs are built as training builds them: univtg_op_attention_fwd (pinned by tests/test_forward_ops_gpu.py) gives O and lse with the
same rng, p and layer the backward regenerates its dropout from; dO is a loss-scaled gradient 2^10 N(0, 10^-3) in the activation
format; delta comes from univtg_op_attn_delta and is checked on the way.  The reference and its bounds are tests/attn_bwd_ref.py:
fp64 from the exact 16-bit operands and the given fp32 lse and delta, with the dropout multipliers read back through
univtg_attention_dropout_mask.  Outputs are NaN-filled first: masked keys must get exact zeros in dK and dV, the fused 16-bit mode
must leave dqkv32 untouched and the fp32 modes must write every entry.  Each case asserts the instantiation and the dQ mode the
routing (attention_bwd_route, the rule univtg_backward uses) reached; the module asserts the coverage at the end (pytest -s prints
it with the worst ratio per family).
"""
import ctypes

import pytest
import torch

from tests.attn_bwd_ref import attn_bwd_reference, delta_reference, key_mask_gap
from tests.bounds import WORST, all_nan, check, offset_view, report_fixture
from tests.test_backward_ops_gpu import DT, P, gen, lib, nan, randn
from univtg_b200 import _lib

pytestmark = pytest.mark.gpu

_SEEN = {"bwd_kernel": set(), "delta_vec": set(), "dq_mode": set()}
_RUNS = {"case": 0, "delta": 0}  # cases that ran: the coverage test needs the whole module
_report = report_fixture(_SEEN)

LAYER = 2


def _kexp(dh, impl, fmt, drop):
    return 8 + drop if impl == 1 else (4 if dh == 128 else 0) + 2 * fmt + drop


def run_delta(dO, fmt_do, O, fmt_o, B, L, H, dh):
    delta = nan((B, H, L))
    vec = ctypes.c_int32(-9)
    _lib.check(lib().univtg_op_attn_delta(P(dO), fmt_do, P(O), fmt_o, P(delta), B, L, H, dh, ctypes.byref(vec), None), "op_attn_delta")
    torch.cuda.synchronize()
    _SEEN["delta_vec"].add(vec.value)
    return delta, vec.value


def check_delta(tag, delta, dO, O, B, L, H, dh):
    ref, S = delta_reference(dO, O, B, L, H, dh)
    check("attn_delta", tag, delta, ref, S, dh)


def run_bwd(qkv, dO, km, lse, delta, B, L, H, dh, fmt, impl, fused, rng, p):
    d = H * dh
    dqkv32 = nan((B * L, 3 * d))
    dqkv16 = torch.full((B * L, 3 * d), float("nan"), dtype=DT[fmt], device="cuda") if fused else None
    a = _lib.AttnBwd(P(qkv), P(dO), P(km), P(lse), P(delta), P(dqkv32), P(dqkv16), B, L, H, dh, fmt, impl)
    used, mode = ctypes.c_int32(-9), ctypes.c_int32(-9)
    _lib.check(lib().univtg_op_attention_bwd_full(ctypes.byref(a), ctypes.byref(rng) if rng else None, p, LAYER, ctypes.byref(used),
                                                  ctypes.byref(mode), None), "op_attention_bwd_full")
    torch.cuda.synchronize()
    _SEEN["bwd_kernel"].add(used.value)
    _SEEN["dq_mode"].add(mode.value)
    return dqkv32, dqkv16, used.value, mode.value


def run_case(tag, fam, B, L, H, dh, fmt, impl, km, p=0.0, seed=0, plant=None):
    """Forward -> attn_delta -> backward in every dQ mode the shape allows, each checked against the fp64 reference."""
    d = H * dh
    g = gen(seed)
    x = randn((B * L, 3 * d), g)
    dO32 = randn((B * L, d), g, 1e-3 * 2.0 ** 10)
    if plant == "large_scores":  # sigma S ~ +-36 with spread: P one-hot in many rows, most entries underflow to 0 in fp32
        x[:L, :2 * d] *= 6.0
    if plant == "zero_do_row":
        dO32[L // 2] = 0.0
        dO32[L + 1] = 0.0
    qkv = x.to(DT[fmt])
    dO = dO32.to(DT[fmt])
    kmc = km.cuda()
    rng = _lib.Rng(900 + seed, 0.0, 0.0) if p > 0 else None
    # ---- forward: O and lse exactly as training stores them ----
    out, lse = torch.full((B * L, d), float("nan"), dtype=DT[fmt], device="cuda"), nan((B, H, L))
    fa = _lib.AttnFwd(P(qkv), P(kmc), P(out), P(lse), B, L, H, dh, fmt, impl, 0)
    _lib.check(lib().univtg_op_attention_fwd(ctypes.byref(fa), ctypes.byref(rng) if rng else None, p, LAYER, None, None), "op_attention_fwd")
    delta, _ = run_delta(dO, fmt, out, fmt, B, L, H, dh)
    check_delta(f"{tag}/delta", delta, dO, out, B, L, H, dh)
    mul = None
    if p > 0:
        mul = nan((B, H, L, L))
        _lib.check(lib().univtg_attention_dropout_mask(ctypes.byref(rng), p, LAYER, B, H, L, P(mul), None), "attention_dropout_mask")
        torch.cuda.synchronize()
    ref = attn_bwd_reference(qkv, dO, kmc, lse, delta, B, L, H, dh, fmt, impl == 0, mul)
    _RUNS["case"] += 1
    masked = (kmc == 0).flatten()  # key rows that must get exact zeros
    modes = [False] + ([True] if impl == 0 and L <= 128 else [])
    for fused in modes:
        dqkv32, dqkv16, used, mode = run_bwd(qkv, dO, kmc, lse, delta, B, L, H, dh, fmt, impl, fused, rng, p)
        assert used == _kexp(dh, impl, fmt, int(p > 0)), f"routing reached backward kernel {used}"
        assert mode == (0 if fused else (1 if impl == 0 and L <= 128 else 2)), f"dq_mode {mode}"
        if fused:
            all_nan(dqkv32, "dqkv32 (fused 16-bit mode)")
            got, f16, fam_ = dqkv16, fmt, fam + "_fused"
        else:
            got, f16, fam_ = dqkv32, None, fam
        for i, n in enumerate(("dq", "dk", "dv")):
            r, S, E = ref[n]
            gv = got[:, i * d:(i + 1) * d]
            check(fam_, f"{tag}/{'fused' if fused else 'fp32'}/{n}", gv, r, S, L, fmt=f16, extra=E)
            if n != "dq" and masked.any():
                assert (gv[masked].float() == 0).all(), f"{tag}: {n} rows of masked keys must be exact zeros"


# ================================================= attn_delta =================================================
# (dh, H, fmt_do, fmt_o, O misaligned by 2 bytes, vector path expected); d = H dh below and above 256
DELTA_CASES = [(32, 4, 0, 0, False, 1), (32, 12, 1, 1, False, 1), (64, 2, 0, 0, False, 1), (64, 16, 1, 1, False, 1),
               (128, 1, 1, 1, False, 1), (128, 2, 0, 0, False, 1), (128, 8, 1, 0, False, 1),
               (40, 2, 0, 0, False, 0), (40, 8, 1, 1, False, 0), (96, 2, 1, 1, False, 0), (96, 5, 0, 0, False, 0),
               (64, 6, 0, 0, True, 0), (128, 3, 1, 1, True, 0)]


@pytest.mark.parametrize("dh,H,fmt_do,fmt_o,mis,vexp", DELTA_CASES)
def test_attn_delta(dh, H, fmt_do, fmt_o, mis, vexp):
    B, L = 3, 107  # 321 rows: the last block of 8 rows is partial
    d = H * dh
    g = gen(100 + dh + H)
    dO = randn((B * L, d), g, 1e-3 * 2.0 ** 10).to(DT[fmt_do])
    dO[5] = 0.0
    O = offset_view(B * L, d, DT[fmt_o], 2) if mis else torch.empty((B * L, d), dtype=DT[fmt_o], device="cuda")
    O.copy_(randn((B * L, d), g).to(DT[fmt_o]))
    delta, vec = run_delta(dO, fmt_do, O, fmt_o, B, L, H, dh)
    _RUNS["delta"] += 1
    assert vec == vexp, f"attn_delta took the {'vector' if vec else 'scalar'} path"
    check_delta(f"dh{dh}_H{H}_f{fmt_do}{fmt_o}{'_mis' if mis else ''}", delta, dO, O, B, L, H, dh)
    assert (delta[0, :, 5] == 0).all(), "an all-zero dO row gives delta exactly 0"


# ================================================= wgmma =================================================
WG_L = [1, 63, 64, 65, 107, 127, 128, 129, 182, 255, 256, 257, 300, 1277]


@pytest.mark.parametrize("L", WG_L)
@pytest.mark.parametrize("dh", [64, 128])
@pytest.mark.parametrize("fmt", [0, 1])
def test_attention_bwd_wgmma(L, dh, fmt):
    B, H = 2, 2
    run_case(f"L{L}_dh{dh}_f{fmt}", "attn_bwd_wgmma", B, L, H, dh, fmt, 0, key_mask_gap(B, L, None), seed=1000 + L + dh + fmt)


@pytest.mark.parametrize("H,dh,fmt", [(8, 128, 0), (8, 128, 1), (16, 64, 0)])
def test_attention_bwd_benchmark_shape(H, dh, fmt):
    """cfg2_full's encoder attention (B 32, L = 75 clips + 32 text tokens): one key tile, the fused 16-bit path training takes."""
    B, L = 32, 107
    run_case(f"B32_L107_H{H}_dh{dh}_f{fmt}", "attn_bwd_wgmma", B, L, H, dh, fmt, 0, key_mask_gap(B, L, None), seed=2000 + H + fmt)


# ================================================= SIMT =================================================
@pytest.mark.parametrize("L", [1, 65, 300, 1277])
@pytest.mark.parametrize("dh", [32, 40, 96])
@pytest.mark.parametrize("fmt", [0, 1])
def test_attention_bwd_simt(L, dh, fmt):
    B, H = 2, 2
    run_case(f"L{L}_dh{dh}_f{fmt}", "attn_bwd_simt", B, L, H, dh, fmt, 1, key_mask_gap(B, L, None), seed=3000 + L + dh + fmt)


# ================================================= dropout =================================================
@pytest.mark.parametrize("dh,impl,fmt", [(64, 0, 0), (64, 0, 1), (128, 0, 0), (128, 0, 1), (32, 1, 0), (96, 1, 1)])
@pytest.mark.parametrize("L", [65, 107, 300])
@pytest.mark.parametrize("p", [0.1, 0.25])
def test_attention_bwd_dropout(dh, impl, fmt, L, p):
    B, H = 2, 2
    run_case(f"p{p}_L{L}_dh{dh}_i{impl}_f{fmt}", "attn_bwd_dropout", B, L, H, dh, fmt, impl, key_mask_gap(B, L, None), p=p,
             seed=4000 + L + dh + fmt + int(100 * p))


# ================================================= planted edges =================================================
def _edge_mask(edge, B, L):
    km = key_mask_gap(B, L, None)
    if edge == "one_key":  # sample 1 attends to exactly one key
        km[1] = 0
        km[1, L // 3] = 1
    elif edge == "masked_127_129":  # masked keys on both sides of the first key-tile boundary
        km[:, 127:130] = 0
    return km


EDGE_PATHS = [(64, 0, 0), (128, 0, 1), (40, 1, 0)]


@pytest.mark.parametrize("edge,L", [("one_key", 107), ("one_key", 300), ("masked_127_129", 300), ("large_scores", 107),
                                    ("large_scores", 300), ("zero_do_row", 107), ("zero_do_row", 257)])
@pytest.mark.parametrize("dh,impl,fmt", EDGE_PATHS)
def test_attention_bwd_edges(edge, L, dh, impl, fmt):
    B, H = 2, 2
    fam = "attn_bwd_wgmma" if impl == 0 else "attn_bwd_simt"
    plant = edge if edge in ("large_scores", "zero_do_row") else None
    run_case(f"{edge}_L{L}_dh{dh}_i{impl}_f{fmt}", fam, B, L, H, dh, fmt, impl, _edge_mask(edge, B, L), seed=5000 + L + dh, plant=plant)


N_CASES = (len(WG_L) * 2 * 2 + 3) + 4 * 3 * 2 + 6 * 3 * 2 + 7 * len(EDGE_PATHS)
FAMILIES = ["attn_delta (fp32)", "attn_bwd_wgmma (fp32)", "attn_bwd_wgmma_fused (16-bit)", "attn_bwd_simt (fp32)",
            "attn_bwd_dropout (fp32)", "attn_bwd_dropout_fused (16-bit)"]


def test_attention_bwd_covers_every_instantiation():
    """Runs last in the module: the cases above reached all 10 backward instantiations, both attn_delta paths and all three dQ
    modes, and every family was checked."""
    if _RUNS["case"] < N_CASES or _RUNS["delta"] < len(DELTA_CASES):
        pytest.skip("needs every case of the module to have run")
    assert _SEEN["bwd_kernel"] == set(range(10)), sorted(set(range(10)) - _SEEN["bwd_kernel"])
    assert _SEEN["delta_vec"] == {0, 1}, _SEEN["delta_vec"]
    assert _SEEN["dq_mode"] == {0, 1, 2}, _SEEN["dq_mode"]
    for fam in FAMILIES:
        assert fam in WORST and WORST[fam][0] <= 1.0, (fam, WORST.get(fam))
