"""Host-side plan of the backward's merged GEMM launches: per-problem split-K factors and the static unit-to-CTA deal.

Each data gradient of the backward shares one launch with the weight gradients that read the same operand (train.cu,
univtg_backward).  choose_tile gives each problem of such a launch its own split-K factor, and gemm_wgmma_kernel deals the
launch's units (output tile x k-split) to its persistent CTAs longest first, in waves of alternating direction.
univtg_debug_choose_tile_group asks the cost model, univtg_debug_gemm_deal walks the deal as the kernel's CTAs walk it.
No GPU is needed.
"""
import ctypes
import random

import pytest

from univtg_b200 import _lib, synth

SMS = 132


def lib():
    return _lib.load_library()


def arr(xs):
    return (ctypes.c_int32 * len(xs))(*xs)


def choose(problems, sms=SMS, step=64):
    """problems: (M, N, K, max_split) -> (bn, [ksplit per problem])"""
    n = len(problems)
    bn, ks = ctypes.c_int32(0), (ctypes.c_int32 * n)()
    rc = lib().univtg_debug_choose_tile_group(arr([p[0] for p in problems]), arr([p[1] for p in problems]),
                                              arr([(p[2] + 63) // 64 for p in problems]), arr([p[3] for p in problems]), n, sms,
                                              step, ctypes.byref(bn), ks)
    assert rc == 0, _lib.last_error()
    return bn.value, list(ks)


def deal(problems, ks, bn, sms=SMS):
    """CTA of every unit (problem by problem, tile order), as the kernel runs the launch"""
    n = len(problems)
    args = (arr([p[0] for p in problems]), arr([p[1] for p in problems]), arr([(p[2] + 63) // 64 for p in problems]), arr(ks), n,
            sms, bn)
    total = lib().univtg_debug_gemm_deal(*args, None, 0)
    assert total > 0, _lib.last_error()
    cta = (ctypes.c_int32 * total)()
    assert lib().univtg_debug_gemm_deal(*args, cta, total) == total
    return list(cta)


def units(problems, ks, bn):
    """(problem, k-blocks) of every unit, in the numbering univtg_debug_gemm_deal uses"""
    out = []
    for p, (M, N, K, _), s in zip(range(len(problems)), problems, ks):
        kb = (K + 63) // 64
        per = (kb + s - 1) // s
        tiles = ((M + 127) // 128) * ((N + bn - 1) // bn)
        for split in range(s):
            out += [(p, min(kb, (split + 1) * per) - split * per)] * tiles
    return out


def backward_launches(cfg_name):
    """The merged launches of one encoder layer and of a later projector layer (train.cu), (M, N, K, max_split) each;
    the data gradients come first."""
    c = synth.CONFIGS[cfg_name]
    B, Lv, Lt, d, ff = c["batch"], c["l_vid"], c["l_txt"], c["hidden_dim"], c["dim_feedforward"]
    M, Mv, Mt = B * (Lv + Lt), B * Lv, B * Lt
    return {
        "ffn2": [(M, ff, d, 1), (d, ff, M, 4)],
        "ffn1": [(M, d, ff, 1), (ff, d, M, 4)],
        "out_proj": [(M, d, d, 1), (d, d, M, 4)],
        "qkv": [(M, d, 3 * d, 1), (2 * d, d, M, 4), (d, d, M, 4)],
        "qkv_txt_pos": [(M, d, 3 * d, 1), (Mt, d, 2 * d, 1), (2 * d, d, M, 4), (d, d, M, 4)],
        "proj1": [(d, d, Mv, 4), (d, d, Mt, 4), (Mv, d, d, 1), (Mt, d, d, 1)],
    }


@pytest.mark.parametrize("cfg_name", ["cfg2", "cfg4"])
def test_merged_launches_split_only_weight_gradients(cfg_name):
    for name, probs in backward_launches(cfg_name).items():
        bn, ks = choose(probs)
        assert 64 <= bn <= 256 and bn % 64 == 0, (name, bn)
        for (M, N, K, lim), s in zip(probs, ks):
            if lim == 1:
                assert s == 1, (name, ks)  # data gradients are never split
            else:
                assert s in (1, 2, 4) and (s == 1 or 4 * s <= (K + 63) // 64), (name, ks)


def test_cfg2_data_gradient_launches():
    """At cfg2 the d-wide data gradient alone is one wave of 108 tiles: the merged launch gives it ksplit 1 and the weight
    gradient a split the deal can place beside it."""
    bn, ks = choose(backward_launches("cfg2")["ffn2"])
    assert ks[0] == 1 and ks[1] in (1, 2, 4)


def check_deal(probs, ks, bn, sms=SMS):
    cta = deal(probs, ks, bn, sms)
    us = units(probs, ks, bn)
    assert len(cta) == len(us)
    grid = min(len(us), sms)
    # every unit is run, by exactly one CTA of the grid (no -1 = never, -2 = twice)
    assert all(0 <= c < grid for c in cta), sorted(set(c for c in cta if not 0 <= c < grid))
    # each CTA runs at most one unit per wave, and every CTA of the grid has work
    per = [0] * grid
    for c in cta:
        per[c] += 1
    assert min(per) >= 1 and max(per) == (len(us) + grid - 1) // grid
    # longest first: the units in deal order (sorted by k-blocks per unit, problems otherwise in order) fill wave after wave
    load = [0] * grid
    for (p, kb), c in zip(us, cta):
        load[c] += kb
    assert sum(load) == sum(kb for _, kb in us)
    return load


@pytest.mark.parametrize("cfg_name", ["cfg2", "cfg4"])
def test_deal_covers_every_unit_of_the_merged_launches(cfg_name):
    for name, probs in backward_launches(cfg_name).items():
        bn, ks = choose(probs)
        check_deal(probs, ks, bn)
        for s in (1, 2, 4):  # every split the model may pick, at every width
            ks2 = [1 if lim == 1 else (s if 4 * s <= (K + 63) // 64 else 1) for (_, _, K, lim) in probs]
            for w in (64, 128, 192, 256):
                check_deal(probs, ks2, w)


def test_deal_covers_every_unit_random():
    rng = random.Random(7)
    for _ in range(200):
        n = rng.randint(1, 4)
        probs = [(rng.randint(1, 2000), rng.randint(1, 1500), rng.randint(1, 4000), 1) for _ in range(n)]
        ks = [rng.choice([s for s in (1, 2, 4, 8) if s <= (K + 63) // 64]) for (_, _, K, _) in probs]
        check_deal(probs, ks, rng.choice([64, 128, 192, 256]), sms=rng.choice([1, 7, 114, 132]))


def test_deal_balances_long_and_short_units():
    """32 long weight-gradient tiles beside 108 short data-gradient tiles on 132 SMs: dealt in problem order round-robin, eight
    CTAs would run a long and a short unit; longest first with the direction reversed in the second wave, the eight short units
    left over go to CTAs that ran a short one."""
    probs = [(3424, 1024, 1024, 1), (1024, 1024, 3424, 1)]
    load = check_deal(probs, [1, 1], 256)
    assert max(load) == 54 and sorted(load)[-33] == 32


def test_bad_arguments_are_rejected():
    z = ctypes.c_int32(0)
    one = arr([1])
    assert lib().univtg_debug_choose_tile_group(None, one, one, one, 1, SMS, 64, ctypes.byref(z), arr([0])) != 0
    assert lib().univtg_debug_choose_tile_group(one, one, one, arr([3]), 1, SMS, 64, ctypes.byref(z), arr([0])) != 0
    assert lib().univtg_debug_gemm_deal(one, one, one, arr([2]), 1, SMS, 64, None, 0) == -1  # 2 splits of 1 k-block
