"""Host side of the graphed training step (no GPU needed): the new C-ABI entry points are declared, bound and exported; the
seed sequence and the AdamW bias-correction table match Python restatements; ill-formed arguments are refused with a message
before anything would be launched."""
import array
import ctypes
import math
import os
import re

import pytest

from univtg_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW = ("univtg_plan_set_seed_source", "univtg_rng_advance", "univtg_rng_seed_at", "univtg_adamw_step_dev", "univtg_adamw_bias_table",
       "univtg_adamw_bias_table_len")
M64 = (1 << 64) - 1


def _prototypes():
    src = open(os.path.join(ROOT, "include", "univtg_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    out = {}
    for m in re.finditer(r"\b(\w[\w\s\*]*?)\b(univtg_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", src):
        args = [a.strip() for a in m.group(3).split(",") if a.strip() and a.strip() != "void"]
        out[m.group(2)] = (m.group(1).strip(), args)
    return out


def test_new_entry_points_are_declared_bound_and_exported():
    lib = _lib.load_library()
    protos = _prototypes()
    for name in NEW:
        assert name in protos, name
        assert hasattr(lib, name), name
        restype, argtypes = _lib.SIGNATURES[name]
        ret, args = protos[name]
        assert len(argtypes) == len(args), (name, args)
        for a, t in zip(args, argtypes):  # pointers <-> c_void_p / POINTER, 64-bit ints <-> c_uint64, floats <-> c_float
            if "*" in a:
                assert t is ctypes.c_void_p or hasattr(t, "_type_") and t.__name__.startswith("LP_"), (name, a, t)
            elif a.startswith("uint64_t"):
                assert t is ctypes.c_uint64, (name, a, t)
            elif a.startswith("float"):
                assert t is ctypes.c_float, (name, a, t)
            elif a.startswith("int32_t"):
                assert t is ctypes.c_int32, (name, a, t)
            elif a.startswith("size_t"):
                assert t is ctypes.c_size_t, (name, a, t)
        assert (ret.split()[-1] == "uint64_t") == (restype is ctypes.c_uint64), (name, ret)
    assert lib.univtg_abi_version() == 2  # additive change


def _splitmix_at(base, k):
    z = (base + k * 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def test_rng_seed_at_is_the_splitmix64_sequence():
    from univtg_b200.graphs import rng_seed_at

    lib = _lib.load_library()
    bases = [0, 1, 42, 0xDEADBEEF, M64, 1 << 63, 0x9E3779B97F4A7C15, 123456789123456789]
    for base in bases:
        seeds = [lib.univtg_rng_seed_at(base, k) for k in range(0, 300)]
        assert seeds == [_splitmix_at(base, k) for k in range(0, 300)]
        assert len(set(seeds[1:])) == 299  # consecutive replays get distinct keys
        assert rng_seed_at(base, 77) == _splitmix_at(base, 77)
    assert lib.univtg_rng_seed_at(5, M64) == _splitmix_at(5, M64)


@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.9, 0.98), (0.5, 0.9999), (0.0, 0.95)])
def test_bias_table_is_adamw_step_expression(betas):
    """Rows 1 .. 10^6 equal (float)(1 - pow((double)beta1, (double)t)) and (float)sqrt(1 - pow((double)beta2, (double)t)) with
    the float betas widened to double, as univtg_adamw_step computes them; the table length saturates both at 1.0f."""
    from univtg_b200.graphs import bias_correction_table

    b1 = float(array.array("f", [betas[0]])[0])  # the float the C ABI receives, widened to double
    b2 = float(array.array("f", [betas[1]])[0])
    n = 1_000_000
    t = bias_correction_table(betas[0], betas[1], n)
    got1 = array.array("f", t[:, 0].tolist())
    got2 = array.array("f", t[:, 1].tolist())
    want1 = array.array("f", [1.0 - math.pow(b1, s) for s in range(1, n + 1)])
    want2 = array.array("f", [math.sqrt(1.0 - math.pow(b2, s)) for s in range(1, n + 1)])
    assert got1.tobytes() == want1.tobytes()
    assert got2.tobytes() == want2.tobytes()
    lib = _lib.load_library()
    rows = lib.univtg_adamw_bias_table_len(betas[0], betas[1])
    assert 1 <= rows
    full = bias_correction_table(betas[0], betas[1])
    assert full.shape[0] == rows
    assert tuple(full[-1].tolist()) == (1.0, 1.0)
    if rows > 1:
        assert tuple(full[-2].tolist()) != (1.0, 1.0)
    if rows <= n:  # every later step of the eager expression is (1, 1) too
        assert all(v == 1.0 for v in got1[rows - 1:]) and all(v == 1.0 for v in got2[rows - 1:])


def _err(lib, rc, *words):
    assert rc != 0
    msg = _lib.last_error()
    for w in words:
        assert w in msg, msg
    return msg


def test_bad_arguments_are_refused_with_a_message():
    lib = _lib.load_library()
    V = ctypes.c_void_p
    ok = V(4096)  # aligned, never dereferenced: every call below fails its host-side checks first
    _err(lib, lib.univtg_plan_set_seed_source(None, None), "univtg_plan_set_seed_source", "null plan")
    _err(lib, lib.univtg_plan_set_seed_source(ok, V(4100 + 2)), "8-byte aligned")
    _err(lib, lib.univtg_rng_advance(1, None, ok, None), "univtg_rng_advance", "null")
    _err(lib, lib.univtg_rng_advance(1, V(4097), ok, None), "aligned")
    _err(lib, lib.univtg_rng_advance(1, ok, ok, None), "distinct")
    args = dict(params=ok, grads=ok, m=ok, v=ok, n=16, lr=ok, b1=0.9, b2=0.999, eps=1e-8, wd=1e-4, step=ok, clip=0.1, wcg=0,
                scratch=ok, cfg=None, packed=None, bc=ok, rows=10, stream=None)

    def call(**over):
        a = dict(args, **over)
        return lib.univtg_adamw_step_dev(a["params"], a["grads"], a["m"], a["v"], a["n"], a["lr"], a["b1"], a["b2"], a["eps"], a["wd"],
                                         a["step"], a["clip"], a["wcg"], a["scratch"], a["cfg"], a["packed"], a["bc"], a["rows"],
                                         a["stream"])

    _err(lib, call(params=None), "univtg_adamw_step_dev", "null params")
    _err(lib, call(lr=None), "null lr_dev")
    _err(lib, call(step=None), "null lr_dev, step_dev")
    _err(lib, call(bc=None), "bc_table")
    _err(lib, call(n=18), "multiple of 4")
    _err(lib, call(rows=0), "table_len")
    _err(lib, call(grads=V(4104)), "16-byte aligned")
    _err(lib, call(step=V(4098)), "misaligned")
    _err(lib, call(packed=ok), "both be given")
    out = (ctypes.c_float * 8)()
    _err(lib, lib.univtg_adamw_bias_table(0.9, 0.999, 0, out), "len")
    _err(lib, lib.univtg_adamw_bias_table(0.9, 0.999, 4, None), "null out_host")
    _err(lib, lib.univtg_adamw_bias_table(1.0, 0.999, 4, out), "[0, 1)")
    assert lib.univtg_adamw_bias_table_len(0.9, 1.0) == 0
    assert "[0, 1)" in _lib.last_error()
    assert lib.univtg_adamw_bias_table(0.9, 0.999, 4, out) == 0
    b1 = float(array.array("f", [0.9])[0])
    assert out[0] == array.array("f", [1.0 - b1])[0] and out[2] == array.array("f", [1.0 - b1 * b1])[0]


def test_graphed_step_needs_flat_adamw():
    from univtg_b200.graphs import GraphedTrainStep

    class _M:
        pass

    with pytest.raises(TypeError, match="FlatAdamW"):
        GraphedTrainStep(_M(), None, object())
