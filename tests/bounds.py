"""Error bounds shared by the operator-level fp64 parity tests (tests/test_backward_ops_gpu.py, tests/test_forward_ops_gpu.py).

The reference is fp64, computed from exactly the 16-bit and fp32 inputs the kernel was given.  An fp32 result must satisfy
|got - ref| <= c(K) * 2^-24 * S elementwise, with S the same formula with every term replaced by its absolute value and
c(K) = 4 * (ceil(log2 K) + 1): the depth of a K-term reduction plus one level for the few roundings of each term.  A 16-bit result
may additionally differ by half an ulp of its format.  Masked entries, separator rows, padding columns and ReLU zeros have S = 0 and
must be exactly zero; rows and columns a kernel must not write must still hold NaN.  The worst |got - ref| / bound of every check is
printed (pytest -s) and summarised per kernel family at the end of each module (report_fixture).
"""
import math

import pytest
import torch

U = 2.0 ** -24
WORST = {}


def report_fixture(seen):
    """Module-scoped autouse fixture: clears WORST, and after the module prints the worst ratio per family and `seen` (coverage)."""

    @pytest.fixture(scope="module", autouse=True)
    def _report():
        WORST.clear()
        yield
        print("\nworst |got - ref| / bound per kernel family:")
        for fam, (r, case) in sorted(WORST.items()):
            print(f"  {fam:26s} {r:.3f}  ({case})")
        print("coverage:", {k: sorted(v) for k, v in seen.items()})

    return _report


def offset_view(rows, ld, dtype, byte_off, fill=float("nan")):
    """[rows, ld] view that starts byte_off bytes into a fresh allocation (16- but not 32-byte aligned for byte_off = 16)."""
    es = torch.tensor([], dtype=dtype).element_size()
    k = byte_off // es
    flat = torch.full((rows * ld + k + 64,), fill, dtype=dtype, device="cuda")
    v = flat[k:k + rows * ld].view(rows, ld)
    assert v.data_ptr() % 32 == byte_off % 32
    return v


def ulp16(x, fmt):
    """ulp of |x| in fp16 (fmt 0) / bf16 (fmt 1), x fp64 >= 0."""
    p, emin = (10, -14) if fmt == 0 else (7, -126)
    _, e = torch.frexp(x)
    ex = torch.clamp(e.to(torch.float64) - 1, min=emin)
    return torch.pow(2.0, ex - p)


def cfac(K):
    return 4 * (math.ceil(math.log2(max(int(K), 1))) + 1)


def check(family, name, got, ref, S, K, fmt=None, extra=None):
    """|got - ref| <= c(K) 2^-24 S (+ half an ulp of `fmt` for 16-bit results, + `extra`); S == 0 (and no extra) means exact."""
    got = got.double()
    ref = ref.double()
    S = S.double()
    assert got.shape == ref.shape == S.shape, (name, got.shape, ref.shape, S.shape)
    assert torch.isfinite(got).all(), f"{family}/{name}: {int((~torch.isfinite(got)).sum())} non-finite values (not written?)"
    b = cfac(K) * U * S
    if extra is not None:
        b = b + extra
    if fmt is not None:
        b = b + 0.5 * ulp16(ref.abs() + b, fmt) * (S > 0)
    err = (got - ref).abs()
    ratio = float((err / torch.where(b > 0, b, torch.full_like(b, float("inf")))).max()) if err.numel() else 0.0
    bad = err > b
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{family}/{name}: {int(bad.sum())} of {bad.numel()} entries out of bound; first flat index {i}: "
                             f"got {got.flatten()[i].item()!r} ref {ref.flatten()[i].item()!r} bound {b.flatten()[i].item()!r}; "
                             f"worst ratio {ratio:.3g}")
    print(f"  {family}/{name}: worst |got-ref|/bound = {ratio:.3f}")
    fam = family + (" (16-bit)" if fmt is not None else " (fp32)")  # a 16-bit result's ratio is dominated by its half ulp
    if ratio >= WORST.get(fam, (-1.0, ""))[0]:
        WORST[fam] = (ratio, name)


def all_nan(t, what):
    assert torch.isnan(t.float()).all(), f"{what}: a region the kernel must not write was written"
