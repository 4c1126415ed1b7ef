"""ptxas record of the GEMM kernel: every gemm_wgmma_kernel instantiation keeps its wgmma pipeline and spills nothing.

gemm.cu is compiled with the library's own nvcc flags plus `-Xptxas -v`.  ptxas warns with C7511 when it has to serialise the
wgmma.mma_async instructions of a kernel (each one waits for the previous one, so the mainloop's wgmma_wait<1> pipelining is
lost); that happened to every instantiation while one k-loop body switched over all tile widths at run time.  No GPU is needed.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

import __graft_entry__ as G

NVCC = shutil.which("nvcc") or ("/usr/local/cuda/bin/nvcc" if os.path.exists("/usr/local/cuda/bin/nvcc") else None)
KERNELS = ("<1, false>", "<1, true>", "<2, false>", "<2, true>", "<1, false, true>")


@pytest.fixture(scope="module")
def ptxas_log():
    if NVCC is None:
        pytest.skip("nvcc not found")
    with tempfile.TemporaryDirectory() as tmp:
        cmd = [NVCC] + G.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(G.CSRC, "gemm.cu"), "-o", os.path.join(tmp, "gemm.o")]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    return r.stdout


def per_kernel(log):
    """mangled gemm_wgmma_kernel name -> {"regs", "stack", "spill_st", "spill_ld", "c7511", "c7519"}"""
    out, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1) if "gemm_wgmma_kernel" in m.group(1) else None
            if cur:
                out[cur] = dict(regs=None, stack=None, spill_st=None, spill_ld=None, c7511=0, c7519=0)
            continue
        m = re.search(r"\((C75\d\d)\).*function '(\w+)'", line)
        if m and "gemm_wgmma_kernel" in m.group(2):
            out.setdefault(m.group(2), dict(regs=None, stack=None, spill_st=None, spill_ld=None, c7511=0, c7519=0))
            key = m.group(1).lower()
            if key in ("c7511", "c7519"):
                out[m.group(2)][key] += 1
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m:
            out[cur].update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)))
        m = re.search(r"Used (\d+) registers", line)
        if m:
            out[cur]["regs"] = int(m.group(1))
    return out


def test_every_instantiation_is_reported(ptxas_log):
    k = per_kernel(ptxas_log)
    print({n: v for n, v in k.items()})
    assert len(k) == len(KERNELS), f"expected the {len(KERNELS)} instantiations {KERNELS}, ptxas reported {sorted(k)}"
    for name, v in k.items():
        assert v["regs"] is not None and v["spill_st"] is not None, (name, v)


def test_no_serialised_wgmma(ptxas_log):
    assert "C7511" not in ptxas_log, "\n".join(l for l in ptxas_log.splitlines() if "C7511" in l)


def test_no_spills(ptxas_log):
    for name, v in per_kernel(ptxas_log).items():
        assert v["spill_st"] == 0 and v["spill_ld"] == 0, (name, v)
