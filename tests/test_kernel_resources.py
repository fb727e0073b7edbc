"""Register budget of the hex-mesh face kernels, read from ptxas without a GPU.

RevB<6,0> (the transpose product's face kernel on hexahedral meshes) and FwdB<6,0> (the residual's) are compiled alone, with
the product Makefile's flags and the product's launch bounds (csrc/launch_traits.hpp).  Neither may use a stack frame --
an array the kernel indexes through a run-time value or a pointer lives in local memory -- and RevB may not spill: each
local-memory round trip sits in the dependent chain of a kernel that waits on its gathers."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "dafoam_b200", "csrc")

KERNELS = {
    "RevB<6,0>": "_ZN3dab8kernel1dINS_4RevBILi6ELi0EEEEEviT_",
    "FwdB<6,0>": "_ZN3dab8kernel1dINS_4FwdBILi6ELi0EEEEEviT_",
}

TU = """#include "launch_traits.hpp"
namespace dab
{
template __global__ void kernel1d<RevB<6, 0>>(int, RevB<6, 0>);
template __global__ void kernel1d<FwdB<6, 0>>(int, FwdB<6, 0>);
}
"""


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if cand and os.path.isfile(cand) and os.access(cand, os.X_OK):
            return cand
    return None


def _makefile_flags():
    """NVFLAGS of the product Makefile with $(ARCH) expanded, minus what only the shared-library link needs."""
    text = open(os.path.join(CSRC, "Makefile")).read()
    arch = re.search(r"^ARCH\s*:?=\s*(.+)$", text, re.M).group(1).split()
    flags = re.search(r"^NVFLAGS\s*\??=\s*(.+)$", text, re.M).group(1).split()
    out = []
    for f in flags:
        out.extend(arch if f == "$(ARCH)" else [f])
    return out


def _resources(log):
    """{mangled entry name: (stack frame, spill stores, spill loads, registers)} from `ptxas -v` output."""
    res, cur = {}, None
    for line in log.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur:
            res[cur] = tuple(int(v) for v in m.groups())
        m = re.search(r"Used (\d+) registers", line)
        if m and cur in res and len(res[cur]) == 3:
            res[cur] = res[cur] + (int(m.group(1)),)
    return res


@pytest.fixture(scope="module")
def resources(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    d = tmp_path_factory.mktemp("kres")
    src = d / "kres.cu"
    src.write_text(TU)
    flags = _makefile_flags()
    assert "-DDAB_PREFETCH_IDX" in flags and "-O3" in flags and "arch=compute_90a,code=sm_90a" in flags
    if "-Xptxas" not in flags:
        flags += ["-Xptxas", "-v"]
    p = subprocess.run([nvcc, *flags, "-I", CSRC, "-c", "-x", "cu", str(src), "-o", str(d / "kres.o")],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-4000:]
    res = _resources(p.stdout + p.stderr)
    for name, mangled in KERNELS.items():
        assert mangled in res, "no ptxas report for " + name
    return res


@pytest.mark.parametrize("name", sorted(KERNELS))
def test_face_kernel_has_no_stack_frame(resources, name):
    frame, st, ld, regs = resources[KERNELS[name]]
    assert frame == 0, "%s: %d bytes stack frame (%d registers, spills %d/%d bytes)" % (name, frame, regs, st, ld)


def test_revb_does_not_spill(resources):
    frame, st, ld, regs = resources[KERNELS["RevB<6,0>"]]
    assert st == 0 and ld == 0, "RevB<6,0>: %d bytes spill stores, %d bytes spill loads at %d registers" % (st, ld, regs)
