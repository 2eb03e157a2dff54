"""Build-level checks of the persistent tile engine (tc_engine.cuh), which no result can show: a register spill or a
serialized wgmma (ptxas C7510 / C7512 / C7513) leaves every output correct and only costs time.

  * cuobjdump -res-usage of the built libb200asr.so: every tc_engine_kernel instantiation uses no stack and no local
    memory, and the GemmPolicy instantiations are exactly those of tests/test_gpu_gemm_epilogues.py's map;
  * each translation unit that includes tc_engine.cuh recompiled with build.sh's flags and -Xptxas -v,-warn-spills: every
    engine entry spills 0 bytes and no C75xx names one; tc_gemm.cu spills nothing anywhere.  The halo weight-gradient
    kernel (tc_conv_wgrad.cu, not an engine instantiation) spills a few registers and reports C7512 by design (DESIGN.md
    section 8); it is the one kernel allowed to.

Runs without a GPU (nvcc cross-compiles for sm_90a); skips when nvcc, cuobjdump or the library is absent.  The recompile
takes about 30 s of wall time on 8 cores."""
import os
import re
import shlex
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "end2end-asr-pytorch_b200", "csrc")
LIB = os.path.join(ROOT, "end2end-asr-pytorch_b200", "libb200asr.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")           # as build.sh
CUOBJDUMP = os.path.join(os.path.dirname(NVCC), "cuobjdump")

# kernels allowed a C75xx report and spills: the halo weight-gradient kernel's C7512 (too few registers for its second
# fragment buffer), which DESIGN.md documents
ALLOWED_SERIAL = "tc_conv3x3_wgrad_kernel"
_GEMM_MANGLED = re.compile(r"10GemmPolicyILb([01])ELb([01])ELb([01])EEELi(\d+)E")


def _need(*paths):
    for p in paths:
        if not os.path.exists(p):
            pytest.skip(f"{p} not found (needs the CUDA toolkit and build.sh)")


def _gemm_instantiations(names):
    out = set()
    for n in names:
        m = _GEMM_MANGLED.search(n)
        if m and "tc_engine_kernel" in n:
            out.add(tuple(f == "1" for f in m.groups()[:3]) + (int(m.group(4)),))
    return out


def _map_keys():
    from tests.test_gpu_gemm_epilogues import GEMM_INSTANTIATIONS
    return set(GEMM_INSTANTIATIONS)


def test_engine_kernels_use_no_local_memory():
    """cuobjdump -res-usage: STACK:0 LOCAL:0 for every tc_engine_kernel instantiation in the library, and the GemmPolicy ones
    are exactly the instantiation map's 14."""
    _need(CUOBJDUMP, LIB)
    out = subprocess.run([CUOBJDUMP, "-res-usage", LIB], check=True, capture_output=True, text=True).stdout
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out))
    engine = {n: u for n, u in usage.items() if "tc_engine_kernel" in n}
    assert len(engine) >= 14, sorted(engine)
    bad = {n: u for n, u in engine.items() if not (re.search(r"\bSTACK:0\b", u) and re.search(r"\bLOCAL:0\b", u))}
    assert not bad, bad
    assert _gemm_instantiations(engine) == _map_keys()


def _read(path):
    with open(path) as f:
        return f.read()


def _build_flags():
    """build.sh's nvcc flags, without the optional B200ASR_DEFS."""
    m = re.search(r'^FLAGS="([^"]*)"', _read(os.path.join(ROOT, "build.sh")), re.M)
    assert m, "build.sh has no FLAGS line"
    return shlex.split(m.group(1).replace("${B200ASR_DEFS:-}", ""))


def _ptxas_report(log):
    """{function: spill store bytes} and the C75xx lines of one ptxas -v log."""
    spills = {n: int(s) for n, s in re.findall(r"Function properties for (\S+)\s*\n\s*\d+ bytes stack frame, (\d+) bytes spill stores",
                                               log)}
    serial = [ln for ln in log.splitlines() if re.search(r"\(C75\d\d\)", ln)]
    return spills, serial


def test_engine_units_compile_without_spills_or_serialized_wgmma(tmp_path):
    """Every .cu that includes tc_engine.cuh, recompiled in parallel into tmp_path with build.sh's flags and
    -Xptxas -v,-warn-spills: 0 bytes of spill stores for every engine entry and every tc_gemm.cu function, no C75xx naming
    an engine entry, and none at all but the halo weight-gradient kernel's.  tc_gemm.cu reports the 14 GemmPolicy entries
    and gemm_splitk_reduce_kernel."""
    _need(NVCC)
    units = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu") and '#include "tc_engine.cuh"' in _read(os.path.join(CSRC, f)))
    assert "tc_gemm.cu" in units and len(units) >= 2, units
    flags = _build_flags() + ["-Xptxas", "-v,-warn-spills"]
    procs = {u: subprocess.Popen([NVCC, *flags, "-c", os.path.join(CSRC, u), "-o", str(tmp_path / (u + ".o"))],
                                 stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=ROOT) for u in units}
    logs = {}
    for u, p in procs.items():
        logs[u] = p.communicate(timeout=1800)[0]
        assert p.returncode == 0, (u, logs[u][-2000:])
    engine_entries = 0
    for u, log in logs.items():
        spills, serial = _ptxas_report(log)
        assert spills, (u, "no ptxas -v report")
        engine = {n: s for n, s in spills.items() if "tc_engine_kernel" in n}
        engine_entries += len(engine)
        assert not {n: s for n, s in engine.items() if s}, u
        if u == "tc_gemm.cu":
            assert not {n: s for n, s in spills.items() if s}, u
            assert len(spills) == 15 and _gemm_instantiations(spills) == _map_keys(), sorted(spills)
        for ln in serial:
            assert "tc_engine_kernel" not in ln and ALLOWED_SERIAL in ln and "(C7512)" in ln, (u, ln)
    assert engine_entries >= 14
