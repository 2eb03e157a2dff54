"""Build-level checks of the halo weight-gradient kernel (tc_conv_wgrad.cu), which no result can show: a register spill or a
serialized wgmma leaves every output correct and only costs time.

tc_conv_wgrad.cu recompiled with build.sh's flags and -Xptxas -v,-warn-spills; for both tc_conv3x3_wgrad_kernel
instantiations (3xTF32 and TF32):
  * ptxas reports 0 bytes of spill and no C75xx line (C7512: wgmma serialized for lack of registers);
  * cuobjdump -res-usage shows STACK:0 LOCAL:0, and cuobjdump -sass no CALL;
  * in the SASS, every commit group holds the MMAs of one (tap, k-step) unit -- three HGMMA for 3xTF32, one for TF32 -- with
    no WARPGROUP.DEPBAR between them, and the waits leave one group in flight (DEPBAR.LE gsb0, 0x1) except the final drain.

Runs without a GPU (nvcc cross-compiles for sm_90a); skips when nvcc or cuobjdump is absent."""
import os
import re
import subprocess

import pytest

from tests.test_engine_build import CSRC, CUOBJDUMP, NVCC, ROOT, _build_flags, _need, _ptxas_report

KERNEL = "tc_conv3x3_wgrad_kernel"
_INST = re.compile(KERNEL + r"ILi(\d)E")


@pytest.fixture(scope="module")
def wgrad_build(tmp_path_factory):
    """(ptxas log, path of the object) of tc_conv_wgrad.cu compiled with build.sh's flags and -Xptxas -v,-warn-spills."""
    _need(NVCC, CUOBJDUMP)
    obj = str(tmp_path_factory.mktemp("wgrad") / "tc_conv_wgrad.o")
    cmd = [NVCC, *_build_flags(), "-Xptxas", "-v,-warn-spills", "-c", os.path.join(CSRC, "tc_conv_wgrad.cu"), "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, cwd=ROOT, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:]
    return r.stdout, obj


def _sass_functions(obj):
    """{mangled name: [instruction text]} of cuobjdump -sass."""
    out = subprocess.run([CUOBJDUMP, "-sass", obj], check=True, capture_output=True, text=True).stdout
    funcs, cur = {}, None
    for ln in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", ln)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;", ln)
        if m and cur is not None:
            cur.append(m.group(1))
    return funcs


def test_wgrad_kernel_compiles_without_spills_or_serialized_wgmma(wgrad_build):
    log, _ = wgrad_build
    spills, serial = _ptxas_report(log)
    wgrad = {n: s for n, s in spills.items() if KERNEL in n}
    assert sorted(int(_INST.search(n).group(1)) for n in wgrad) == [1, 3], sorted(spills)
    assert not {n: s for n, s in wgrad.items() if s}, wgrad
    assert not [ln for ln in serial if KERNEL in ln], serial


def test_wgrad_kernel_uses_no_local_memory_and_no_calls(wgrad_build):
    _, obj = wgrad_build
    out = subprocess.run([CUOBJDUMP, "-res-usage", obj], check=True, capture_output=True, text=True).stdout
    usage = {n: u for n, u in re.findall(r"Function (\S+):\s*\n\s*(REG:.*)", out) if KERNEL in n}
    assert len(usage) == 2, sorted(usage)
    for n, u in usage.items():
        assert re.search(r"\bSTACK:0\b", u) and re.search(r"\bLOCAL:0\b", u), (n, u)
    funcs = {n: ins for n, ins in _sass_functions(obj).items() if KERNEL in n}
    assert len(funcs) == 2, sorted(funcs)
    for n, ins in funcs.items():
        assert not [i for i in ins if re.match(r"(@!?U?P\w+\s+)?CALL\b", i)], n


def test_wgrad_kernel_pipelines_its_commit_groups(wgrad_build):
    """A commit group ends at the HGMMA that carries gsb0.  Serialized wgmma shows up as groups of one HGMMA, each followed
    by a WARPGROUP.DEPBAR; the pipelined k-loop as groups of NSPLIT and waits that leave one group in flight."""
    _, obj = wgrad_build
    funcs = {n: ins for n, ins in _sass_functions(obj).items() if KERNEL in n}
    assert len(funcs) == 2, sorted(funcs)
    for n, ins in funcs.items():
        nsplit = int(_INST.search(n).group(1))
        sizes, run = [], 0
        for k, i in enumerate(ins):
            if not i.startswith("HGMMA"):
                continue
            run += 1
            if "gsb0" in i:
                sizes.append(run)
                run = 0
            elif k + 1 < len(ins):
                assert not ins[k + 1].startswith("WARPGROUP.DEPBAR"), (n, k, i)
        assert sizes and run == 0 and set(sizes) == {nsplit}, (n, sizes)
        waits = [i for i in ins if i.startswith("WARPGROUP.DEPBAR")]
        assert sum("gsb0, 0x1" in w for w in waits) == len(sizes), (n, waits)
        assert sum("gsb0, 0x0" in w for w in waits) == 1, (n, waits)
