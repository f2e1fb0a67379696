"""Register budget of the fused MBConv kernels (mbconv_tc, mbconv_tc_s2, dwproj_tc): compiled for sm_90a with -Xptxas -v,
no instantiation may spill, keep a stack frame, or have its wgmma serialised by ptxas.  A spill here is silent at run time
and costs up to 2x in these kernels; it is what a change of thread count or launch bounds most easily brings back."""
from __future__ import annotations

import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

import pytest

from efficientsam3_b200 import build

SOURCES = ("mbconv_tc.cu", "mbconv_tc_s2.cu", "dwproj_tc.cu")
KERNELS = ("mbconv_tc_kernel", "mbconv_tc_s2_kernel", "dwproj_tc_kernel")


def _nvcc():
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        return None
    return nvcc if shutil.which(nvcc) else None


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas")

    def compile_one(src):
        cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", str(build.CSRC / src), "-o", str(out / (src + ".o"))]
        r = subprocess.run(cmd, capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        return r.stdout + r.stderr

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        return dict(zip(SOURCES, ex.map(compile_one, SOURCES)))


def _entries(text):
    """(mangled name, stack bytes, spill store bytes, spill load bytes) per function ptxas reports properties for."""
    rows, name = [], None
    for line in text.splitlines():
        m = re.search(r"Function properties for (\w+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name is not None:
            rows.append((name, *map(int, m.groups())))
            name = None
    return rows


@pytest.mark.parametrize("src", SOURCES)
def test_fused_mbconv_kernels_do_not_spill(ptxas_report, src):
    rows = [r for r in _entries(ptxas_report[src]) if any(k in r[0] for k in KERNELS)]
    assert rows, f"{src}: no fused MBConv instantiation in the ptxas report"
    bad = [r for r in rows if r[1] or r[2] or r[3]]
    assert not bad, f"{src}: (kernel, stack, spill stores, spill loads) = {bad}"


@pytest.mark.parametrize("src", SOURCES)
def test_fused_mbconv_wgmma_not_serialised(ptxas_report, src):
    warnings = [l for l in ptxas_report[src].splitlines() if "wgmma.mma_async instructions are serialized" in l]
    assert not warnings, f"{src}: " + "\n".join(warnings)
