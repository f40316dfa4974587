"""Compiler report of the wgmma kernels (no GPU needed): ptxas must keep their MMA pipelines asynchronous and their
registers out of local memory.

- C7510 ("wgmma.mma_async instructions are serialized") appears when a function call sits between wgmma issue and
  wait, e.g. a printf inlined into a K loop: every MMA then waits for its own completion.
- Spill stores / loads of `conv_gemm_kernel` (every instantiation, the 256-wide epilogues included) put local-memory
  traffic into the epilogue of every tile.
"""
import os
import re
import shutil
import subprocess

import pytest

from omnidata_b200 import build

WGMMA_SOURCES = ["conv_gemm.cu", "attention_tc.cu", "bgemm_tc.cu"]


def _nvcc():
    nvcc = build._nvcc()
    return nvcc if (os.path.isabs(nvcc) and os.path.exists(nvcc)) or shutil.which(nvcc) else None


@pytest.fixture(scope="module")
def ptxas_reports(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not found")
    out_dir = tmp_path_factory.mktemp("ptxas")
    procs = {}
    for src in WGMMA_SOURCES:
        assert src in build.FAST_MATH_SOURCES
        cmd = [nvcc, *build.NVCC_FLAGS, "--use_fast_math", "-Xptxas", "-v", "-c", str(build.CSRC / src),
               "-o", str(out_dir / (src + ".o"))]
        procs[src] = subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    reports = {}
    for src, p in procs.items():
        out, _ = p.communicate()
        assert p.returncode == 0, f"nvcc failed on {src}:\n{out}"
        reports[src] = out
    return reports


def _spills(report):
    """{mangled kernel name: (spill store bytes, spill load bytes)}"""
    res, cur = {}, None
    for line in report.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            res[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return res


@pytest.mark.parametrize("src", WGMMA_SOURCES)
def test_wgmma_not_serialized(ptxas_reports, src):
    bad = [line for line in ptxas_reports[src].splitlines() if "C7510" in line]
    assert not bad, "\n".join(bad)


def test_conv_gemm_no_spills(ptxas_reports):
    spills = {k: v for k, v in _spills(ptxas_reports["conv_gemm.cu"]).items() if "conv_gemm_kernel" in k}
    # the launchers instantiate BLOCK_N 32 / 64 / 128 / 256 with every epilogue, single CTAs and pairs
    assert len(spills) >= 40, f"expected every conv_gemm_kernel instantiation in the report, found {len(spills)}"
    assert any("ILi256E" in k for k in spills)
    bad = {k: v for k, v in spills.items() if v != (0, 0)}
    assert not bad, "spilling instantiations (store, load bytes): " + ", ".join(f"{k}: {v}" for k, v in bad.items())
