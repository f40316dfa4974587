"""Compiler report of the fp8 mode's kernels (no GPU needed): the e4m3 instances of conv_gemm_kernel, every
conv_gemm_kernel instance beside them, the e4m3-output LayerNorm and the row-quantise kernel keep their registers out
of local memory, and no wgmma is serialised (ptxas C7510)."""
import os
import re
import shutil
import subprocess

import pytest

from omnidata_b200 import build


def _ptxas_report(src, tmp_path):
    nvcc = build._nvcc()
    if not ((os.path.isabs(nvcc) and os.path.exists(nvcc)) or shutil.which(nvcc)):
        pytest.skip("nvcc not found")
    cmd = [nvcc, *build.NVCC_FLAGS, "--use_fast_math", "-Xptxas", "-v", "-c", str(build.CSRC / src),
           "-o", str(tmp_path / (src + ".o"))]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    found, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None:
            found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    return r.stdout, found


def test_conv_gemm_instances_do_not_spill_or_serialise(tmp_path):
    out, found = _ptxas_report("conv_gemm.cu", tmp_path)
    gemm = {k: v for k, v in found.items() if "conv_gemm_kernel" in k}
    fp8 = [k for k in gemm if "ELb1EEEv" in k]     # the FP8 = true instances (last template argument)
    assert len(fp8) == 8, sorted(gemm)
    assert all(v == (0, 0) for v in gemm.values()), {k: v for k, v in gemm.items() if v != (0, 0)}
    assert "C7510" not in out


def test_e4m3_quantisers_do_not_spill(tmp_path):
    _, found = _ptxas_report("ops.cu", tmp_path)
    q = {k: v for k, v in found.items() if "rowquant_e4m3_kernel" in k or ("layernorm_kernel" in k and "e4m3" in k)}
    assert len(q) == 4 + 8, sorted(q)            # rowquant at 4 widths, LayerNorm at 4 widths x 2 input types
    assert all(v == (0, 0) for v in q.values()), q
