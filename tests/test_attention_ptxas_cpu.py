"""Compiler report of the two attention kernel instances (no GPU needed): the resident (<= 640 tokens) and the
streaming (> 640 tokens) instance of attention_tc_kernel keep their registers out of local memory."""
import os
import re
import shutil
import subprocess

import pytest

from omnidata_b200 import build


def test_attention_instances_do_not_spill(tmp_path):
    nvcc = build._nvcc()
    if not ((os.path.isabs(nvcc) and os.path.exists(nvcc)) or shutil.which(nvcc)):
        pytest.skip("nvcc not found")
    cmd = [nvcc, *build.NVCC_FLAGS, "--use_fast_math", "-Xptxas", "-v", "-c", str(build.CSRC / "attention_tc.cu"),
           "-o", str(tmp_path / "attention_tc.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    found, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur is not None and "attention_tc_kernel" in cur:
            found[cur] = (int(m.group(1)), int(m.group(2)))
            cur = None
    assert any("ILb0E" in k for k in found) and any("ILb1E" in k for k in found), found
    assert all(v == (0, 0) for v in found.values()), found
