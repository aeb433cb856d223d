"""csrc/conv_fma.cu must compile without spills or other local memory: the kernel keeps FMA_PIX positions x 4
channels of accumulators and the positions' input loads in registers, and a spill would put every FMA chain behind
local-memory traffic while every result stays correct.  Compiles with the flags of unflow_b200/build.py; no GPU
needed."""
import os
import re
import subprocess

import pytest

from unflow_b200 import build
from test_tc_kernels_ptxas_cpu import _nvcc


def test_conv_fma_kernels_use_no_local_memory(tmp_path):
    nvcc = _nvcc()
    if not nvcc:
        pytest.skip("nvcc not found")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "conv_fma.cu"),
                                       "-o", str(tmp_path / "conv_fma.o")]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout
    seen, name = 0, None
    for line in p.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and "conv_fma_kernel" in name:
            seen += 1
            assert m.groups() == ("0", "0", "0"), "%s: %s" % (name, line.strip())
        m = re.search(r"(\d+) bytes lmem", line)
        assert not (m and int(m.group(1))), line.strip()
    assert seen == 4, "expected the Cin = 1..4 instances of conv_fma_kernel, found %d" % seen
