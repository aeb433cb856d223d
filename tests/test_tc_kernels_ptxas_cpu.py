"""The wgmma kernels of csrc/tc_conv.cu and csrc/tc_wgrad.cu must compile to a pipelined instruction stream.

ptxas reports, with -v, when it has to serialise wgmma instructions (C7517: a wait inserted because a register
a wgmma writes is used too early; C7518: the wgmma code sits on a path it cannot prove warpgroup-uniform; C7507:
a setmaxnreg it ignored) and how many bytes a kernel spills.  Either costs a large share of the tensor-core rate
while every result stays correct, so no numerical test can see it.  Compiles with the flags of
unflow_b200/build.py; no GPU needed."""
import os
import re
import shutil
import subprocess

import pytest

from unflow_b200 import build

SOURCES = ["tc_conv.cu", "tc_wgrad.cu"]
KERNELS = ["tc_conv_kernel", "tc_wgrad_kernel"]


def _nvcc():
    cand = build._nvcc()
    return cand if os.path.isabs(cand) and os.path.exists(cand) else shutil.which(cand)


@pytest.fixture(scope="module")
def ptxas_logs(tmp_path_factory):
    nvcc = _nvcc()
    if not nvcc:
        pytest.skip("nvcc not found")
    out = tmp_path_factory.mktemp("ptxas")
    procs = []
    for src in SOURCES:
        cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, src),
                                           "-o", str(out / (src + ".o"))]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    logs = {}
    for src, p in procs:
        text, _ = p.communicate()
        assert p.returncode == 0, "nvcc failed on %s:\n%s" % (src, text)
        logs[src] = text
    return logs


def _is_tc_kernel(name):
    return any(k in name for k in KERNELS)


@pytest.mark.parametrize("src", SOURCES)
def test_no_wgmma_serialisation_advisory(ptxas_logs, src):
    bad = [l for l in ptxas_logs[src].splitlines()
           if re.search(r"\(C75(17|18|07)\)", l) and (_is_tc_kernel(l) or "function" not in l)]
    assert not bad, "\n".join(bad)


@pytest.mark.parametrize("src", SOURCES)
def test_no_spills(ptxas_logs, src):
    seen = 0
    name = None
    for line in ptxas_logs[src].splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and _is_tc_kernel(name):
            seen += 1
            assert m.group(1) == "0" and m.group(2) == "0", "%s spills: %s" % (name, line.strip())
    assert seen == 3, "expected the BN = 32, 64, 128 instances of the kernel in %s, found %d" % (src, seen)
