"""Build libunflow.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a.

The reference JIT-compiles each op with nvcc + g++ against TensorFlow headers
(reference src/e2eflow/ops.py:21-48); here one shared library holds every kernel and
is built with ``python -m unflow_b200.build`` (or ``python -m unflow_b200.e2eflow.ops``,
the reference's own "compile" entry point, ops.py:51-52).
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libunflow.so")
SOURCES = ["abi.cu", "correlation.cu", "correlation_tiled.cu", "warp.cu", "forward_warp.cu",
           "downsample.cu", "level_loss.cu", "adam.cu", "split.cu", "checksum.cu", "narrow_conv.cu", "tc_conv.cu", "tc_wgrad.cu", "relayout.cu", "narrow_conv_tma.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def sources():
    return [os.path.join(CSRC, s) for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")]
    deps.append(os.path.join(os.path.dirname(HERE), "include", "unflow.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    """Compile every .cu into unflow_b200/libunflow.so. Returns the library path."""
    if not force and not needs_build():
        return LIB
    objs = []
    env = dict(os.environ)
    env.pop("CC", None); env.pop("CXX", None)
    procs = []
    for src in sources():
        obj = src[:-3] + ".o"
        cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stdout.write(out.decode())
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s" % src)
    cmd = [_nvcc(), "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a",
                                                    "-Xcompiler", "-fPIC"]
    subprocess.check_call(cmd, env=env)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
