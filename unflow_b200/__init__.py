"""unflow_b200 -- H100-native (sm_90a) implementation of the UnFlow hot path.

Layout:
  csrc/        hand-written CUDA kernels + the C ABI (include/unflow.h) -> libunflow.so
  _native.py   ctypes binding of the C ABI (fails loudly if the library is missing)
  e2eflow/     host-side mirror of the reference's e2eflow.ops / e2eflow.core.* API on
               torch CUDA tensors (same names, argument meaning and error behaviour)

``import unflow_b200.e2eflow`` also works as ``import e2eflow`` after
``unflow_b200.install_as_e2eflow()`` so reference-style code (``from e2eflow.core.losses
import compute_losses``) runs unchanged.
"""
import sys

__all__ = ["install_as_e2eflow"]


def install_as_e2eflow():
    """Register unflow_b200.e2eflow under the reference's package name ``e2eflow``."""
    import importlib
    pkg = importlib.import_module("unflow_b200.e2eflow")
    sys.modules.setdefault("e2eflow", pkg)
    for sub in ("ops", "core", "core.flownet", "core.losses", "core.image_warp",
                "core.unsupervised", "core.util"):
        mod = importlib.import_module("unflow_b200.e2eflow." + sub)
        sys.modules.setdefault("e2eflow." + sub, mod)
    return pkg
