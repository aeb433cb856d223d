"""ctypes binding of libunflow.so (the C ABI in include/unflow.h).

There is deliberately NO fallback: if the library is missing or an entry point fails the
caller gets an exception (``NativeLibraryError`` / ``ValueError`` / ``RuntimeError``), never a
silently different code path.  Mirrors the role of ``tf.load_op_library`` in the reference
(src/e2eflow/ops.py:56-63).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libunflow.so")

UNFLOW_OK, UNFLOW_EINVAL, UNFLOW_ECUDA = 0, 1, 2
BORDER_ZERO, BORDER_CLAMP = 0, 1


class NativeLibraryError(RuntimeError):
    pass


_lib = None
_vp = ctypes.c_void_p
_i = ctypes.c_int

# name -> (restype, argtypes); every symbol include/unflow.h declares
SIGNATURES = {
    "unflow_abi_version": (_i, []),
    "unflow_last_error": (ctypes.c_char_p, []),
    "unflow_launch_count": (ctypes.c_ulonglong, []),
    "unflow_reset_launch_count": (None, []),
    "unflow_set_int_option": (_i, [ctypes.c_char_p, _i]),
    "unflow_correlation_out_shape": (_i, [_i] * 7 + [ctypes.POINTER(_i)] * 3),
    "unflow_correlation_workspace_bytes": (ctypes.c_size_t, [_i] * 9),
    "unflow_correlation_fwd": (_i, [_vp, _vp, _vp] + [_i] * 9 + [_vp]),
    "unflow_correlation_bwd": (_i, [_vp] * 5 + [_i] * 9 + [_vp]),
    "unflow_correlation_fwd_path": (_i, [_i] * 8),
    "unflow_correlation_fwd_bidir": (_i, [_vp] * 4 + [_i] * 9 + [_vp]),
    "unflow_correlation_fold_grad": (_i, [_vp] * 3 + [_i] * 9 + [_vp]),
    "unflow_tc_conv_debug": (_i, [_vp]),
    "unflow_planar_to_interleaved": (_i, [_vp, ctypes.c_longlong, _vp, ctypes.c_longlong, ctypes.c_longlong] +
                                     [_i] * 4 + [_vp]),
    "unflow_interleaved_to_planar": (_i, [_vp, ctypes.c_longlong, ctypes.c_longlong, _vp, ctypes.c_longlong] +
                                     [_i] * 3 + [_vp]),
    "unflow_backward_warp_fwd": (_i, [_vp] * 3 + [_i] * 5 + [_vp]),
    "unflow_backward_warp_bwd": (_i, [_vp] * 5 + [_i] * 5 + [_vp]),
    "unflow_forward_warp_fwd": (_i, [_vp] * 2 + [_i] * 3 + [_vp]),
    "unflow_forward_warp_bwd": (_i, [_vp] * 3 + [_i] * 3 + [_vp]),
    "unflow_downsample": (_i, [_vp] * 2 + [_i] * 5 + [_vp]),
    "unflow_conv_operand_tf32": (_i, [_vp, _vp] + [_i] * 4 + [ctypes.c_longlong] * 4 + [_i] * 8 +
                                 [_vp, ctypes.c_float, _vp]),
    "unflow_bias_lrelu": (_i, [_vp, _vp, ctypes.c_longlong, _i, ctypes.c_float, _vp]),
    "unflow_bias_grad_lrelu": (_i, [_vp] + [ctypes.c_longlong] * 4 + [_vp, _vp] + [_i] * 4 +
                               [ctypes.c_float, _vp]),
    "unflow_lrelu_bwd_bias": (_i, [_vp] + [ctypes.c_longlong] * 4 + [_vp, ctypes.c_longlong, _vp, ctypes.c_longlong, _vp] + [_i] * 4 +
                              [ctypes.c_float, _vp]),
    "unflow_adam_step": (_i, [_vp] * 4 + [ctypes.c_longlong] + [ctypes.c_float] * 4 +
                         [ctypes.c_longlong, ctypes.c_float, _i, _vp]),
    "unflow_adam_step_dev": (_i, [_vp] * 4 + [ctypes.c_longlong, _vp, _i, _vp]),
    "unflow_adam_step_l2": (_i, [_vp] * 4 + [ctypes.c_longlong] + [ctypes.c_float] * 4 +
                            [ctypes.c_longlong, ctypes.c_float, _i, _vp, ctypes.c_float, _vp]),
    "unflow_adam_step_dev_l2": (_i, [_vp] * 4 + [ctypes.c_longlong, _vp, _i, _vp, ctypes.c_float, _vp]),
    "unflow_level_loss_workspace_bytes": (ctypes.c_size_t, [_i] * 3),
    "unflow_level_loss_fwd": (_i, [_vp] * 11 + [_i] * 5 + [ctypes.c_uint, _vp]),
    "unflow_level_loss_bwd": (_i, [_vp] * 11 + [_i] * 5 + [ctypes.c_uint, _vp]),
    "unflow_supervised_loss_workspace_bytes": (ctypes.c_size_t, [_i] * 3),
    "unflow_supervised_loss_fwd": (_i, [_vp] * 5 + [_i] * 5 + [ctypes.c_float, _vp]),
    "unflow_supervised_loss_bwd": (_i, [_vp] * 5 + [_i] * 5 + [ctypes.c_float, _vp]),
    "unflow_conv3x3_narrow_fwd": (_i, [_vp, ctypes.c_longlong] + [_vp] * 3 + [ctypes.c_longlong] + [_i] * 5 + [_vp]),
    "unflow_conv3x3_narrow_wgrad_workspace_bytes": (ctypes.c_size_t, [_i] * 4),
    "unflow_conv3x3_narrow_wgrad": (_i, [_vp, ctypes.c_longlong, _vp] + [ctypes.c_longlong] * 4 + [_vp, _vp] + [_i] * 5 + [_vp]),
    "unflow_crc32c": (ctypes.c_uint, [_vp, ctypes.c_size_t, ctypes.c_uint]),
    "unflow_tc_wsplit": (_i, [_vp, _vp, _vp, _i, _i, _i] + [ctypes.c_longlong] * 3 + [_vp]),
    "unflow_tc_conv_plan": (_i, [_i] * 13 + [ctypes.POINTER(_i), _i]),
    "unflow_tc_wgrad_plan": (_i, [_i] * 10 + [ctypes.POINTER(_i)]),
    "unflow_tc_wgrad": (_i, [_vp, _i, _i, _i, _i, ctypes.c_longlong, _vp, _i, _i, _i, ctypes.c_longlong, _vp,
                             ctypes.c_longlong, ctypes.c_longlong] + [_i] * 5 + [_vp]),
    "unflow_tc_conv_window": (_i, [_vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _i, _i, ctypes.c_longlong, _vp,
                                   ctypes.c_float, _i, _i, _i, _i, _vp]),
    "unflow_tc_wgrad_window": (_i, [_vp, _i, _i, _i, _i, ctypes.c_longlong, _vp, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "unflow_tc_conv": (_i, [_vp, _i, _i, _i, _i, ctypes.c_longlong, _vp, _vp, _vp, _i, _i, _i,
                            ctypes.c_longlong, _vp, ctypes.c_float, _i, _i] + [_i] * 6 + [_vp]),
}


def lib():
    """Load libunflow.so once.  Raises NativeLibraryError when it is absent or incomplete."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            "%s not found: build it with `python -m unflow_b200.build` (nvcc, sm_90a). "
            "There is no CPU / PyTorch fallback for the UnFlow ops." % LIB_PATH)
    try:
        handle = ctypes.CDLL(LIB_PATH)
    except OSError as e:
        raise NativeLibraryError("cannot load %s: %s" % (LIB_PATH, e))
    for name, (restype, argtypes) in SIGNATURES.items():
        try:
            fn = getattr(handle, name)
        except AttributeError:
            raise NativeLibraryError("%s does not export %s (stale build?)" % (LIB_PATH, name))
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = handle
    return _lib


def last_error():
    return lib().unflow_last_error().decode("utf-8", "replace")


def check(rc, what):
    """Map the C-ABI return code onto the reference's error behaviour: invalid arguments raise
    ValueError (TF: InvalidArgumentError), CUDA failures RuntimeError."""
    if rc == UNFLOW_OK:
        return
    msg = "%s: %s" % (what, last_error())
    if rc == UNFLOW_EINVAL:
        raise ValueError(msg)
    raise RuntimeError(msg)


def launch_count():
    return int(lib().unflow_launch_count())


def reset_launch_count():
    lib().unflow_reset_launch_count()
