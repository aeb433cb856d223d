"""Every entry point of libunflow.so (unflow_b200/_native.SIGNATURES) in exactly one of four groups.

tests/test_gpu_step_launches.py wraps the library during one training step and checks each call of a STEP_CHECKED
entry point against float64; TC_DELEGATED calls pass through to the tensor-core shadow check of
tests/test_gpu_tc_step_launches.py; HOST_ONLY entry points launch nothing; STANDALONE entry points are not
called by the FlowNetC step and name the float64 test that covers them.  tests/test_native_entry_points_cpu.py
keeps the table complete, so a new entry point has to be placed in one of the groups.

tests/test_gpu_variant_step_launches.py runs the same check on the other configurations the project trains (FlowNetS,
the stacks, the small networks, the supervised fine-tune, other resolutions); VARIANT_CHECKED are the STANDALONE
entry points those steps call, which its checker table adds.
"""

STEP_CHECKED = (
    "unflow_correlation_fwd_bidir",
    "unflow_correlation_fold_grad",
    "unflow_correlation_bwd",
    "unflow_planar_to_interleaved",
    "unflow_interleaved_to_planar",
    "unflow_downsample",
    "unflow_level_loss_fwd",
    "unflow_level_loss_bwd",
    "unflow_conv3x3_narrow_fwd",
    "unflow_conv3x3_narrow_wgrad",
    "unflow_lrelu_bwd_bias",
    "unflow_bias_grad_lrelu",
    "unflow_bias_lrelu",
    "unflow_tc_wsplit",
    "unflow_adam_step_l2",
    "unflow_backward_warp_fwd",
)

TC_DELEGATED = (
    "unflow_tc_conv",
    "unflow_tc_wgrad",
    "unflow_tc_conv_window",
    "unflow_tc_wgrad_window",
)

HOST_ONLY = (
    "unflow_abi_version",
    "unflow_last_error",
    "unflow_launch_count",
    "unflow_reset_launch_count",
    "unflow_set_int_option",
    "unflow_tc_conv_debug",
    "unflow_correlation_out_shape",
    "unflow_correlation_workspace_bytes",
    "unflow_correlation_fwd_path",
    "unflow_level_loss_workspace_bytes",
    "unflow_supervised_loss_workspace_bytes",
    "unflow_conv3x3_narrow_wgrad_workspace_bytes",
    "unflow_tc_conv_plan",
    "unflow_tc_wgrad_plan",
    "unflow_crc32c",
)

# STANDALONE entry points that the variant steps call and tests/test_gpu_variant_step_launches.py checks in the step
VARIANT_CHECKED = (
    "unflow_correlation_fwd",
    "unflow_backward_warp_bwd",
    "unflow_supervised_loss_fwd",
    "unflow_supervised_loss_bwd",
)

# not launched by the FlowNetC step -> the float64 test that covers it ("<file>::<test>")
STANDALONE = {
    "unflow_correlation_fwd": "test_gpu_float64_kernels.py::test_correlation_generic_kernel_vs_float64",
    "unflow_backward_warp_bwd": "test_gpu_float64_kernels.py::test_warp_vs_float64",
    "unflow_forward_warp_fwd": "test_gpu_float64_kernels.py::test_forward_warp_vs_float64",
    "unflow_forward_warp_bwd": "test_gpu_float64_kernels.py::test_forward_warp_vs_float64",
    "unflow_adam_step": "test_gpu_float64_kernels.py::test_adam_entry_points_vs_float64",
    "unflow_adam_step_dev_l2": "test_gpu_float64_kernels.py::test_adam_entry_points_vs_float64",
    "unflow_adam_step_dev": "test_gpu_float64_kernels.py::test_adam_entry_points_vs_float64",
    "unflow_conv_operand_tf32": "test_gpu_conv3x.py::test_operand_kernel_exact",
    "unflow_supervised_loss_fwd": "test_gpu_supervised.py::test_kernel_vs_float64",
    "unflow_supervised_loss_bwd": "test_gpu_supervised.py::test_kernel_vs_float64",
}

# The entry points one eager FlowNetC step calls (batch 4, 384x1280, 3xTF32, default options), as observed on
# an H100.  The eager step runs Adam with host hyper-parameters (unflow_adam_step_l2); a captured step graph
# runs unflow_adam_step_dev_l2, covered by its standalone test.  test_gpu_step_launches.py asserts these sets, so
# a dispatch change that moves a launch onto another entry point fails there.
PLAIN_STEP_CALLS = frozenset((
    "unflow_adam_step_l2",
    "unflow_bias_grad_lrelu",
    "unflow_conv3x3_narrow_fwd",
    "unflow_conv3x3_narrow_wgrad",
    "unflow_conv3x3_narrow_wgrad_workspace_bytes",
    "unflow_correlation_bwd",
    "unflow_correlation_fold_grad",
    "unflow_correlation_fwd_bidir",
    "unflow_correlation_fwd_path",
    "unflow_correlation_out_shape",
    "unflow_downsample",
    "unflow_interleaved_to_planar",
    "unflow_level_loss_bwd",
    "unflow_level_loss_fwd",
    "unflow_level_loss_workspace_bytes",
    "unflow_lrelu_bwd_bias",
    "unflow_planar_to_interleaved",
    "unflow_tc_conv",
    "unflow_tc_conv_window",
    "unflow_tc_wgrad",
    "unflow_tc_wgrad_window",
    "unflow_tc_wsplit",
))
AUGMENT_STEP_CALLS = PLAIN_STEP_CALLS | {"unflow_backward_warp_fwd"}     # the BORDER_STN sampler

# The entry points one eager step of each configuration of tests/test_gpu_variant_step_launches.py calls (3xTF32,
# default options), as observed on an H100; that test asserts them as test_gpu_step_launches.py asserts the sets above.
_CORR_BIDIR = frozenset(("unflow_correlation_fwd_bidir", "unflow_correlation_fwd_path", "unflow_correlation_out_shape",
                         "unflow_interleaved_to_planar", "unflow_planar_to_interleaved"))
_CORR_BIDIR_GRAD = frozenset(("unflow_correlation_bwd", "unflow_correlation_fold_grad"))
_LEVEL_LOSS = frozenset(("unflow_downsample", "unflow_level_loss_bwd", "unflow_level_loss_fwd",
                         "unflow_level_loss_workspace_bytes"))
_FROZEN_C_STACK_CALLS = PLAIN_STEP_CALLS - _CORR_BIDIR_GRAD | {"unflow_backward_warp_fwd"}   # the stacks' image_warp
VARIANT_STEP_CALLS = {
    "C-chairs": PLAIN_STEP_CALLS,
    "C-kitti1152": PLAIN_STEP_CALLS,
    "S-synthia": PLAIN_STEP_CALLS - _CORR_BIDIR - _CORR_BIDIR_GRAD,
    "cs-cityscapes": _FROZEN_C_STACK_CALLS,
    "CSS-bench": _FROZEN_C_STACK_CALLS,
    # the supervised FlowNetC correlates one direction (unflow_correlation_fwd); train_all adds the warp gradient
    "CSS-ft-train_all": (PLAIN_STEP_CALLS - _CORR_BIDIR - _CORR_BIDIR_GRAD - _LEVEL_LOSS) | {
        "unflow_correlation_fwd", "unflow_correlation_out_shape", "unflow_correlation_bwd",
        "unflow_backward_warp_fwd", "unflow_backward_warp_bwd",
        "unflow_supervised_loss_fwd", "unflow_supervised_loss_bwd", "unflow_supervised_loss_workspace_bytes"},
}
