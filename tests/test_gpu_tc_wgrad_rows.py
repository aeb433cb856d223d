"""Weight gradients whose 128-row blocks are partly or wholly past R, against float64.

tc_wgrad_kernel gives each 128-row block of dW to two consumer warpgroups of 64 rows; a warpgroup whose rows all
lie at or past R issues no MMAs and writes nothing, but still splits its half of the G tile, which the other
warpgroup reads.  The cases: the first layer's row-window form (R = 64: every tile has an idle warpgroup), the
R = 2 flow-upsampling deconvolutions, and conv layers whose last row block keeps 2, 63 or 64 rows.  Same bound as
the step test: |got - ref| <= TAU * A elementwise, A the same float64 operation on |operands|.
"""
import ctypes

import pytest
import torch

from test_gpu_tc_step_launches import TAU, ref_wgrad, ref_wgrad_window, worst_ratio

pytestmark = pytest.mark.gpu


def _uniform(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(shape, generator=g) * 2 - 1


def _nhwc(N, C, H, W, seed):
    """[N, C, H, W] with NHWC memory, a channel slice of a buffer whose pitch is C rounded up to 4."""
    from unflow_b200.e2eflow.core import tc_conv
    t = tc_conv.empty_nhwc(N, tc_conv.round4(C), H, W, "cuda")[:, :C]
    t.copy_(_uniform((N, C, H, W), seed))
    return t


def _plan(N, Hp, Wp, R, C, stride, kh, kw, pad_t, pad_l):
    from unflow_b200 import _native
    v = (ctypes.c_int * 15)()
    assert _native.lib().unflow_tc_wgrad_plan(N, Hp, Wp, R, C, stride, kh, kw, pad_t, pad_l, v) == 15
    return dict(r_blocks=v[9], BN=v[11], n_chunks=v[8])


@pytest.mark.parametrize("R, C, stride, k, pad, H, W", [
    (130, 64, 1, 3, 1, 24, 40),       # last row block: 2 rows
    (191, 96, 1, 3, 1, 20, 36),       # 63 rows
    (192, 64, 2, 5, 2, 16, 30),       # 64 rows: the second warpgroup of that block is idle
    (2, 2, 2, 4, 1, 24, 40),          # flow upsampling: R = 2 (deconv weight gradient form)
    (2, 64, 1, 3, 1, 12, 20),
])
def test_weight_gradient_rows_past_R(R, C, stride, k, pad, H, W):
    from unflow_b200.e2eflow.core import tc_conv
    N = 2
    Hg, Wg = stride * H, stride * W
    P, G = _nhwc(N, R, H, W, seed=R + C), _nhwc(N, C, Hg, Wg, seed=R * C + 1)
    plan = _plan(N, H, W, R, C, stride, k, k, pad, pad)
    assert R - 128 * (plan["r_blocks"] - 1) <= 64          # the last block's second warpgroup is idle
    dw = torch.zeros((R, k, k, C), device="cuda").permute(0, 3, 1, 2)
    tc_conv.wgrad(P, G, dw, stride=stride, kh=k, kw=k, pad_t=pad, pad_l=pad)
    torch.cuda.synchronize()
    P64, G64 = P.double(), G.double()
    ref = ref_wgrad(P64, G64, stride, k, k, pad, pad)
    A = ref_wgrad(P64.abs(), G64.abs(), stride, k, k, pad, pad)
    ratio = worst_ratio(dw, ref, A)
    print("R %d C %d plan %s: worst |err|/A %.3e" % (R, C, plan, ratio))
    assert ratio <= TAU


@pytest.mark.parametrize("Cp, stride, kh", [(4, 2, 7), (8, 1, 3)])
def test_row_window_weight_gradient_R64(Cp, stride, kh):
    from unflow_b200.e2eflow.core import tc_conv
    N, R, Ho, Wo, H = 2, 64, 20, 36, 40
    pad_t = kh // 2
    Wp = stride * (Wo - 1) + 8
    P = _nhwc(N, R, Ho, Wo, seed=11)
    xp = _uniform((N, H, Wp, Cp), seed=12).cuda().contiguous()
    plan = _plan(N, Ho, Wo, R, 8 * Cp, stride, kh, 1, pad_t, 0)
    assert plan["r_blocks"] == 1
    dw = torch.zeros((R, kh, 1, 8 * Cp), device="cuda").permute(0, 3, 1, 2)
    tc_conv.wgrad_window(P, xp, dw, kh=kh, stride=stride, pad_t=pad_t)
    torch.cuda.synchronize()
    P64, x64 = P.double(), xp.double()
    ref = ref_wgrad_window(P64, x64, stride, kh, pad_t)
    A = ref_wgrad_window(P64.abs(), x64.abs(), stride, kh, pad_t)
    ratio = worst_ratio(dw, ref, A)
    print("window Cp %d plan %s: worst |err|/A %.3e" % (Cp, plan, ratio))
    assert ratio <= TAU
