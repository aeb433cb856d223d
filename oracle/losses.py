"""CPU restatement of the reference loss module (TEST INFRASTRUCTURE ONLY).

Each function cites the lines of /root/reference/src/e2eflow/core/losses.py it
follows.  Tensors are float32 torch CPU tensors in the reference's NHWC
layout; gradients come from torch autograd exactly where TF autodiff provides
them in the reference (casts and masks carry no gradient).

Pinned by reference KATs (tests/test_oracle_reference_kats.py):
``_smoothness_deltas``, ``create_outgoing_mask``, ``gradient_loss``.
The rest (ternary_loss, compute_losses in all occlusion modes, masks, single
terms; values and gradients) is pinned against the reference file itself,
executed unmodified under the TensorFlow-API stand-in of tests/golden/
(tests/test_oracle_vs_reference_run.py).  PARITY UNPINNED below that: the
arithmetic of the TF primitives (rgb_to_grayscale, conv2d SAME), restated from
their documentation.
"""
import math

import numpy as np
import torch

from . import ops as _ops
from .image_warp import image_warp
from . import tf_compat as tfc

DISOCC_THRESH = 0.8  # losses.py:9


def length_sq(x):  # losses.py:12-13
    return torch.sum(x * x, 3, keepdim=True)


def compute_losses(im1, im2, flow_fw, flow_bw, border_mask=None, mask_occlusion='',
                   data_max_distance=1):  # losses.py:16-87
    losses = {}

    im2_warped = image_warp(im2, flow_fw)
    im1_warped = image_warp(im1, flow_bw)
    im_diff_fw = im1 - im2_warped
    im_diff_bw = im2 - im1_warped

    disocc_fw = (_ops.forward_warp(flow_fw) < DISOCC_THRESH).float()
    disocc_bw = (_ops.forward_warp(flow_bw) < DISOCC_THRESH).float()

    if border_mask is None:
        mask_fw = create_outgoing_mask(flow_fw)
        mask_bw = create_outgoing_mask(flow_bw)
    else:
        mask_fw = border_mask
        mask_bw = border_mask

    flow_bw_warped = image_warp(flow_bw, flow_fw)
    flow_fw_warped = image_warp(flow_fw, flow_bw)
    flow_diff_fw = flow_fw + flow_bw_warped
    flow_diff_bw = flow_bw + flow_fw_warped

    mag_sq_fw = length_sq(flow_fw) + length_sq(flow_bw_warped)
    mag_sq_bw = length_sq(flow_bw) + length_sq(flow_fw_warped)
    occ_thresh_fw = 0.01 * mag_sq_fw + 0.5
    occ_thresh_bw = 0.01 * mag_sq_bw + 0.5

    fb_occ_fw = (length_sq(flow_diff_fw) > occ_thresh_fw).float()
    fb_occ_bw = (length_sq(flow_diff_bw) > occ_thresh_bw).float()

    if mask_occlusion == 'fb':
        mask_fw = mask_fw * (1 - fb_occ_fw)
        mask_bw = mask_bw * (1 - fb_occ_bw)
    elif mask_occlusion == 'disocc':
        mask_fw = mask_fw * (1 - disocc_bw)
        mask_bw = mask_bw * (1 - disocc_fw)

    occ_fw = 1 - mask_fw
    occ_bw = 1 - mask_bw

    losses['sym'] = charbonnier_loss(occ_fw - disocc_bw) + charbonnier_loss(occ_bw - disocc_fw)
    losses['occ'] = charbonnier_loss(occ_fw) + charbonnier_loss(occ_bw)
    losses['photo'] = photometric_loss(im_diff_fw, mask_fw) + photometric_loss(im_diff_bw, mask_bw)
    losses['grad'] = gradient_loss(im1, im2_warped, mask_fw) + gradient_loss(im2, im1_warped, mask_bw)
    losses['smooth_1st'] = smoothness_loss(flow_fw) + smoothness_loss(flow_bw)
    losses['smooth_2nd'] = second_order_loss(flow_fw) + second_order_loss(flow_bw)
    losses['fb'] = charbonnier_loss(flow_diff_fw, mask_fw) + charbonnier_loss(flow_diff_bw, mask_bw)
    losses['ternary'] = (ternary_loss(im1, im2_warped, mask_fw, max_distance=data_max_distance) +
                         ternary_loss(im2, im1_warped, mask_bw, max_distance=data_max_distance))
    # auxiliary tensors for mask-parity tests (not part of the reference return value)
    losses['_aux'] = dict(mask_fw=mask_fw, mask_bw=mask_bw, fb_occ_fw=fb_occ_fw, fb_occ_bw=fb_occ_bw,
                          disocc_fw=disocc_fw, disocc_bw=disocc_bw,
                          im2_warped=im2_warped, im1_warped=im1_warped,
                          flow_diff_fw=flow_diff_fw, flow_diff_bw=flow_diff_bw)
    return losses


def ternary_transform(image, max_distance):  # losses.py:93-108
    patch_size = 2 * max_distance + 1
    intensities = tfc.rgb_to_grayscale(image) * 255
    out_channels = patch_size * patch_size
    w = np.eye(out_channels).reshape((patch_size, patch_size, 1, out_channels))
    weights = torch.tensor(w, dtype=torch.float32)
    patches = tfc.conv2d_same_nhwc(intensities, weights)
    transf = patches - intensities
    return transf / torch.sqrt(0.81 + transf * transf)


def hamming_distance(t1, t2):  # losses.py:110-114
    dist = (t1 - t2) ** 2
    dist_norm = dist / (0.1 + dist)
    return torch.sum(dist_norm, 3, keepdim=True)


def ternary_loss(im1, im2_warped, mask, max_distance=1):  # losses.py:90-122
    t1 = ternary_transform(im1, max_distance)
    t2 = ternary_transform(im2_warped, max_distance)
    dist = hamming_distance(t1, t2)
    transform_mask = create_mask(mask, [[max_distance, max_distance],
                                        [max_distance, max_distance]])
    return charbonnier_loss(dist, mask * transform_mask)


def occlusion(flow_fw, flow_bw):  # losses.py:125-134 (note: unwarped |f_bw|^2 in the threshold)
    mag_sq = length_sq(flow_fw) + length_sq(flow_bw)
    flow_bw_warped = image_warp(flow_bw, flow_fw)
    flow_fw_warped = image_warp(flow_fw, flow_bw)
    flow_diff_fw = flow_fw + flow_bw_warped
    flow_diff_bw = flow_bw + flow_fw_warped
    occ_thresh = 0.01 * mag_sq + 0.5
    occ_fw = (length_sq(flow_diff_fw) > occ_thresh).float()
    occ_bw = (length_sq(flow_diff_bw) > occ_thresh).float()
    return occ_fw, occ_bw


def _const_filter(arr):
    return torch.tensor(np.asarray(arr), dtype=torch.float32)


def divergence(flow):  # losses.py:148-162
    filter_x = np.array([[-1, 0, 1], [-2, 0, 2], [-1, 0, 1]], dtype=np.float64)
    filter_y = filter_x.T
    wx = np.zeros([3, 3, 1, 1]); wx[:, :, 0, 0] = filter_x
    wy = np.zeros([3, 3, 1, 1]); wy[:, :, 0, 0] = filter_y
    flow_u, flow_v = flow[..., 0:1], flow[..., 1:2]
    grad_x = conv2d(flow_u, _const_filter(wx))
    grad_y = conv2d(flow_v, _const_filter(wy))
    return torch.sum(torch.cat([grad_x, grad_y], 3), 3, keepdim=True)


def norm(x, sigma):  # losses.py:165-170: N(0,sigma).pdf(x) / N(0,sigma).pdf(0)
    return torch.exp(-0.5 * (x / sigma) ** 2)


def photometric_loss(im_diff, mask):  # losses.py:198-199
    return charbonnier_loss(im_diff, mask, beta=255)


def conv2d(x, weights):  # losses.py:202-203
    return tfc.conv2d_same_nhwc(x, weights)


def _smoothness_deltas(flow):  # losses.py:206-222
    mask_x = create_mask(flow, [[0, 0], [0, 1]])
    mask_y = create_mask(flow, [[0, 1], [0, 0]])
    mask = torch.cat([mask_x, mask_y], 3)
    filter_x = [[0, 0, 0], [0, 1, -1], [0, 0, 0]]
    filter_y = [[0, 0, 0], [0, 1, 0], [0, -1, 0]]
    w = np.ones([3, 3, 1, 2])
    w[:, :, 0, 0] = filter_x
    w[:, :, 0, 1] = filter_y
    weights = _const_filter(w)
    flow_u, flow_v = flow[..., 0:1], flow[..., 1:2]
    return conv2d(flow_u, weights), conv2d(flow_v, weights), mask


def _gradient_delta(im1, im2_warped):  # losses.py:225-237
    filter_x = np.array([[-1, 0, 1], [-2, 0, 2], [-1, 0, 1]], dtype=np.float64)
    filter_y = filter_x.T
    w = np.zeros([3, 3, 3, 6])
    for c in range(3):
        w[:, :, c, 2 * c] = filter_x
        w[:, :, c, 2 * c + 1] = filter_y
    weights = _const_filter(w)
    return conv2d(im1, weights) - conv2d(im2_warped, weights)


def gradient_loss(im1, im2_warped, mask):  # losses.py:240-247
    mask_x = create_mask(im1, [[0, 0], [1, 1]])
    mask_y = create_mask(im1, [[1, 1], [0, 0]])
    gradient_mask = torch.cat([mask_x, mask_y], 3).repeat(1, 1, 1, 3)
    diff = _gradient_delta(im1, im2_warped)
    return charbonnier_loss(diff, mask * gradient_mask)


def smoothness_loss(flow):  # losses.py:250-255
    delta_u, delta_v, mask = _smoothness_deltas(flow)
    return charbonnier_loss(delta_u, mask) + charbonnier_loss(delta_v, mask)


def _second_order_deltas(flow):  # losses.py:258-287
    mask_x = create_mask(flow, [[0, 0], [1, 1]])
    mask_y = create_mask(flow, [[1, 1], [0, 0]])
    mask_diag = create_mask(flow, [[1, 1], [1, 1]])
    mask = torch.cat([mask_x, mask_y, mask_diag, mask_diag], 3)
    filter_x = [[0, 0, 0], [1, -2, 1], [0, 0, 0]]
    filter_y = [[0, 1, 0], [0, -2, 0], [0, 1, 0]]
    filter_diag1 = [[1, 0, 0], [0, -2, 0], [0, 0, 1]]
    filter_diag2 = [[0, 0, 1], [0, -2, 0], [1, 0, 0]]
    w = np.ones([3, 3, 1, 4])
    w[:, :, 0, 0] = filter_x
    w[:, :, 0, 1] = filter_y
    w[:, :, 0, 2] = filter_diag1
    w[:, :, 0, 3] = filter_diag2
    weights = _const_filter(w)
    flow_u, flow_v = flow[..., 0:1], flow[..., 1:2]
    return conv2d(flow_u, weights), conv2d(flow_v, weights), mask


def second_order_loss(flow):  # losses.py:290-295
    delta_u, delta_v, mask = _second_order_deltas(flow)
    return charbonnier_loss(delta_u, mask) + charbonnier_loss(delta_v, mask)


def charbonnier_loss(x, mask=None, truncate=None, alpha=0.45, beta=1.0, epsilon=0.001):
    """losses.py:298-322: sum(mask * ((x*beta)^2 + eps^2)^alpha) / numel(x)."""
    normalization = float(x.numel())
    error = torch.pow((x * beta) ** 2 + epsilon ** 2, alpha)
    if mask is not None:
        error = mask * error
    if truncate is not None:
        error = torch.clamp(error, max=truncate)
    return torch.sum(error) / normalization


def create_mask(tensor, paddings):  # losses.py:325-335
    B, H, W = tensor.shape[0], tensor.shape[1], tensor.shape[2]
    inner_h = H - (paddings[0][0] + paddings[0][1])
    inner_w = W - (paddings[1][0] + paddings[1][1])
    inner = torch.ones(max(inner_h, 0), max(inner_w, 0))
    mask2d = torch.nn.functional.pad(inner, (paddings[1][0], paddings[1][1],
                                             paddings[0][0], paddings[0][1]))
    return mask2d.view(1, H, W, 1).repeat(B, 1, 1, 1).to(tensor.device)


def create_border_mask(tensor, border_ratio=0.1):  # losses.py:338-344
    H, W = tensor.shape[1], tensor.shape[2]
    min_dim = np.float32(min(H, W))
    sz = int(math.ceil(np.float32(min_dim * np.float32(border_ratio))))
    return create_mask(tensor, [[sz, sz], [sz, sz]])


def create_outgoing_mask(flow):  # losses.py:347-366
    B, H, W, _ = flow.shape
    grid_x = torch.arange(W, dtype=torch.float32).view(1, 1, W)
    grid_y = torch.arange(H, dtype=torch.float32).view(1, H, 1)
    pos_x = grid_x + flow[..., 0]
    pos_y = grid_y + flow[..., 1]
    inside_x = (pos_x <= float(W - 1)) & (pos_x >= 0.0)
    inside_y = (pos_y <= float(H - 1)) & (pos_y >= 0.0)
    return (inside_x & inside_y).float().unsqueeze(3)
