"""CPU restatement of the supervised fine-tuning loss (TEST INFRASTRUCTURE ONLY).

Follows /root/reference/src/e2eflow/core/supervised.py:12-65.  The photometric jitter is applied
with given draws (``photometric_draws``: the contrast / gamma / colour / noise / brightness tensors
random_photometric draws, in that order) or skipped (None).  Pinned against the reference file
itself, executed unmodified under the TensorFlow-API stand-in of tests/golden/ (loss value and
variable gradients for specs c / s / cs with train_all and cs without:
tests/test_oracle_vs_reference_supervised.py).
"""
import torch

from . import tf_compat as tfc
from .augment import photometric
from .flownet import flownet, FLOW_SCALE
from .losses import charbonnier_loss
from .unsupervised import regularization_loss


def supervised_loss(variables, batch, params, normalization=None, photometric_draws=None):
    mean = torch.tensor(normalization[0], dtype=torch.float32) / 255.0        # :13
    im1, im2, flow_gt, mask_gt = batch                                         # :14
    im1, im2 = im1 / 255.0, im2 / 255.0                                        # :15-16
    im_shape = im1.shape[1:3]
    if photometric_draws is not None:                                          # :21-26
        im1, im2 = photometric([im1, im2], *photometric_draws)
    im1, im2 = im1 - mean, im2 - mean                                          # :33-35

    train_all = params.get('train_all')
    full_res = params.get('full_res')
    flows_fw = flownet(variables, im1, im2, flownet_spec=params.get('flownet', 'S'),
                       full_resolution=full_res, train_all=train_all)          # :41-45
    if not train_all:                                                          # :47-48
        flows_fw = [flows_fw[-1]]
    final_loss = 0.0
    for i, net_flows in enumerate(reversed(flows_fw)):                         # :50-57
        flow_fw = net_flows[0]
        if full_res:
            final_flow_fw = flow_fw * FLOW_SCALE * 4
        else:
            final_flow_fw = tfc.resize_bilinear_legacy(flow_fw, im_shape) * FLOW_SCALE * 4
        final_loss = final_loss + charbonnier_loss(final_flow_fw - flow_gt, mask_gt) / (2 ** i)
    return final_loss + regularization_loss(variables)                        # :59-60
