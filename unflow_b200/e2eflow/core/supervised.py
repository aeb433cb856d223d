"""The supervised fine-tuning objective with the reference's signature
(/root/reference/src/e2eflow/core/supervised.py:12-65):

    supervised_loss(batch, params, normalization=None, augment=True, variables=None)

``batch = (im1, im2, flow_gt, mask_gt)``: NHWC images in [0, 255], the ground-truth flow in pixels
[B,H,W,2] and its 0/1 validity mask [B,H,W,1] (KITTI's flow_occ, kitti/input.py:82-146).  Both
frames get the photometric jitter (``augment=False`` skips it; the reference always applies it),
the network predicts the forward flow only, and every scored network adds
``charbonnier_loss(resize_bilinear(flow2, [H, W]) * FLOW_SCALE * 4 - flow_gt, mask_gt) / 2**i``
(i = 0 for the last network; only the last one unless ``train_all``).

On CUDA float32 inputs each network's term is one forward and one backward launch of
csrc/supervised_loss.cu (the upsampled flow is never materialised); otherwise the same expression
runs unfused from ``charbonnier_loss`` and ``tf_image.resize_bilinear``.
"""
import torch

from ... import _native
from ..._native import check
from . import tf_image
from .flownet import FLOW_SCALE, flownet, get_variables
from .losses import charbonnier_loss
from .unsupervised import _device_constant, _track_loss


def fused_available(flow, flow_gt):
    """Can the fused kernel serve this term?  (CUDA float32 flows.)"""
    return all(torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 for t in (flow, flow_gt))


class _SupervisedLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, flow, flow_gt, mask_gt, scale):
        from ..ops import _stream, kernel_timer
        B, h, w, _ = flow.shape
        H, W = flow_gt.shape[1], flow_gt.shape[2]
        dev = flow.device
        lib = _native.lib()
        loss = torch.empty(1, device=dev, dtype=torch.float32)
        ws = torch.empty(int(lib.unflow_supervised_loss_workspace_bytes(B, H, W)), device=dev, dtype=torch.uint8)
        nbytes = 4 * B * H * W * (3 if mask_gt is not None else 2) + 8 * B * h * w
        with torch.cuda.device(dev), kernel_timer.span("supervised_loss_fwd_%dx%d" % (H, W), nbytes):
            check(lib.unflow_supervised_loss_fwd(
                flow.data_ptr(), flow_gt.data_ptr(), mask_gt.data_ptr() if mask_gt is not None else None,
                loss.data_ptr(), ws.data_ptr(), B, h, w, H, W, float(scale), _stream()), "supervised_loss")
        ctx.save_for_backward(flow, flow_gt, mask_gt)
        ctx.scale = float(scale)
        return loss.view(())

    @staticmethod
    def backward(ctx, grad_loss):
        from ..ops import _stream, kernel_timer
        flow, flow_gt, mask_gt = ctx.saved_tensors
        B, h, w, _ = flow.shape
        H, W = flow_gt.shape[1], flow_gt.shape[2]
        grad_loss = grad_loss.reshape(1).contiguous().float()
        dflow = torch.empty_like(flow)
        nbytes = 4 * B * H * W * (3 if mask_gt is not None else 2) + 16 * B * h * w
        with torch.cuda.device(flow.device), kernel_timer.span("supervised_loss_bwd_%dx%d" % (H, W), nbytes):
            check(_native.lib().unflow_supervised_loss_bwd(
                grad_loss.data_ptr(), flow.data_ptr(), flow_gt.data_ptr(),
                mask_gt.data_ptr() if mask_gt is not None else None, dflow.data_ptr(),
                B, h, w, H, W, ctx.scale, _stream()), "supervised_loss_grad")
        return dflow, None, None, None


def flow_loss(flow, flow_gt, mask_gt=None, scale=FLOW_SCALE * 4, fused=None):
    """``charbonnier_loss(resize_bilinear(flow, gt size) * scale - flow_gt, mask_gt)``; the resize is
    skipped when the sizes already agree (the ``full_res`` networks, supervised.py:51-52).
    ``fused``: force (True) / forbid (False) the CUDA kernel; None = use it on CUDA float32 inputs."""
    use_fused = fused_available(flow, flow_gt) if fused is None else fused
    if use_fused:
        from ..ops import _prep
        B, H, W = flow_gt.shape[0], flow_gt.shape[1], flow_gt.shape[2]
        flow = _prep(flow, "flow")
        flow_gt = _prep(flow_gt.detach(), "flow_gt")
        if flow.shape[0] != B or flow.shape[3] != 2 or flow_gt.shape[3] != 2:
            raise ValueError("supervised_loss: flow [B,h,w,2] and flow_gt [B,H,W,2] expected")
        if mask_gt is not None:
            mask_gt = _prep(mask_gt.detach(), "mask_gt")
            if tuple(mask_gt.shape) != (B, H, W, 1):
                raise ValueError("supervised_loss: mask_gt must be [B,H,W,1]")
        return _SupervisedLoss.apply(flow, flow_gt, mask_gt, float(scale))
    size = flow_gt.shape[1:3]
    if tuple(flow.shape[1:3]) == tuple(size):
        final = flow * scale
    else:
        final = tf_image.resize_bilinear(flow, size) * scale
    return charbonnier_loss(final - flow_gt, mask_gt)


def supervised_loss(batch, params, normalization=None, augment=True, variables=None):
    im1, im2, flow_gt, mask_gt = batch
    im1 = im1 / 255.0
    im2 = im2 / 255.0
    mean = _device_constant([m / 255.0 for m in normalization[0]], im1.device)

    if augment:
        from .augment import random_photometric
        im1_photo, im2_photo = random_photometric(
            [im1, im2], noise_stddev=0.04, min_contrast=-0.3, max_contrast=0.3,
            brightness_stddev=0.02, min_colour=0.9, max_colour=1.1, min_gamma=0.7, max_gamma=1.5)
    else:
        im1_photo, im2_photo = im1, im2

    spec = params.get('flownet', 'S')
    full_res = params.get('full_res')
    train_all = params.get('train_all')
    if variables is None:
        variables = get_variables(spec, full_res, device=im1.device)
    flows_fw = flownet(im1_photo - mean, im2_photo - mean, flownet_spec=spec,
                       full_resolution=full_res, train_all=train_all, variables=variables)
    if not train_all:
        flows_fw = [flows_fw[-1]]

    final_loss = 0.0
    for i, net_flows in enumerate(reversed(flows_fw)):
        # the last network of a full_res stack predicts at full resolution: a ratio-1 "resize"
        net_loss = flow_loss(net_flows[0], flow_gt, mask_gt, scale=FLOW_SCALE * 4)
        final_loss = final_loss + net_loss / (2 ** i)

    regularization_loss = variables.regularization_loss()
    final_loss = final_loss + regularization_loss
    _track_loss(regularization_loss, 'loss/regularization')
    _track_loss(final_loss, 'loss/combined')
    return final_loss
