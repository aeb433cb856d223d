"""Seeded synthetic image pairs, flows and the KITTI parameter set (SURVEY.md section 8d); used by
bench.py, run.py --synthetic and the parity tests (there is no network for datasets)."""
import torch
import torch.nn.functional as F

KITTI_NORMALIZATION = ([104.920005, 110.1753, 114.785955], 1 / 0.0039216)  # core/input.py:45-46

# config_template/config.ini [train] + [train_kitti] (:166-174)
KITTI_PARAMS = dict(flownet='C', pyramid_loss=True, border_mask=True, ternary_weight=1.0,
                    smooth_2nd_weight=3.0, fb_weight=0.2, mask_occlusion='fb', occ_weight=12.4)


def _box3(x):
    k = torch.ones(x.shape[1], 1, 3, 3) / 9.0
    return F.conv2d(F.pad(x, (1, 1, 1, 1), mode='replicate'), k, groups=x.shape[1])


def image_pair(B, H, W, seed=1234, max_flow=8.0):
    """im1 ~ smoothed U{0..255}; im2 = im1 shifted by a smooth flow (|f| <= max_flow) + N(0,2)
    noise, clipped to [0,255].  Returns float32 NHWC CPU tensors (im1, im2, flow)."""
    g = torch.Generator().manual_seed(seed)
    im1 = torch.randint(0, 256, (B, 3, H, W), generator=g).float()
    im1 = _box3(_box3(im1))
    coarse = (torch.rand(B, 2, max(H // 32, 2), max(W // 32, 2), generator=g) * 2 - 1) * max_flow
    flow = F.interpolate(coarse, size=(H, W), mode='bilinear', align_corners=True)
    ys, xs = torch.meshgrid(torch.arange(H).float(), torch.arange(W).float(), indexing='ij')
    gx = (xs + flow[:, 0]) / (W - 1) * 2 - 1
    gy = (ys + flow[:, 1]) / (H - 1) * 2 - 1
    im2 = F.grid_sample(im1, torch.stack([gx, gy], 3), mode='bilinear', padding_mode='border',
                        align_corners=True)
    im2 = (im2 + torch.randn(im2.shape, generator=g) * 2.0).clamp(0, 255)
    return (im1.permute(0, 2, 3, 1).contiguous(), im2.permute(0, 2, 3, 1).contiguous(),
            flow.permute(0, 2, 3, 1).contiguous())


def supervised_batch(B, H, W, seed=1234, max_flow=8.0, density=0.4):
    """A ground-truth batch ``(im1, im2, flow_gt, mask_gt)`` like ``KITTIInput.input_train_gt``
    delivers: float32 NHWC CPU tensors, flow in pixels [B,H,W,2], mask 0/1 [B,H,W,1].
    ``flow_gt`` is the flow of frame 1, so ``image_warp(im2, flow_gt) ~ im1`` (``image_pair``'s flow
    maps its second image onto its first, so its frames are swapped here).  The mask is a seeded
    sparse set of valid pixels (``density`` of them); elsewhere the flow holds -512, what an invalid
    KITTI ground-truth pixel (0 in the 16-bit file) decodes to."""
    a, b, flow = image_pair(B, H, W, seed=seed, max_flow=max_flow)
    g = torch.Generator().manual_seed(seed + 1)
    mask = (torch.rand(B, H, W, 1, generator=g) < density).float()
    flow_gt = torch.where(mask > 0, flow, torch.full_like(flow, -512.0))
    return b, a, flow_gt.contiguous(), mask


def level_inputs(B, h, w, seed=7, flow_mag=3.0):
    """Inputs of one compute_losses call: images in [0,1], smooth flows in pixels, border mask."""
    im1, im2, flow = image_pair(B, h, w, seed=seed, max_flow=flow_mag)
    g = torch.Generator().manual_seed(seed + 1)
    flow_fw = flow + torch.randn(flow.shape, generator=g) * 0.3
    flow_bw = -flow + torch.randn(flow.shape, generator=g) * 0.3
    return im1 / 255.0, im2 / 255.0, flow_fw.contiguous(), flow_bw.contiguous()
