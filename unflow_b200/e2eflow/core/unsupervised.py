"""The unsupervised training objective with the reference's signature
(/root/reference/src/e2eflow/core/unsupervised.py:27-164):

    unsupervised_loss(batch, params, normalization=None, augment=True, return_flow=False)

``params`` carries the keys of config.ini [train] plus the dataset section, read the way the
reference reads them: flownet, full_res, train_all, pyramid_loss, mask_occlusion, border_mask and
the ``<term>_weight`` entries.  ``augment=True`` runs the reference's random affine / photometric
augmentation (core/augment.py) on torch's random stream instead of TF's.

Mechanics that differ from the TF graph: the network variables come from a ``FlowNetVariables``
module (keyword ``variables``; default: the module-level store of core.flownet) instead of TF's
graph collections; only the loss terms that carry a weight are evaluated (graph mode prunes the
others, here the set is handed to ``compute_losses``); each pyramid level is one fused forward /
backward kernel pair.
"""
import torch

from . import fused_loss, tf_image
from .flownet import FLOW_SCALE, flownet, get_variables
from .losses import compute_losses, create_border_mask
from .util import downsample

# every loss term a config may weight (reference :15)
LOSSES = ['occ', 'sym', 'fb', 'grad', 'ternary', 'photo', 'smooth_1st', 'smooth_2nd']

# Per-level weights and census patch radii of the loss pyramid (reference :87-92): the five
# decoder resolutions, preceded by two more when the network predicts at full resolution.
_LEVEL_WEIGHTS = [12.7, 4.35, 3.9, 3.4, 1.1]
_LEVEL_DISTANCES = [3, 2, 2, 1, 1]
_FULL_RES_WEIGHTS = [12.7, 5.5, 5.0, 4.35, 3.9, 3.4, 1.1]
_FULL_RES_DISTANCES = [3, 3] + _LEVEL_DISTANCES

# TF collects tracked values in graph collections (reference :18-24, :158-159); the eager counterparts
# are dicts refilled on every call, keyed by the reference's op names ('loss2/ternary', 'loss/combined',
# 'weight/ternary', 'train/augmented1') in the order TF creates the ops.  ``tracked_images`` is filled
# only while ``track_images`` is set (core/train.py sets it when image summaries are written): it keeps
# the tracked batches alive until the next call.  Its values are ``(tensor, to_image)``, the callable
# turning the tensor into the summarised image when a summary is written (None: the tensor itself).
tracked = {}
tracked_params = {}
tracked_images = {}
track_images = False
_const_cache = {}


def _track_loss(op, name):
    tracked[name] = op.detach() if torch.is_tensor(op) else op


def _track_image(op, name, to_image=None):
    if track_images:
        tracked_images['train/' + name] = (op.detach(), to_image)


def _clear_tracked():
    tracked.clear()
    tracked_params.clear()
    tracked_images.clear()


def _device_constant(values, device):
    """Small host constants as cached device tensors: the step holds no host->device copy, so it
    can be captured in a CUDA graph."""
    key = (tuple(float(v) for v in values), str(device))
    if key not in _const_cache:
        _const_cache[key] = torch.tensor(list(values), device=device, dtype=torch.float32)
    return _const_cache[key]


def _augmented(frame1, frame2, border_mask):
    """Reference :39-60: one global affine for both frames and the mask, a second small affine for
    frame 2 only, then photometric jitter on the network inputs.  Returns the geometric pair (for
    the loss), the photometric pair (for the network) and the combined validity mask."""
    from .augment import random_affine, random_photometric
    mask = border_mask.contiguous()
    geo1, geo2, mask_global = random_affine([frame1, frame2, mask], horizontal_flipping=True,
                                            min_scale=0.9, max_scale=1.1)
    geo2, mask_local = random_affine([geo2, mask], min_scale=0.9, max_scale=1.1)
    net1, net2 = random_photometric([geo1, geo2], noise_stddev=0.04,
                                    min_contrast=-0.3, max_contrast=0.3, brightness_stddev=0.02,
                                    min_colour=0.9, max_colour=1.1, min_gamma=0.7, max_gamma=1.5)
    return geo1, geo2, net1, net2, mask_local * mask_global


def unsupervised_loss(batch, params, normalization=None, augment=True,
                      return_flow=False, variables=None):
    _clear_tracked()
    frame1, frame2 = (f / 255.0 for f in batch)
    size = frame1.shape[1:3]
    mean = _device_constant([m / 255.0 for m in normalization[0]], frame1.device)
    border_mask = create_border_mask(frame1, 0.1)

    # the loss compares images in [0, 1]; the network sees mean-subtracted (and jittered) copies
    if augment:
        loss_im1, loss_im2, net_im1, net_im2, border_mask = _augmented(frame1, frame2, border_mask)
        _track_image(net_im1, 'augmented1')
        _track_image(net_im2, 'augmented2')
    else:
        loss_im1, loss_im2, net_im1, net_im2 = frame1, frame2, frame1, frame2

    spec = params.get('flownet', 'S')
    full_res = params.get('full_res')
    if variables is None:
        variables = get_variables(spec, full_res, device=frame1.device)
    stack_fw, stack_bw = flownet(net_im1 - mean, net_im2 - mean, flownet_spec=spec,
                                 full_resolution=full_res, backward_flow=True,
                                 train_all=params.get('train_all'), variables=variables)
    pyramid_fw, pyramid_bw = stack_fw[-1], stack_bw[-1]      # only the last network is scored

    if full_res:
        weights, distances = _FULL_RES_WEIGHTS, _FULL_RES_DISTANCES
        level_im1, level_im2, level_mask = loss_im1, loss_im2, border_mask
        top_scale = FLOW_SCALE * 4
    else:
        weights, distances = _LEVEL_WEIGHTS, _LEVEL_DISTANCES
        level_im1, level_im2 = downsample(loss_im1, 4), downsample(loss_im2, 4)
        level_mask = downsample(border_mask.contiguous(), 4)
        top_scale = FLOW_SCALE

    def final_flow(finest):
        """The full-size output flow in pixels (reference :97-98, :105-106).  Only evaluated when
        it is returned: a TF session prunes it from the training step, eager code has to ask."""
        if full_res:
            return finest * top_scale
        return tf_image.resize_bilinear(finest, size) * top_scale * 4

    n_levels = len(pyramid_fw) if params.get('pyramid_loss') else 1
    active = [t for t in LOSSES if params.get(t + '_weight')]
    mask_occlusion = params.get('mask_occlusion', '')
    assert mask_occlusion in ['fb', 'disocc', '']

    per_term = {t: 0.0 for t in LOSSES}
    per_vec = None
    total = 0.0
    for lvl in range(n_levels):
        scope = 'loss%d/' % (lvl + 2)                      # the level's variable scope (reference :117-121)
        to_pixels = top_scale / (2 ** lvl)                 # network units -> pixels at this level
        terms = compute_losses(level_im1, level_im2,
                               pyramid_fw[lvl] * to_pixels, pyramid_bw[lvl] * to_pixels,
                               border_mask=level_mask if params.get('border_mask') else None,
                               mask_occlusion=mask_occlusion,
                               data_max_distance=distances[lvl],
                               _terms=active)
        vec = terms.get(fused_loss.VECTOR_KEY)
        if vec is not None:
            # fused kernel: the terms come as one vector -- weight them with one dot product instead of a
            # scalar multiply + add per term and level (about 100 one-element kernels per step and as many
            # again in the backward pass); same sum, order of the fp32 additions aside
            for t in active:
                _track_loss(terms[t], scope + t)
            wvec = _device_constant([(params.get(t + '_weight') or 0.0) if t in active else 0.0
                                     for t in fused_loss.TERM_ORDER], vec.device)
            level_sum = torch.dot(vec, wvec)
            per_vec = (per_vec if per_vec is not None else 0.0) + weights[lvl] * vec.detach()
        else:
            level_sum = 0.0
            for t in active:
                _track_loss(terms[t], scope + t)
                level_sum = level_sum + params[t + '_weight'] * terms[t]
                per_term[t] = per_term[t] + weights[lvl] * terms[t]
        total = total + weights[lvl] * level_sum
        if lvl + 1 < n_levels:      # (the reference also builds one level more, which TF prunes)
            level_im1, level_im2 = downsample(level_im1, 2), downsample(level_im2, 2)
            level_mask = downsample(level_mask, 2)

    final_loss = total + variables.regularization_loss()

    if per_vec is not None:
        for i, t in enumerate(fused_loss.TERM_ORDER):
            if t in active:
                per_term[t] = per_vec[i]
    _track_loss(final_loss, 'loss/combined')
    for t in LOSSES:
        _track_loss(per_term[t], 'loss/' + t)
        if params.get(t + '_weight'):
            tracked_params['weight/' + t] = params[t + '_weight']

    if return_flow:
        return final_loss, final_flow(pyramid_fw[0]), final_flow(pyramid_bw[0])
    return final_loss
