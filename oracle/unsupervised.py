"""CPU restatement of the unsupervised loss assembly (TEST INFRASTRUCTURE ONLY).

Follows /root/reference/src/e2eflow/core/unsupervised.py:27-164 with
``augment=False`` (the random augmentation cannot be parity-pinned and is out
of scope, SURVEY.md section 2).  Pinned against the reference file itself,
executed unmodified under the TensorFlow-API stand-in of tests/golden/ (loss
value, output flows and variable gradients for specs c / s / cs, pyramid on /
off, train_all: tests/test_oracle_vs_reference_run.py); PARITY UNPINNED below
that for the TF primitives it rests on (see oracle/__init__.py).
"""
import torch

from . import tf_compat as tfc
from .flownet import flownet, FLOW_SCALE
from .losses import compute_losses, create_border_mask
from .util import downsample

LOSSES = ['occ', 'sym', 'fb', 'grad', 'ternary', 'photo', 'smooth_1st', 'smooth_2nd']  # :15


def regularization_loss(variables, scale=0.0004):
    """slim.l2_regularizer(0.0004) on every conv / deconv ``weights`` variable
    (flownet.py:176,200,218): scale * sum(w^2) / 2, summed over variables, in their dtype."""
    ws = [torch.as_tensor(v) for name, v in variables.items() if name.endswith('/weights')]
    total = torch.zeros((), dtype=ws[0].dtype, device=ws[0].device) if ws else torch.zeros(())
    for w in ws:
        total = total + scale * (torch.sum(w ** 2) / 2)
    return total


def _pyramid_table(full_resolution):
    """(weight, census radius) per loss level, finest first (unsupervised.py:87-92)."""
    table = [(12.7, 3), (4.35, 2), (3.9, 2), (3.4, 1), (1.1, 1)]
    if full_resolution:
        table = [(12.7, 3), (5.5, 3), (5.0, 3)] + table[1:]
    return table


def unsupervised_loss(variables, batch, params, normalization=None, augment=False,
                      return_flow=False, return_terms=False):
    if augment:
        raise NotImplementedError("the oracle restates the augment=False graph only")
    mean = torch.tensor(normalization[0], dtype=batch[0].dtype, device=batch[0].device) / 255.0  # :31
    a, b = batch[0] / 255.0, batch[1] / 255.0                                 # :32-33
    out_hw = a.shape[1:3]
    valid = create_border_mask(a, 0.1)                                         # :38

    spec = params.get('flownet', 'S')
    full = params.get('full_res')
    # without augmentation the loss images are the inputs and the network images are the
    # mean-subtracted inputs (:62-68); only the last network of a stack is scored (:79-80)
    fw_all, bw_all = flownet(variables, a - mean, b - mean, flownet_spec=spec, full_resolution=full,
                             backward_flow=True, train_all=params.get('train_all'))
    fw, bw = fw_all[-1], bw_all[-1]

    table = _pyramid_table(full)
    if full:                                                                   # :93-99
        unit = FLOW_SCALE * 4
        pyr = [(a, b, valid)]
        flow_fw, flow_bw = fw[0] * unit, bw[0] * unit
    else:                                                                      # :100-106
        unit = FLOW_SCALE
        pyr = [(downsample(a, 4), downsample(b, 4), downsample(valid, 4))]
        flow_fw = tfc.resize_bilinear_legacy(fw[0], out_hw) * unit * 4
        flow_bw = tfc.resize_bilinear_legacy(bw[0], out_hw) * unit * 4

    depth = len(fw) if params.get('pyramid_loss') else 1                       # :113-116
    while len(pyr) < depth:                                                    # :147-149
        pyr.append(tuple(downsample(t, 2) for t in pyr[-1]))

    occlusion = params.get('mask_occlusion', '')
    assert occlusion in ['fb', 'disocc', '']
    weighted = [(name, params[name + '_weight']) for name in LOSSES if params.get(name + '_weight')]

    by_term = dict.fromkeys(LOSSES, 0.0)
    objective = 0.0
    for k in range(depth):                                                     # :118-145
        (lam, radius), (pa, pb, pm) = table[k], pyr[k]
        px = unit / (2 ** k)
        got = compute_losses(pa, pb, fw[k] * px, bw[k] * px,
                             border_mask=pm if params.get('border_mask') else None,
                             mask_occlusion=occlusion, data_max_distance=radius)
        acc = 0.0
        for name, w in weighted:
            acc = acc + w * got[name]
            by_term[name] = by_term[name] + lam * got[name]
        objective = objective + lam * acc

    objective = objective + regularization_loss(variables)                     # :151-152

    ret = [objective]
    if return_flow:
        ret += [flow_fw, flow_bw]
    if return_terms:
        ret.append(by_term)
    return ret[0] if len(ret) == 1 else tuple(ret)
