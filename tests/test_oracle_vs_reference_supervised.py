"""The supervised fine-tuning loss against the reference's own supervised.py, executed unmodified
under tests/golden/tf_shim.py (tests/golden/reference_supervised.npz, made by
tests/golden/make_reference_supervised.py): the oracle's restatement, and the product's host path
with its CUDA entry points swapped for the oracle's CPU ops and the unfused loss.  The recorded
photometric draws are replayed."""
import os

import numpy as np
import pytest
import torch

from oracle import flownet as oflownet
from oracle import supervised as osup
from unflow_b200 import synthetic as usynth
import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_supervised.npz')
DRAWS = ('contrast', 'gamma', 'colour', 'noise', 'brightness')
# must match tests/golden/make_reference_supervised.py CASES
CASES = {'c': ('c', True, 2, 64, 128, 61), 's': ('s', True, 2, 64, 64, 62),
         'cs': ('cs', True, 1, 64, 64, 63), 'cs_last': ('cs', False, 1, 64, 64, 64)}


@pytest.fixture(scope='module')
def ref():
    return dict(np.load(GOLDEN))


def _case(ref, tag):
    spec, train_all, B, h, w, seed = CASES[tag]
    params = dict(flownet=spec, train_all=train_all)
    batch = usynth.supervised_batch(B, h, w, seed=seed + 100)
    draws = [torch.as_tensor(ref['sl_%s_photo_%s' % (tag, n)]) for n in DRAWS]
    return spec, params, batch, draws, seed


def _check_grads(ref, tag, grads, rtol):
    names = [str(n) for n in ref['sl_%s_grad_names' % tag]]
    assert sorted(grads) == names
    norms = ref['sl_%s_grad_norms' % tag]
    for name, want in zip(names, norms):
        g = grads[name]
        got = 0.0 if g is None else float(g.double().norm())
        np.testing.assert_allclose(got, want, rtol=rtol, atol=1e-9, err_msg=name)
        key = 'sl_%s_grad/%s' % (tag, name)
        if key in ref:
            np.testing.assert_allclose(g.detach().numpy(), ref[key], rtol=rtol, atol=rtol * float(np.abs(ref[key]).max()),
                                       err_msg=name)


@pytest.mark.parametrize("tag", list(CASES))
def test_oracle_supervised_loss_vs_reference(ref, tag):
    spec, params, batch, draws, seed = _case(ref, tag)
    tfv = {k: v.clone().requires_grad_(True) for k, v in oflownet.init_variables(spec, False, seed=seed).items()}
    loss = osup.supervised_loss(tfv, batch, params, synth.KITTI_NORMALIZATION, photometric_draws=draws)
    np.testing.assert_allclose(float(loss.detach()), float(ref['sl_%s_loss' % tag]), rtol=1e-6)
    names = sorted(tfv)
    grads = torch.autograd.grad(loss, [tfv[k] for k in names], allow_unused=True)
    _check_grads(ref, tag, dict(zip(names, grads)), rtol=1e-4)


@pytest.mark.parametrize("tag", list(CASES))
def test_product_supervised_loss_host_path_vs_reference(ref, tag, monkeypatch):
    """supervised_loss's control flow (photometric jitter, mean, networks scored, 2**-i weights,
    regularisation) with the network served by the oracle on the CPU and the unfused loss."""
    from unflow_b200.e2eflow.core import augment
    from unflow_b200.e2eflow.core import supervised as S
    from unflow_b200.e2eflow.core import unsupervised as U
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    spec, params, batch, draws, seed = _case(ref, tag)
    tfv = oflownet.init_variables(spec, False, seed=seed)
    v = FlowNetVariables(spec, False, seed=0).load_tf_dict(tfv)
    leaves = {k: t.clone().requires_grad_(True) for k, t in tfv.items()}

    def cpu_flownet(im1, im2, flownet_spec='S', full_resolution=False, train_all=False, backward_flow=False,
                    variables=None):
        assert variables is v and not backward_flow
        return oflownet.flownet(leaves, im1, im2, flownet_spec=flownet_spec, full_resolution=full_resolution,
                                train_all=train_all)

    def replayed_photometric(ims, **kw):
        return augment.photometric(ims, *draws)

    monkeypatch.setattr(S, 'flownet', cpu_flownet)
    monkeypatch.setattr(augment, 'random_photometric', replayed_photometric)
    loss = S.supervised_loss(batch, params, synth.KITTI_NORMALIZATION, augment=True, variables=v)
    np.testing.assert_allclose(float(loss.detach()), float(ref['sl_%s_loss' % tag]), rtol=2e-5)
    assert float(U.tracked['loss/combined']) == float(loss.detach())
    np.testing.assert_allclose(float(U.tracked['loss/regularization']), float(v.regularization_loss().detach()))
    loss.backward()
    grads = {}
    for name, t in leaves.items():              # the data term reaches the oracle's leaves, the L2 term v's own
        scope, kind = name.rsplit('/', 1)
        w, b = v.weights(scope)
        reg = (w.grad.permute(2, 3, 1, 0) if kind == 'weights' else b.grad)
        reg = torch.zeros_like(t) if reg is None else reg
        grads[name] = (t.grad if t.grad is not None else torch.zeros_like(t)) + reg
    _check_grads(ref, tag, grads, rtol=1e-4)
