#!/usr/bin/env python
"""Run the reference's OWN supervised fine-tuning code (src/e2eflow/core/supervised.py and
kitti/input.py, unmodified) under the TensorFlow-API stand-in of tests/golden/tf_shim.py and store
the results in tests/golden/reference_supervised.npz.

    python tests/golden/make_reference_supervised.py      (needs the reference source tree)

Stored: for specs c, s and cs with train_all and cs without, the loss value of
``supervised_loss`` with the photometric draws it made (recorded, so a test replays them), the
L2 norm of the gradient of every variable and the small gradients in full; and the
``input_train_gt(hold_out)`` file lists on a stub tree holding both KITTI training sets.  The
inputs are redrawn from their seeds by the tests (``synthetic.supervised_batch``, the oracle's
``init_variables``).  tests/test_oracle_vs_reference_supervised.py compares the oracle and the
product's host path with these vectors.

The stand-in serves the unsupervised graph; ``extend_shim`` adds, for this script only, the few
TensorFlow calls the supervised code makes beyond it (``slim.losses.get_regularization_losses``,
and the int32 shape arithmetic and integer draw of a three-tensor ``random_crop``).
"""
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_reference_run import N, T, load_reference  # noqa: E402
import tf_shim  # noqa: E402
from oracle import flownet as oflownet  # noqa: E402
from unflow_b200 import synthetic as synth  # noqa: E402

# tag -> (spec, train_all, batch, height, width, seed)
CASES = {'c': ('c', True, 2, 64, 128, 61), 's': ('s', True, 2, 64, 64, 62),
         'cs': ('cs', True, 1, 64, 64, 63), 'cs_last': ('cs', False, 1, 64, 64, 64)}
# stub tree of input_train_gt: pairs per set (2015 image_2, 2012 colored_0) and the hold-out
LISTING_PAIRS = {'data_scene_flow': 9, 'data_stereo_flow': 7}
LISTING_HOLD_OUT = 3


class _Int32:
    """``tf.int32`` as a tensor's dtype attribute: augment.random_crop draws its offsets with
    ``maxval=size.dtype.max``."""
    max = 2 ** 31 - 1


class _IntTensor(tf_shim.Tensor):
    @property
    def dtype(self):
        return _Int32

    def __rsub__(self, other):              # shape list - size tensor
        return tf_shim._t(other, 'int32').as_subclass(_IntTensor) - self


def extend_shim(tf):
    """Add to the installed stand-in what supervised.py and input_train_gt call beyond the
    unsupervised graph."""
    shape, convert_to_tensor, random_uniform = tf.shape, tf.convert_to_tensor, tf.random_uniform

    def shape_ext(x):
        if isinstance(x, (list, tuple)):    # the shape of a shape vector (augment.random_crop)
            return [len(x)]
        return shape(x)

    def convert_to_tensor_ext(value, dtype=None, name=None):
        if dtype in ('int32', tf.int32):
            return tf_shim._t(value, dtype).as_subclass(_IntTensor)
        return convert_to_tensor(value, dtype, name)

    def random_uniform_ext(shape=None, minval=0, maxval=1, dtype='float32', seed=None):      # noqa: A002
        if dtype is _Int32:                 # integers in [minval, maxval)
            u = torch.randint(int(minval), int(maxval), [int(s) for s in shape], generator=tf_shim.STATE.rng,
                              dtype=torch.int64)
            tf_shim.STATE.draws.append(u.clone())
            return tf_shim._t(u)
        return random_uniform(shape, minval, maxval, dtype, seed)

    tf.shape, tf.convert_to_tensor, tf.random_uniform = shape_ext, convert_to_tensor_ext, random_uniform_ext
    tf.contrib.slim.losses = types.SimpleNamespace(
        get_regularization_losses=lambda: list(tf_shim.STATE.reg_losses))


def main():
    tf, ref = load_reference()
    extend_shim(tf)
    import importlib
    sup = importlib.import_module('e2eflow.core.supervised')
    assert os.path.realpath(sup.__file__).startswith(os.path.realpath(os.path.dirname(ref['losses'].__file__)))
    out = {}
    for tag, (spec, train_all, B, h, w, seed) in CASES.items():
        variables = oflownet.init_variables(spec, False, seed=seed)
        leaves = {k: v.clone().requires_grad_(True) for k, v in variables.items()}
        tf_shim.STATE.reset(leaves)
        tf_shim.STATE.rng.manual_seed(seed)
        batch = synth.supervised_batch(B, h, w, seed=seed + 100)
        params = dict(flownet=spec, train_all=train_all)
        loss = sup.supervised_loss(tuple(T(t) for t in batch), params, synth.KITTI_NORMALIZATION)
        assert len(tf_shim.STATE.draws) == 5
        for name, d in zip(('contrast', 'gamma', 'colour', 'noise', 'brightness'), tf_shim.STATE.draws):
            out['sl_%s_photo_%s' % (tag, name)] = N(d)
        names = sorted(leaves)
        grads = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
        out['sl_%s_loss' % tag] = N(loss)
        out['sl_%s_grad_names' % tag] = np.array(names)
        out['sl_%s_grad_norms' % tag] = np.array([0.0 if g is None else float(g.double().norm()) for g in grads])
        for k, g in zip(names, grads):
            if g is not None and g.numel() <= 4096:
                out['sl_%s_grad/%s' % (tag, k)] = N(g)

    # ---- input_train_gt: which (frame 1, frame 2, ground truth) triples, in which order ---------------
    with tempfile.TemporaryDirectory() as root:
        for top, n in LISTING_PAIRS.items():
            img = 'image_2' if top == 'data_scene_flow' else 'colored_0'
            for sub, names in ((img, ['%06d_%d.png' % (i, j) for i in range(n) for j in (10, 11)]),
                               ('flow_occ', ['%06d_10.png' % i for i in range(n)])):
                os.makedirs(os.path.join(root, top, 'training', sub))
                for name in names:
                    open(os.path.join(root, top, 'training', sub, name), 'w').close()

        class Data:
            current_dir = root

        tf_shim.STATE.reset({})
        tf_shim.STATE.decode_shape = (6, 8, 3)
        inp = ref['kitti_input'].KITTIInput(Data(), batch_size=1, dims=(4, 6), normalize=False)
        inp.input_train_gt(LISTING_HOLD_OUT)
        q = tf_shim.STATE.queues
        assert q[0] is not None and q[2] == q[3]          # the ground-truth list feeds two readers
        rel = lambda files: [os.path.relpath(f, root) for f in files]
        listing = {'hold_out': LISTING_HOLD_OUT, 'pairs': LISTING_PAIRS,
                   'im1': rel(q[0]), 'im2': rel(q[1]), 'gt': rel(q[2])}
    out['train_gt_listing_json'] = np.array(json.dumps(listing))

    path = os.path.join(HERE, 'reference_supervised.npz')
    np.savez_compressed(path, **out)
    print("wrote %s: %d arrays, %.1f KB" % (path, len(out), os.path.getsize(path) / 1024.0))


if __name__ == '__main__':
    main()
