#!/usr/bin/env python
"""Record the TensorBoard summary tags the reference writes, by running its OWN code (unmodified):
``unsupervised_loss`` / ``supervised_loss`` and the summary helpers of core/train.py, under the
TensorFlow-API stand-in of tests/golden/tf_shim.py, and store them in
tests/golden/reference_summaries.json.

    python tests/golden/make_reference_summaries.py      (needs the reference source tree)

The stand-in has no graph, so op names do not exist there.  ``Naming`` wraps it -- the stand-in
itself is not edited -- with TF 1.x's naming rules for the calls that name things: ``variable_scope``
and ``name_scope`` open a name scope made unique with ``Graph.unique_name`` (a scope object re-enters
its original scope), ``identity`` and ``placeholder`` create an op named by the same rule inside the
current scope, and ``summary.scalar`` / ``summary.image`` open a name scope of their ``name`` whose
unique name is the tag (summary_op_util.summary_scope).  The ops the stand-in evaluates without a
name (``mul``, ``Mean``, ``Const``, ...) are not registered; they take TF's generated names, which
are op-type names and cannot equal a tracked name, but that is argued here, not modelled: the JSON
says so under ``unmodelled``.

Recorded per configuration (config_template's [train] with [train_kitti], [train_synthia], and
[train_kitti_ft] with flownet = CSS, train_all = True): the op names of the 'losses', 'params' and
'train_images' collections, the training graph's summary tags in creation order (Trainer.train with
the learning-rate placeholder, ``get_train_and_loss_ops``' ``_add_summaries`` with the image
summaries of ``debug``), and the evaluation graph's tags (Trainer.eval: ``unsupervised_loss`` with
augment=False, then the AEE / outlier and loss placeholders).  tests/test_summary_cpu.py compares
the product's tags with them.
"""
import ast
import contextlib
import importlib
import json
import os
import re
import sys
import textwrap
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_reference_run import REF_SRC, T, load_reference  # noqa: E402
from make_reference_supervised import extend_shim  # noqa: E402
import tf_shim  # noqa: E402
from oracle import flownet as oflownet  # noqa: E402
from unflow_b200 import synthetic as synth  # noqa: E402

# tag -> (config_template sections, overrides, supervised, frame size of the stand-in run)
CONFIGS = {'train_kitti': (('train', 'train_kitti'), {}, False, (128, 256)),
           'train_synthia': (('train', 'train_synthia'), {}, False, (128, 256)),
           'kitti_ft_CSS_train_all': (('train', 'train_kitti_ft'), {'flownet': 'CSS', 'train_all': True}, True,
                                      (128, 256))}


class Naming:
    """TF 1.x op / scope naming over the stand-in (module docstring)."""

    def __init__(self, tf):
        self.tf = tf
        self.reset()

    def reset(self):
        self.in_use = {}
        self.stack = ''
        self.summaries = []             # (collection, kind, tag) in creation order

    def unique(self, name):
        """ops.py Graph.unique_name."""
        if self.stack:
            name = self.stack + '/' + name
        key = name.lower()
        i = self.in_use.get(key, 0)
        self.in_use[key] = i + 1
        if i == 0:
            return name
        base = key
        while key in self.in_use:
            key = '%s_%d' % (base, i)
            i += 1
        self.in_use[key] = 1
        return '%s_%d' % (name, i - 1)

    @contextlib.contextmanager
    def scope(self, name):
        """ops.name_scope: None / '' -> root, 'a/b/' -> absolute, else unique."""
        old = self.stack
        if not name:
            self.stack = ''
        elif name.endswith('/'):
            self.stack = name[:-1]
        else:
            self.stack = self.unique(name)
        try:
            yield self.stack + '/' if self.stack else ''
        finally:
            self.stack = old

    def _named(self, x, name):
        t = x if isinstance(x, torch.Tensor) else torch.as_tensor(float(x))
        t = t.as_subclass(tf_shim.Tensor)
        with self.scope(name) as sc:
            t.op = types.SimpleNamespace(name=sc[:-1])
        return t

    def install(self):
        tf, me = self.tf, self
        variable_scope, shim_summary = tf.variable_scope, tf.summary

        @contextlib.contextmanager
        def variable_scope_named(name_or_scope, default_name=None, values=None, reuse=None):
            with variable_scope(name_or_scope, default_name, values, reuse) as vs:
                original = getattr(name_or_scope, 'original_name_scope', None)
                with me.scope(original if original is not None else (name_or_scope or default_name)) as sc:
                    vs.original_name_scope = sc
                    yield vs

        def summary_op(kind):
            def fn(name, tensor, *args, collections=None, **kw):
                with me.scope(re.sub(r'[^-/\w\.]', '_', name)) as sc:
                    tag = sc.rstrip('/')
                for key in collections or [tf.GraphKeys.SUMMARIES]:
                    me.summaries.append((key, kind, tag))
                    tf.add_to_collection(key, tag)
                return tag
            return fn

        tf.variable_scope = variable_scope_named
        tf.name_scope = lambda name, default_name=None, values=None: me.scope(name or default_name)
        tf.identity = lambda x, name=None: me._named(x, name or 'Identity')
        tf.placeholder = lambda dtype, shape=None, name=None: me._named(0.0, name or 'Placeholder')
        tf.get_collection = lambda key, scope=None: list(tf_shim.STATE.collections.get(key, []))
        tf.summary = types.SimpleNamespace(scalar=summary_op('scalar'), image=summary_op('image'),
                                           merge=lambda *a, **k: None, merge_all=lambda *a, **k: None,
                                           **{k: getattr(shim_summary, k) for k in ()})


def train_py_functions(names, scope):
    """The named top-level functions of the reference's core/train.py, compiled as they are."""
    src = open(os.path.join(REF_SRC, 'e2eflow', 'core', 'train.py')).read()
    mod = ast.parse(src)
    body = [n for n in mod.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert sorted(n.name for n in body) == sorted(names)
    exec(compile(ast.Module(body=body, type_ignores=[]), 'train.py', 'exec'), scope)
    return src.split('\n')


def cut(lines, first_marker, end_marker, inclusive_first=True):
    first = next(i for i, l in enumerate(lines) if first_marker in l)
    last = next(i for i in range(first + 1, len(lines)) if end_marker in lines[i])
    return textwrap.dedent('\n'.join(lines[first if inclusive_first else first + 1:last]))


def main():
    tf, ref = load_reference()
    extend_shim(tf)
    naming = Naming(tf)
    naming.install()
    core_util = importlib.import_module('e2eflow.core.util')
    sup = importlib.import_module('e2eflow.core.supervised')
    unsup = ref['unsupervised']
    flow_util = ref['flow_util']
    for m in (core_util, sup):
        assert os.path.realpath(m.__file__).startswith(os.path.realpath(REF_SRC)), m.__file__
    cfg = ref['util'].config_dict(os.path.join(os.path.dirname(REF_SRC), 'config_template', 'config.ini'))

    helpers = {'tf': tf, 're': re}
    lines = train_py_functions(['_add_loss_summaries', '_add_param_summaries', '_add_image_summaries'], helpers)
    lr_block = cut(lines, "with tf.name_scope('params') as scope:", 'global_step_ = tf.placeholder')
    assert 'summarized_placeholder' in lr_block
    eval_block = cut(lines, 'for name, gt_flow, mask in truth_tuples:', 'ckpt = tf.train.get_checkpoint_state')
    assert "losses = tf.get_collection('losses')" in eval_block

    out = {'unmodelled': ["ops the stand-in evaluates without a name (mul, Mean, Const, ...) are not registered "
                          "with the naming model; TF names them after their op type, which no tracked name equals",
                          "multi-GPU towers: one graph without tower_N/ scopes is recorded"],
           'configs': {}}
    for tag, (sections, overrides, supervised, (h, w)) in CONFIGS.items():
        params = {}
        for s in sections:
            params.update(cfg[s])
        params.update(overrides)
        ref['util'].convert_input_strings(params, cfg['dirs'])
        spec = params['flownet']
        variables = oflownet.init_variables(spec, False, seed=5)
        rec = {'params': {k: v for k, v in params.items() if not isinstance(v, list)}}

        # ---- training graph (Trainer.train, get_train_and_loss_ops with one device, debug) ----------------
        tf_shim.STATE.reset({k: v.clone() for k, v in variables.items()})
        naming.reset()
        exec(lr_block, {'tf': tf, 'util': core_util})
        if supervised:
            batch = tuple(T(t) for t in synth.supervised_batch(1, h, w, seed=7))
            sup.supervised_loss(batch, params, synth.KITTI_NORMALIZATION)
        else:
            i1, i2, _ = synth.image_pair(1, h, w, seed=7)
            unsup.unsupervised_loss((T(i1), T(i2)), params, synth.KITTI_NORMALIZATION)     # augment=True
        coll = tf_shim.STATE.collections
        rec['losses'] = [t.op.name for t in coll.get('losses', [])]
        rec['params_collection'] = [t.op.name for t in coll.get('params', [])]
        rec['train_images'] = [t.op.name for t in coll.get('train_images', [])]
        helpers['_add_loss_summaries']()
        helpers['_add_param_summaries']()
        helpers['_add_image_summaries']()
        rec['train_summaries'] = [[kind, t] for key, kind, t in naming.summaries if key == 'summaries']

        # ---- evaluation graph (Trainer.eval) ----------------------------------------------------------------
        tf_shim.STATE.reset({k: v.clone() for k, v in variables.items()})
        naming.reset()
        i1, i2, gt = synth.image_pair(1, h, w, seed=8)
        _, flow, _ = unsup.unsupervised_loss((T(i1), T(i2)), params, synth.KITTI_NORMALIZATION, augment=False,
                                             return_flow=True)
        mask = T(torch.ones(1, h, w, 1))
        scope = {'tf': tf, 're': re, 'flow': flow, 'flow_error_avg': flow_util.flow_error_avg,
                 'outlier_pct': flow_util.outlier_pct, 'summarized_placeholder': core_util.summarized_placeholder,
                 'truth_tuples': [('occluded', T(gt), mask), ('non-occluded', T(gt), mask)],
                 'values_': [], 'averages_': []}
        exec(eval_block, scope)
        rec['eval_losses'] = [t.op.name for t in tf_shim.STATE.collections.get('losses', [])]
        rec['eval_summaries'] = [[kind, t] for key, kind, t in naming.summaries if key == 'eval_avg']
        out['configs'][tag] = rec

    path = os.path.join(HERE, 'reference_summaries.json')
    with open(path, 'w') as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write('\n')
    print("wrote %s" % path)


if __name__ == '__main__':
    main()
