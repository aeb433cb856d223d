"""FlowNetC / FlowNetS / stacked networks -- the reference's ``flownet`` entry point
(/root/reference/src/e2eflow/core/flownet.py:14-81) on torch.

Differences in mechanism, not in results:
  * TF keeps variables in the graph's variable store, keyed by scope name; here a
    ``FlowNetVariables`` module holds them under the SAME names
    (``flownet_c_features/conv1/weights`` ... ``stack_1_flownet/flownet_s/flow2/biases``), in the
    layout cuDNN wants (OIHW / IOHW); ``to_tf_dict`` / ``load_tf_dict`` convert to and from the
    reference checkpoint layout (HWIO; conv2d_transpose [kh,kw,out,in]).
  * the two directions share weights (``reuse``) and are independent per sample, so the
    forward and backward passes are batched into ONE pass over 2B samples instead of two
    passes over B -- same arithmetic per sample, half the launches, larger GEMMs.
  * conv / deconv stacks run on cuDNN through torch (dense contractions; fp32 accumulate),
    with TF ``SAME`` padding reproduced exactly (asymmetric for the stride-2 layers).
  * ``correlation`` and ``image_warp`` are the hand-written sm_90a kernels.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import correlation, correlation_bidir
from .image_warp import image_warp
from . import tf_image
from . import conv_ops

FLOW_SCALE = 5.0


def set_conv_precision(mode='fp32'):
    """Arithmetic of the conv / deconv stacks (see core/conv_ops.py).

    'fp32' (default): exact float32 cuDNN convolutions, what the reference's TF1 graph computes.
    torch enables single-pass TF32 convolutions by default, which costs ~1e-3 relative on the flow
    fields and breaks the 1e-4 parity bar (measured) -- so it is switched off on import.
    '3xtf32': convolutions on the hand-written tensor-core kernels at fp32-level accuracy (every operand
    split into TF32 hi + lo, three products accumulated in fp32)."""
    return conv_ops.set_mode(mode)


set_conv_precision(__import__('os').environ.get('UNFLOW_CONV_PRECISION', 'fp32'))


# ---------------------------------------------------------------------------------------------
# Variables
# ---------------------------------------------------------------------------------------------
def _upconv_specs(prefix, m, in6, c5, c4, c3, c2, c1=None, c0=None, full_res=False, ch=2):
    """(name, kind, cin, cout, k) for _flownet_upconv (reference flownet.py:89-155)."""
    s = []
    s.append((prefix + 'flow6', 'conv', in6, ch, 3))
    s.append((prefix + 'deconv5', 'deconv', in6, int(512 * m), 4))
    s.append((prefix + 'flow6_up5', 'deconv', ch, ch, 4))
    cat5 = c5 + int(512 * m) + ch
    s.append((prefix + 'flow5', 'conv', cat5, ch, 3))
    s.append((prefix + 'deconv4', 'deconv', cat5, int(256 * m), 4))
    s.append((prefix + 'flow5_up4', 'deconv', ch, ch, 4))
    cat4 = c4 + int(256 * m) + ch
    s.append((prefix + 'flow4', 'conv', cat4, ch, 3))
    s.append((prefix + 'deconv3', 'deconv', cat4, int(128 * m), 4))
    s.append((prefix + 'flow4_up3', 'deconv', ch, ch, 4))
    cat3 = c3 + int(128 * m) + ch
    s.append((prefix + 'flow3', 'conv', cat3, ch, 3))
    s.append((prefix + 'deconv2', 'deconv', cat3, int(64 * m), 4))
    s.append((prefix + 'flow3_up2', 'deconv', ch, ch, 4))
    cat2 = c2 + int(64 * m) + ch
    s.append((prefix + 'flow2', 'conv', cat2, ch, 3))
    if full_res:
        p = prefix + 'full_res/'
        s.append((p + 'deconv1', 'deconv', cat2, int(32 * m), 4))
        s.append((p + 'flow2_up1', 'deconv', ch, ch, 4))
        cat1 = c1 + int(32 * m) + ch
        s.append((p + 'flow1', 'conv', cat1, ch, 3))
        s.append((p + 'deconv0', 'deconv', cat1, int(16 * m), 4))
        s.append((p + 'flow1_up0', 'deconv', ch, ch, 4))
        cat0 = c0 + int(16 * m) + ch
        s.append((p + 'flow0', 'conv', cat0, ch, 3))
    return s


def layer_specs(flownet_spec='S', full_resolution=False):
    """Every slim.conv2d / conv2d_transpose the reference graph would create for a spec."""
    specs = []
    n = len(flownet_spec)
    for i, name in enumerate(flownet_spec):
        assert name in ('C', 'c', 'S', 's')
        m = 1 if name in ('C', 'S') else 3 / 8
        full_res = full_resolution and i == n - 1
        root = '' if i == 0 else 'stack_%d_flownet/' % i
        c64, c128, c256 = int(64 * m), int(128 * m), int(256 * m)
        c512, c1024 = int(512 * m), int(1024 * m)
        if name.lower() == 'c':
            assert i == 0, 'FlowNetS must be used for refinement networks'
            if full_res:   # flownet_c hands no conv1 / inputs to the up-convolutions (flownet.py:235-236)
                raise ValueError("full_res needs a FlowNetS as the last network of the stack")
            f = root + 'flownet_c_features/'
            specs += [(f + 'conv1', 'conv', 3, c64, 7), (f + 'conv2', 'conv', c64, c128, 5),
                      (f + 'conv3', 'conv', c128, c256, 5)]
            t = root + 'flownet_c/'
            specs += [(t + 'conv_redir', 'conv', c256, int(32 * m), 1),
                      (t + 'conv3_1', 'conv', int(32 * m) + 441, c256, 3)]
            cin = None
        else:
            t = root + 'flownet_s/'
            cin = 6 if i == 0 else 14
            specs += [(t + 'conv1', 'conv', cin, c64, 7), (t + 'conv2', 'conv', c64, c128, 5),
                      (t + 'conv3', 'conv', c128, c256, 5), (t + 'conv3_1', 'conv', c256, c256, 3)]
        specs += [(t + 'conv4', 'conv', c256, c512, 3), (t + 'conv4_1', 'conv', c512, c512, 3),
                  (t + 'conv5', 'conv', c512, c512, 3), (t + 'conv5_1', 'conv', c512, c512, 3),
                  (t + 'conv6', 'conv', c512, c1024, 3), (t + 'conv6_1', 'conv', c1024, c1024, 3)]
        specs += _upconv_specs(t, m, c1024, c512, c512, c256, c128, c64, cin, full_res=full_res)
    return specs


def _key(name):
    return name.replace('.', '_')


class FlowNetVariables(nn.Module):
    """The trainable variables of a (stacked) FlowNet, addressed by TF variable name."""

    def __init__(self, flownet_spec='S', full_resolution=False, seed=None, device=None):
        super().__init__()
        self.flownet_spec = flownet_spec
        self.full_resolution = bool(full_resolution)
        self.params = nn.ParameterDict()
        self.kinds = {}
        gen = None
        if seed is not None:
            gen = torch.Generator().manual_seed(int(seed))
        for (name, kind, cin, cout, k) in layer_specs(flownet_spec, full_resolution):
            if kind == 'conv':
                w = torch.empty(cout, cin, k, k)      # OIHW  <-> TF [k,k,cin,cout]
                fan_in = k * k * cin
            else:
                w = torch.empty(cin, cout, k, k)      # IOHW  <-> TF [k,k,cout,cin]
                fan_in = k * k * cout                 # TF fan_in = shape[-2] * receptive field
            # layers.variance_scaling_initializer(): factor 2, FAN_IN, truncated normal
            std = math.sqrt(1.3 * 2.0 / fan_in)
            nn.init.trunc_normal_(w, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=gen)
            # stored NHWC-ordered ([dim0, kh, kw, dim1] in memory): cuDNN's tensor-core kernels and
            # their weight gradients are NHWC, so the operand kernel reads the weights contiguously and
            # the gradient accumulates into .grad without a layout conversion
            self.params[_key(name + '/weights')] = nn.Parameter(w.contiguous(memory_format=torch.channels_last))
            self.params[_key(name + '/biases')] = nn.Parameter(torch.zeros(cout))
            self.kinds[name] = kind
        if device is not None:
            self.to(device)

    # -- access ---------------------------------------------------------------------------
    def weights(self, scope):
        return self.params[_key(scope + '/weights')], self.params[_key(scope + '/biases')]

    def variable_names(self):
        out = []
        for name in self.kinds:
            out += [name + '/weights', name + '/biases']
        return out

    def scopes_of_net(self, i):
        """Variable scopes belonging to network ``i`` of the stack."""
        root = '' if i == 0 else 'stack_%d_flownet/' % i
        if i == 0:
            return [s for s in self.kinds if not s.startswith('stack_')]
        return [s for s in self.kinds if s.startswith(root)]

    # -- reference checkpoint layout -----------------------------------------------------
    def to_tf_dict(self):
        """name -> tensor in TF layout (conv HWIO; conv2d_transpose [kh,kw,out,in])."""
        out = {}
        for name, kind in self.kinds.items():
            w, b = self.weights(name)
            out[name + '/weights'] = w.detach().permute(2, 3, 1, 0).contiguous().cpu()
            out[name + '/biases'] = b.detach().cpu().clone()
        return out

    def load_tf_dict(self, tf_vars, strict=True):
        with torch.no_grad():
            for name, kind in self.kinds.items():
                for suffix in ('/weights', '/biases'):
                    full = name + suffix
                    if full not in tf_vars:
                        if strict:
                            raise KeyError(full)
                        continue
                    v = torch.as_tensor(tf_vars[full]).float()
                    p = self.params[_key(full)]
                    if suffix == '/weights':
                        v = v.permute(3, 2, 0, 1)
                    if tuple(v.shape) != tuple(p.shape):
                        raise ValueError("shape mismatch for %s: %s vs %s" % (full, tuple(v.shape), tuple(p.shape)))
                    p.copy_(v)
        return self

    L2_SCALE = 0.0004

    def regularization_loss(self, scale=L2_SCALE):
        """slim.l2_regularizer(0.0004) on every ``weights`` variable (flownet.py:176,200,218):
        sum_v scale * sum(v^2) / 2  ==  tf.losses.get_regularization_loss().

        ``l2_in_optimizer`` (set by the Trainer on CUDA): only the VALUE is formed here; the gradient
        ``scale * w`` is added to the weight gradients by the fused Adam kernel (csrc/adam.cu, l2mask), which
        reads the weights anyway -- instead of 36 scaled copies that autograd adds to the gradients."""
        ws = [self.params[_key(n + '/weights')] for n in self.kinds]
        if getattr(self, 'l2_in_optimizer', False):
            with torch.no_grad():
                return _L2Reg.apply(float(scale), *[w.detach() for w in ws])
        return _L2Reg.apply(float(scale), *ws)


class _L2Reg(torch.autograd.Function):
    """0.5 * scale * sum_k ||w_k||^2 with multi-tensor kernels (a handful of launches instead of
    three per variable)."""

    @staticmethod
    def forward(ctx, scale, *ws):
        ctx.scale = scale
        ctx.save_for_backward(*ws)
        norms = torch._foreach_norm([w.detach() for w in ws], 2)
        return ((0.5 * scale) * torch.stack(norms).double().square().sum()).float()

    @staticmethod
    def backward(ctx, gout):
        ws = ctx.saved_tensors
        grads = torch._foreach_mul([w.detach() for w in ws], gout * ctx.scale)
        return (None,) + tuple(g if w.requires_grad else None for g, w in zip(grads, ws))


_default_store = {}


def get_variables(flownet_spec='S', full_resolution=False, device=None, seed=None):
    """The default variable store (TF: the graph's variable collection)."""
    key = (flownet_spec, bool(full_resolution), str(device))
    if key not in _default_store:
        _default_store[key] = FlowNetVariables(flownet_spec, full_resolution, seed=seed, device=device)
    return _default_store[key]


def reset_default_variables():
    _default_store.clear()


# ---------------------------------------------------------------------------------------------
# Layers
# ---------------------------------------------------------------------------------------------
def _leaky_relu(x):
    return F.leaky_relu(x, 0.1)  # == tf.maximum(0.1 * x, x)


def _same_pad(in_size, k, stride):
    out = -(-in_size // stride)
    total = max((out - 1) * stride + k - in_size, 0)
    return total // 2, total - total // 2


class _Scope:
    def __init__(self, variables, prefix):
        self.v, self.p = variables, prefix

    def sub(self, name):
        return _Scope(self.v, self.p + name + '/')

    def conv(self, x, name, stride=1, act=True, out=None):
        w, b = self.v.weights(self.p + name)
        k = w.shape[2]
        # TF SAME padding: asymmetric for the stride-2 layers at even sizes
        pads = _same_pad(x.shape[2], k, stride) + _same_pad(x.shape[3], k, stride)
        return conv_ops.conv2d(x, w, b, stride, pads, act=act, out=out)

    def deconv(self, x, name, act=True, out=None):
        w, b = self.v.weights(self.p + name)
        return conv_ops.conv_transpose2d(x, w, b, act=act, out=out)  # slim.conv2d_transpose(k=4, s=2, SAME)

    def cout(self, name):
        w, _ = self.v.weights(self.p + name)
        return w.shape[0] if self.v.kinds[self.p + name] == 'conv' else w.shape[1]


class _Cat:
    """A pre-allocated NHWC concat buffer (pixel pitch rounded up to 4 floats) and the NCHW-shaped views of
    its members: the tensor-core layers store their outputs straight into their slot, so the concat
    itself copies only what was produced elsewhere (the 2-channel up-sampled flow)."""

    def __init__(self, n, h, w, channels, device):
        c = sum(channels)
        self.buf = torch.empty((n, h, w, (c + 3) // 4 * 4), device=device, dtype=torch.float32)
        self.slots, off = [], 0
        for ci in channels:
            self.slots.append(self.buf[..., off:off + ci].permute(0, 3, 1, 2))
            off += ci


def _decoder_cats(s, like, n, hw3, hw2, c2):
    """Concat buffers of _flownet_upconv for a trunk whose conv3_1 is ``hw3`` and whose conv2 (``c2``
    channels) is ``hw2`` in size; None when the tensor-core path is not active for ``like``."""
    if not conv_ops.tc_active(like):
        return None
    half = lambda v: -(-v // 2)
    (h3, w3), (h2, w2) = hw3, hw2
    h4, w4 = half(h3), half(w3)
    h5, w5 = half(h4), half(w4)
    dev = like.device
    return {2: _Cat(n, h2, w2, [c2, s.cout('deconv2'), 2], dev),
            3: _Cat(n, h3, w3, [s.cout('conv3_1'), s.cout('deconv3'), 2], dev),
            4: _Cat(n, h4, w4, [s.cout('conv4_1'), s.cout('deconv4'), 2], dev),
            5: _Cat(n, h5, w5, [s.cout('conv5_1'), s.cout('deconv5'), 2], dev)}


def _flownet_upconv(s, conv6_1, conv5_1, conv4_1, conv3_1, conv2, conv1=None, inputs=None,
                    channel_mult=1, full_res=False, channels=2, cats=None):
    slot = (lambda lvl: cats[lvl].slots[1]) if cats else (lambda lvl: None)
    buf = (lambda lvl: cats[lvl].buf) if cats else (lambda lvl: None)
    conv6_1 = conv_ops.backward_point(conv6_1, s.p + 'decoder')     # decoder gradients complete behind this point
    flow6 = s.conv(conv6_1, 'flow6', act=False)
    deconv5 = s.deconv(conv6_1, 'deconv5', out=slot(5))
    flow6_up5 = s.deconv(flow6, 'flow6_up5', act=False)
    concat5 = _cat_c([conv5_1, deconv5, flow6_up5], buf(5))
    flow5 = s.conv(concat5, 'flow5', act=False)

    deconv4 = s.deconv(concat5, 'deconv4', out=slot(4))
    flow5_up4 = s.deconv(flow5, 'flow5_up4', act=False)
    concat4 = _cat_c([conv4_1, deconv4, flow5_up4], buf(4))
    flow4 = s.conv(concat4, 'flow4', act=False)

    deconv3 = s.deconv(concat4, 'deconv3', out=slot(3))
    flow4_up3 = s.deconv(flow4, 'flow4_up3', act=False)
    concat3 = _cat_c([conv3_1, deconv3, flow4_up3], buf(3))
    flow3 = s.conv(concat3, 'flow3', act=False)

    deconv2 = s.deconv(concat3, 'deconv2', out=slot(2))
    flow3_up2 = s.deconv(flow3, 'flow3_up2', act=False)
    concat2 = _cat_c([conv2, deconv2, flow3_up2], buf(2))
    flow2 = s.conv(concat2, 'flow2', act=False)

    flows = [flow2, flow3, flow4, flow5, flow6]

    if full_res:
        f = s.sub('full_res')
        deconv1 = f.deconv(concat2, 'deconv1')
        flow2_up1 = f.deconv(flow2, 'flow2_up1', act=False)
        concat1 = _cat_c([conv1, deconv1, flow2_up1])
        flow1 = f.conv(concat1, 'flow1', act=False)

        deconv0 = f.deconv(concat1, 'deconv0')
        flow1_up0 = f.deconv(flow1, 'flow1_up0', act=False)
        concat0 = _cat_c([inputs, deconv0, flow1_up0])
        flow0 = f.conv(concat0, 'flow0', act=False)
        flows = [flow0, flow1] + flows
    return flows


def nhwc_to_nchw(tensors):
    return [t.permute(0, 3, 1, 2) for t in tensors]


def nchw_to_nhwc(tensors):
    return [t.permute(0, 2, 3, 1) for t in tensors]


def flownet_s(inputs, channel_mult=1, full_res=False, _scope=None):
    """Given stacked inputs, returns flow predictions in decreasing resolution (FlowNetSimple)."""
    s = _scope
    x = conv_ops.network_input(inputs)
    conv1 = s.conv(x, 'conv1', 2)
    half = lambda v: -(-v // 2)
    h2, w2 = half(conv1.shape[2]), half(conv1.shape[3])
    cats = _decoder_cats(s, x, x.shape[0], (half(h2), half(w2)), (h2, w2), s.cout('conv2'))
    first = (lambda lvl: cats[lvl].slots[0]) if cats else (lambda lvl: None)
    conv2 = s.conv(conv1, 'conv2', 2, out=first(2))
    conv3 = s.conv(conv2, 'conv3', 2)
    conv3 = conv_ops.backward_point(conv3, s.p + 'trunk')
    conv3_1 = s.conv(conv3, 'conv3_1', out=first(3))
    conv4 = s.conv(conv3_1, 'conv4', 2)
    conv4_1 = s.conv(conv4, 'conv4_1', out=first(4))
    conv5 = s.conv(conv4_1, 'conv5', 2)
    conv5_1 = s.conv(conv5, 'conv5_1', out=first(5))
    conv6 = s.conv(conv5_1, 'conv6', 2)
    conv6_1 = s.conv(conv6, 'conv6_1')
    res = _flownet_upconv(s, conv6_1, conv5_1, conv4_1, conv3_1, conv2, conv1, x,
                          channel_mult=channel_mult, full_res=full_res, cats=cats)
    return nchw_to_nhwc(res)


def flownet_c_features(im, channel_mult=1, reuse=None, _scope=None, _conv2_out=None):
    s = _scope
    x = conv_ops.network_input(im)
    conv1 = s.conv(x, 'conv1', 2)
    conv2 = s.conv(conv1, 'conv2', 2, out=_conv2_out)       # (its slot in the decoder's concat2 buffer, if any)
    conv3 = s.conv(conv2, 'conv3', 2)
    return conv1, conv2, conv3


def _flownet_c_trunk(s, conv_redir_and_corr, conv2_a, channel_mult, full_res, cats=None):
    x = conv_ops.backward_point(conv_redir_and_corr, s.p + 'trunk')   # conv3_1 .. conv6_1 complete behind this point
    if cats is None:
        cats = _decoder_cats(s, x, x.shape[0], (x.shape[2], x.shape[3]), (conv2_a.shape[2], conv2_a.shape[3]),
                             conv2_a.shape[1])
    first = (lambda lvl: cats[lvl].slots[0]) if cats else (lambda lvl: None)
    conv3_1 = s.conv(x, 'conv3_1', out=first(3))
    conv4 = s.conv(conv3_1, 'conv4', 2)
    conv4_1 = s.conv(conv4, 'conv4_1', out=first(4))
    conv5 = s.conv(conv4_1, 'conv5', 2)
    conv5_1 = s.conv(conv5, 'conv5_1', out=first(5))
    conv6 = s.conv(conv5_1, 'conv6', 2)
    conv6_1 = s.conv(conv6, 'conv6_1')
    res = _flownet_upconv(s, conv6_1, conv5_1, conv4_1, conv3_1, conv2_a,
                          channel_mult=channel_mult, full_res=full_res, cats=cats)
    return nchw_to_nhwc(res)


class _ConcatCL(torch.autograd.Function):
    """Channel concat written straight into ONE channels_last buffer.

    forward: each source (dense, NCHW or a channel-sliced view) is read once -- no intermediate
    concat in another layout followed by a layout transform.  backward: the gradients are channel
    (and batch) slices of the incoming gradient, returned as VIEWS.  (Building the buffer with
    ``out[:, a:b] = t`` costs one full-size clone of the gradient per assignment in autograd's
    CopySlices backward -- 14 % of the step when profiled.)

    Inputs: ``n_first`` tensors concatenated along C, then optionally tensors that are first
    concatenated along N and appended along C (the two correlation directions of FlowNetC)."""

    @staticmethod
    def forward(ctx, n_first, buf, *tensors):
        first, second = tensors[:n_first], tensors[n_first:]
        n = first[0].shape[0]
        c = sum(t.shape[1] for t in first) + (second[0].shape[1] if second else 0)
        h, w = first[0].shape[2], first[0].shape[3]
        # NHWC buffer whose pixel pitch is a multiple of 4 floats (16 bytes): the tensor-core conv
        # kernels read channel slices of it in place through TMA tensor maps (csrc/tc_conv.cu); the
        # returned tensor is the [:, :c] view (the 1..3 slack channels are never read).  ``buf``: the
        # buffer was allocated up front and some members already live in their slot (written there by
        # the producing kernel's epilogue) -- those are not copied.
        if buf is None:
            buf = torch.empty((n, h, w, (c + 3) // 4 * 4), device=first[0].device, dtype=first[0].dtype)
        assert tuple(buf.shape) == (n, h, w, (c + 3) // 4 * 4)
        out = buf[..., :c].permute(0, 3, 1, 2)
        spans, off = [], 0
        for t in first:
            slot = out[:, off:off + t.shape[1]]
            if not (t.data_ptr() == slot.data_ptr() and t.stride() == slot.stride()):
                slot.copy_(t)
            spans.append((0, n, off, off + t.shape[1]))
            off += t.shape[1]
        b0 = 0
        for t in second:
            out[b0:b0 + t.shape[0], off:].copy_(t)
            spans.append((b0, b0 + t.shape[0], off, c))
            b0 += t.shape[0]
        ctx.spans = spans
        ctx.gen = conv_ops._generation
        # keys of the members as their other consumers see them (pointer + shape), for the gradient slots
        ctx.member_keys = [(t.data_ptr(), tuple(t.shape)) for t in tensors]
        return out

    @staticmethod
    def backward(ctx, g):
        views = tuple(g[b0:b1, c0:c1] for (b0, b1, c0, c1) in ctx.spans)
        # a member's other consumers (conv5_1 also feeds conv6) add their input gradient into this view
        # instead of handing autograd a second tensor to sum (conv_ops: gradient slots)
        for key, v in zip(ctx.member_keys, views):
            conv_ops.grad_slot_put(ctx.gen, key, v)
        return (None, None) + views


def _concat_channels_last(first, second_batch_parts=None, buf=None):
    return _ConcatCL.apply(len(first), buf, *(list(first) + list(second_batch_parts or [])))


def _cat_c(tensors, buf=None):
    """tf.concat(tensors, 1) of NCHW-shaped tensors (``buf``: pre-allocated NHWC destination, see _Cat)."""
    if conv_ops.tc_active(tensors[0]):
        return _concat_channels_last(list(tensors), buf=buf)
    return torch.cat(tensors, 1)


FUSED_TRUNK_INPUT = True      # tests switch it off to compare with the unfused correlation + concat


def _trunk_input_bidir(cs, conv3_ab, kw):
    """concat([conv_redir(conv3), correlation]) of both directions (batch [a|b] against [b|a]) in one NHWC
    buffer: conv_redir's epilogue writes its channel slice, the two cost volumes follow it (ops.
    correlation_bidir_concat).  None when the tiled correlation kernel does not serve the shape."""
    from ..ops import correlation_bidir_concat, _corr_attrs
    from ... import _native
    from . import tc_conv
    n2, C, H, W = conv3_ab.shape
    attrs = _corr_attrs(kw)
    if n2 % 2 or _native.lib().unflow_correlation_fwd_path(C, H, W, *attrs) != 1 or not tc_conv.supported(conv3_ab):
        return None
    md, s2 = attrs[1], attrs[4]
    D = (2 * (md // s2) + 1) ** 2
    c0 = cs.cout('conv_redir')
    buf = torch.empty((n2, H, W, (c0 + D + 3) // 4 * 4), device=conv3_ab.device, dtype=torch.float32)
    conv_redir = cs.conv(conv3_ab, 'conv_redir', out=buf[..., :c0].permute(0, 3, 1, 2))
    if conv_redir.data_ptr() != buf.data_ptr():
        raise RuntimeError("conv_redir did not write into its concat slot")
    return correlation_bidir_concat(buf, c0, conv3_ab, [conv_redir], **kw)


def flownet_c(conv3_a, conv3_b, conv2_a, channel_mult=1, full_res=False, _scope=None):
    """Given two feature maps, returns flow predictions in decreasing resolution (FlowNetCorr)."""
    s = _scope
    corr = correlation(conv3_a, conv3_b,
                       pad=20, kernel_size=1, max_displacement=20, stride_1=1, stride_2=2)
    conv_redir = s.conv(conv3_a, 'conv_redir')
    if conv_ops.tc_active(conv_redir):
        trunk_in = _concat_channels_last([conv_redir], [corr])
    else:
        trunk_in = torch.cat([conv_redir, corr], 1)
    return _flownet_c_trunk(s, trunk_in, conv2_a, channel_mult, full_res)


def flownet(im1, im2, flownet_spec='S', full_resolution=False, train_all=False,
            backward_flow=False, variables=None):
    """Reference flownet.py:14-81.  Returns ``flows_fw`` (and ``flows_bw``): one entry per
    network in the stack, each a list [flow2, flow3, flow4, flow5, flow6] of NHWC tensors.

    ``variables``: FlowNetVariables (default: the module-level store, created on first use, as
    TF creates variables on first graph construction)."""
    B, height, width, _ = im1.shape
    flownet_num = len(flownet_spec)
    assert flownet_num > 0
    conv_ops.new_forward_generation()
    if variables is None:
        variables = get_variables(flownet_spec, full_resolution, device=im1.device)
    flows_fw = []
    flows_bw = []
    for i, name in enumerate(flownet_spec):
        assert name in ('C', 'c', 'S', 's')
        channel_mult = 1 if name in ('C', 'S') else 3 / 8
        full_res = full_resolution and i == flownet_num - 1
        root = _Scope(variables, '' if i == 0 else 'stack_%d_flownet/' % i)

        if name.lower() == 'c':
            assert i == 0, 'FlowNetS must be used for refinement networks'
            fs = root.sub('flownet_c_features')
            cs = root.sub('flownet_c')
            if backward_flow:
                # both images through the shared feature extractor as one 2B batch; the decoder's concat
                # buffers exist up front so that conv2 is born in its concat2 slot (no 126 MB copy later)
                half = lambda v: -(-v // 2)
                hw2 = (half(half(height)), half(half(width)))
                cats = _decoder_cats(cs, im1, 2 * B, (half(hw2[0]), half(hw2[1])), hw2, fs.cout('conv2'))
                _, conv2_ab, conv3_ab = flownet_c_features(torch.cat([im1, im2], 0),
                                                           channel_mult=channel_mult, _scope=fs,
                                                           _conv2_out=cats[2].slots[0] if cats else None)
                conv3_a, conv3_b = conv3_ab[:B], conv3_ab[B:]
                kw = dict(pad=20, kernel_size=1, max_displacement=20, stride_1=1, stride_2=2)
                trunk_in = (_trunk_input_bidir(cs, conv3_ab, kw)
                            if FUSED_TRUNK_INPUT and conv_ops.tc_active(conv3_ab) else None)
                if trunk_in is not None:
                    pass        # conv_redir and both cost volumes written into one NHWC buffer (ops.py)
                else:
                    # both cost volumes from one pass over the features (the reverse one is a re-indexing)
                    if conv3_a.is_cuda:
                        corr_ab, corr_ba = correlation_bidir(conv3_a, conv3_b, **kw)
                    else:   # (CPU: only reachable with the op swapped for a stand-in, as the host-logic tests do)
                        corr_ab, corr_ba = correlation(conv3_a, conv3_b, **kw), correlation(conv3_b, conv3_a, **kw)
                    conv_redir = cs.conv(conv3_ab, 'conv_redir')
                    if conv_ops.tc_active(conv_redir):
                        trunk_in = _concat_channels_last([conv_redir], [corr_ab, corr_ba])
                    else:
                        trunk_in = torch.cat([conv_redir, torch.cat([corr_ab, corr_ba], 0)], 1)
                flows = _flownet_c_trunk(cs, trunk_in, conv2_ab, channel_mult, full_res, cats=cats)
                flows_fw.append([f[:B] for f in flows])
                flows_bw.append([f[B:] for f in flows])
            else:
                _, conv2_a, conv3_a = flownet_c_features(im1, channel_mult=channel_mult, _scope=fs)
                _, conv2_b, conv3_b = flownet_c_features(im2, channel_mult=channel_mult, reuse=True,
                                                         _scope=fs)
                flows_fw.append(flownet_c(conv3_a, conv3_b, conv2_a, full_res=full_res,
                                          channel_mult=channel_mult, _scope=cs))
        else:
            ss = root.sub('flownet_s')

            def _inputs(a, b, flow=None):
                if flow is not None:
                    flow = tf_image.resize_bilinear(flow, [height, width]) * 4 * FLOW_SCALE
                    warp = image_warp(b, flow)
                    diff = torch.abs(warp - a)
                    if not train_all:
                        flow, warp, diff = flow.detach(), warp.detach(), diff.detach()
                    return torch.cat([a, b, flow, warp, diff], 3)
                return torch.cat([a, b], 3)

            stacked = len(flows_fw) > 0
            if backward_flow:
                prev_fw = flows_fw[-1][0] if stacked else None
                prev_bw = flows_bw[-1][0] if stacked else None
                both = torch.cat([_inputs(im1, im2, prev_fw), _inputs(im2, im1, prev_bw)], 0)
                flows = flownet_s(both, full_res=full_res, channel_mult=channel_mult, _scope=ss)
                flows_fw.append([f[:B] for f in flows])
                flows_bw.append([f[B:] for f in flows])
            else:
                prev_fw = flows_fw[-1][0] if stacked else None
                flows_fw.append(flownet_s(_inputs(im1, im2, prev_fw), full_res=full_res,
                                          channel_mult=channel_mult, _scope=ss))

    if backward_flow:
        return flows_fw, flows_bw
    return flows_fw
