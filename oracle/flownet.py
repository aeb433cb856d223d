"""CPU restatement of the reference FlowNetC / FlowNetS / stacked model (TEST INFRASTRUCTURE ONLY).

Follows /root/reference/src/e2eflow/core/flownet.py (whole file).  Pinned
against that file itself, executed unmodified under the TensorFlow-API stand-in
of tests/golden/ (every output of every network for specs c / s / cs, and the
variable names / shapes the graph asks for: tests/test_oracle_vs_reference_run.py).
PARITY UNPINNED below that: the reference has no test for the model and TF1 /
slim cannot run here, so the TF primitives (SAME padding, conv2d_transpose,
legacy resize_bilinear) are restated in oracle/tf_compat.py from their
documentation.

Variables are passed explicitly as a dict  TF-variable-name -> tensor in TF
layout (conv ``weights``: [kh,kw,in,out]; conv2d_transpose ``weights``:
[kh,kw,out,in]; ``biases``: [out]) -- the checkpoint contract of the
reference (train.py:23-65, scopes flownet.py:30-75).

The graph runs in the dtype and on the device of its inputs (the variables are cast to them), so the
same restatement serves as a float64 GPU reference.  The two custom ops it calls are the module
attributes ``correlation`` and ``image_warp``: the CPU float32 ops by default, replaceable by ops of
another precision (tests/test_gpu_float64_network.py), as is the activation ``leaky_relu``.
"""
import torch

from . import ops as _ops
from . import tf_compat as tfc
from .image_warp import image_warp

FLOW_SCALE = 5.0  # flownet.py:11


def correlation(in0, in1):
    """The FlowNetC cost volume with the reference's attributes (flownet.py:209-211)."""
    return _ops.correlation(in0, in1, pad=20, kernel_size=1, max_displacement=20, stride_1=1, stride_2=2)


def _leaky_relu(x):  # flownet.py:84-86
    return torch.maximum(0.1 * x, x)


def leaky_relu(x, scope):
    """The activation of layer ``scope``; replaceable (e.g. by one that takes its side of the kink from another
    run of the network)."""
    return _leaky_relu(x)


def _var(t, like):
    return torch.as_tensor(t).to(dtype=like.dtype, device=like.device)


class _Scope:
    def __init__(self, variables, prefix):
        self.v = variables
        self.p = prefix

    def sub(self, name):
        return _Scope(self.v, self.p + name + '/')

    def conv(self, x, name, stride=1, act=True):
        w = _var(self.v[self.p + name + '/weights'], x).permute(3, 2, 0, 1).contiguous()
        b = _var(self.v[self.p + name + '/biases'], x)
        y = tfc.conv2d_same(x, w, b, stride)
        return leaky_relu(y, self.p + name) if act else y

    def deconv(self, x, name, act=True):
        w = _var(self.v[self.p + name + '/weights'], x).permute(3, 2, 0, 1).contiguous()
        b = _var(self.v[self.p + name + '/biases'], x)
        y = tfc.conv2d_transpose_same(x, w, b, 2)
        return leaky_relu(y, self.p + name) if act else y


def _flownet_upconv(s, conv6_1, conv5_1, conv4_1, conv3_1, conv2, conv1=None, inputs=None,
                    full_res=False):  # flownet.py:89-155
    flow6 = s.conv(conv6_1, 'flow6', act=False)
    deconv5 = s.deconv(conv6_1, 'deconv5')
    flow6_up5 = s.deconv(flow6, 'flow6_up5', act=False)
    concat5 = torch.cat([conv5_1, deconv5, flow6_up5], 1)
    flow5 = s.conv(concat5, 'flow5', act=False)

    deconv4 = s.deconv(concat5, 'deconv4')
    flow5_up4 = s.deconv(flow5, 'flow5_up4', act=False)
    concat4 = torch.cat([conv4_1, deconv4, flow5_up4], 1)
    flow4 = s.conv(concat4, 'flow4', act=False)

    deconv3 = s.deconv(concat4, 'deconv3')
    flow4_up3 = s.deconv(flow4, 'flow4_up3', act=False)
    concat3 = torch.cat([conv3_1, deconv3, flow4_up3], 1)
    flow3 = s.conv(concat3, 'flow3', act=False)

    deconv2 = s.deconv(concat3, 'deconv2')
    flow3_up2 = s.deconv(flow3, 'flow3_up2', act=False)
    concat2 = torch.cat([conv2, deconv2, flow3_up2], 1)
    flow2 = s.conv(concat2, 'flow2', act=False)

    flows = [flow2, flow3, flow4, flow5, flow6]
    if full_res:
        f = s.sub('full_res')
        deconv1 = f.deconv(concat2, 'deconv1')
        flow2_up1 = f.deconv(flow2, 'flow2_up1', act=False)
        concat1 = torch.cat([conv1, deconv1, flow2_up1], 1)
        flow1 = f.conv(concat1, 'flow1', act=False)
        deconv0 = f.deconv(concat1, 'deconv0')
        flow1_up0 = f.deconv(flow1, 'flow1_up0', act=False)
        concat0 = torch.cat([inputs, deconv0, flow1_up0], 1)
        flow0 = f.conv(concat0, 'flow0', act=False)
        flows = [flow0, flow1] + flows
    return flows


def _nhwc(ts):
    return [t.permute(0, 2, 3, 1) for t in ts]


def flownet_s(s, inputs, full_res=False):  # flownet.py:166-192
    x = inputs.permute(0, 3, 1, 2)
    conv1 = s.conv(x, 'conv1', 2)
    conv2 = s.conv(conv1, 'conv2', 2)
    conv3 = s.conv(conv2, 'conv3', 2)
    conv3_1 = s.conv(conv3, 'conv3_1')
    conv4 = s.conv(conv3_1, 'conv4', 2)
    conv4_1 = s.conv(conv4, 'conv4_1')
    conv5 = s.conv(conv4_1, 'conv5', 2)
    conv5_1 = s.conv(conv5, 'conv5_1')
    conv6 = s.conv(conv5_1, 'conv6', 2)
    conv6_1 = s.conv(conv6, 'conv6_1')
    return _nhwc(_flownet_upconv(s, conv6_1, conv5_1, conv4_1, conv3_1, conv2, conv1, x,
                                 full_res=full_res))


def flownet_c_features(s, im):  # flownet.py:195-206
    x = im.permute(0, 3, 1, 2)
    conv1 = s.conv(x, 'conv1', 2)
    conv2 = s.conv(conv1, 'conv2', 2)
    conv3 = s.conv(conv2, 'conv3', 2)
    return conv1, conv2, conv3


def flownet_c(s, conv3_a, conv3_b, conv2_a, full_res=False):  # flownet.py:209-237
    corr = correlation(conv3_a, conv3_b)
    conv_redir = s.conv(conv3_a, 'conv_redir')
    conv3_1 = s.conv(torch.cat([conv_redir, corr], 1), 'conv3_1')
    conv4 = s.conv(conv3_1, 'conv4', 2)
    conv4_1 = s.conv(conv4, 'conv4_1')
    conv5 = s.conv(conv4_1, 'conv5', 2)
    conv5_1 = s.conv(conv5, 'conv5_1')
    conv6 = s.conv(conv5_1, 'conv6', 2)
    conv6_1 = s.conv(conv6, 'conv6_1')
    # NB the reference passes no conv1/inputs here, so full_res is unusable for 'C' (flownet.py:235-236)
    return _nhwc(_flownet_upconv(s, conv6_1, conv5_1, conv4_1, conv3_1, conv2_a, full_res=full_res))


def flownet(variables, im1, im2, flownet_spec='S', full_resolution=False, train_all=False,
            backward_flow=False):  # flownet.py:14-81
    B, H, W, _ = im1.shape
    n = len(flownet_spec)
    assert n > 0
    flows_fw, flows_bw = [], []
    for i, name in enumerate(flownet_spec):
        assert name in ('C', 'c', 'S', 's')
        full_res = full_resolution and i == n - 1
        root = _Scope(variables, '' if i == 0 else 'stack_%d_flownet/' % i)
        if name.lower() == 'c':
            assert i == 0, 'FlowNetS must be used for refinement networks'
            fs = root.sub('flownet_c_features')
            _, conv2_a, conv3_a = flownet_c_features(fs, im1)
            _, conv2_b, conv3_b = flownet_c_features(fs, im2)
            cs = root.sub('flownet_c')
            flows_fw.append(flownet_c(cs, conv3_a, conv3_b, conv2_a, full_res=full_res))
            if backward_flow:
                flows_bw.append(flownet_c(cs, conv3_b, conv3_a, conv2_b, full_res=full_res))
        else:
            ss = root.sub('flownet_s')

            def _net(a, b, flow=None):
                if flow is not None:
                    flow = tfc.resize_bilinear_legacy(flow, [H, W]) * 4 * FLOW_SCALE
                    warp = image_warp(b, flow)
                    diff = torch.abs(warp - a)
                    if not train_all:
                        flow, warp, diff = flow.detach(), warp.detach(), diff.detach()
                    inputs = torch.cat([a, b, flow, warp, diff], 3)
                else:
                    inputs = torch.cat([a, b], 3)
                return flownet_s(ss, inputs, full_res=full_res)

            stacked = len(flows_fw) > 0
            prev_fw = flows_fw[-1][0] if stacked else None
            prev_bw = flows_bw[-1][0] if (stacked and backward_flow) else None
            flows_fw.append(_net(im1, im2, prev_fw))
            if backward_flow:
                flows_bw.append(_net(im2, im1, prev_bw))
    if backward_flow:
        return flows_fw, flows_bw
    return flows_fw


# ---------------------------------------------------------------------------
# Variable inventory (shapes in TF layout) -- what slim would create for a spec.
# ---------------------------------------------------------------------------
def _upconv_shapes(prefix, m, in6, c5, c4, c3, c2, c1=None, c0=None, full_res=False, ch=2):
    out = {}

    def conv(name, k, cin, cout):
        out[prefix + name + '/weights'] = (k, k, cin, cout)
        out[prefix + name + '/biases'] = (cout,)

    def deconv(name, cin, cout):
        out[prefix + name + '/weights'] = (4, 4, cout, cin)
        out[prefix + name + '/biases'] = (cout,)

    conv('flow6', 3, in6, ch)
    deconv('deconv5', in6, int(512 * m))
    deconv('flow6_up5', ch, ch)
    cat5 = c5 + int(512 * m) + ch
    conv('flow5', 3, cat5, ch)
    deconv('deconv4', cat5, int(256 * m))
    deconv('flow5_up4', ch, ch)
    cat4 = c4 + int(256 * m) + ch
    conv('flow4', 3, cat4, ch)
    deconv('deconv3', cat4, int(128 * m))
    deconv('flow4_up3', ch, ch)
    cat3 = c3 + int(128 * m) + ch
    conv('flow3', 3, cat3, ch)
    deconv('deconv2', cat3, int(64 * m))
    deconv('flow3_up2', ch, ch)
    cat2 = c2 + int(64 * m) + ch
    conv('flow2', 3, cat2, ch)
    if full_res:
        p = 'full_res/'
        deconv(p + 'deconv1', cat2, int(32 * m))
        deconv(p + 'flow2_up1', ch, ch)
        cat1 = c1 + int(32 * m) + ch
        conv(p + 'flow1', 3, cat1, ch)
        deconv(p + 'deconv0', cat1, int(16 * m))
        deconv(p + 'flow1_up0', ch, ch)
        cat0 = c0 + int(16 * m) + ch
        conv(p + 'flow0', 3, cat0, ch)
    return out


def variable_shapes(flownet_spec='S', full_resolution=False):
    shapes = {}
    n = len(flownet_spec)
    for i, name in enumerate(flownet_spec):
        m = 1 if name in ('C', 'S') else 3 / 8
        full_res = full_resolution and i == n - 1
        root = '' if i == 0 else 'stack_%d_flownet/' % i

        def conv(prefix, nm, k, cin, cout):
            shapes[prefix + nm + '/weights'] = (k, k, cin, cout)
            shapes[prefix + nm + '/biases'] = (cout,)

        c64, c128, c256, c512, c1024 = (int(64 * m), int(128 * m), int(256 * m), int(512 * m),
                                        int(1024 * m))
        if name.lower() == 'c':
            f = root + 'flownet_c_features/'
            conv(f, 'conv1', 7, 3, c64)
            conv(f, 'conv2', 5, c64, c128)
            conv(f, 'conv3', 5, c128, c256)
            c = root + 'flownet_c/'
            conv(c, 'conv_redir', 1, c256, int(32 * m))
            conv(c, 'conv3_1', 3, int(32 * m) + 441, c256)
            tail = c
        else:
            s = root + 'flownet_s/'
            cin = 6 if i == 0 else 14
            conv(s, 'conv1', 7, cin, c64)
            conv(s, 'conv2', 5, c64, c128)
            conv(s, 'conv3', 5, c128, c256)
            conv(s, 'conv3_1', 3, c256, c256)
            tail = s
        conv(tail, 'conv4', 3, c256, c512)
        conv(tail, 'conv4_1', 3, c512, c512)
        conv(tail, 'conv5', 3, c512, c512)
        conv(tail, 'conv5_1', 3, c512, c512)
        conv(tail, 'conv6', 3, c512, c1024)
        conv(tail, 'conv6_1', 3, c1024, c1024)
        c0 = (6 if i == 0 else 14) if name.lower() == 's' else None
        shapes.update(_upconv_shapes(tail, m, c1024, c512, c512, c256, c128, c64, c0,
                                     full_res=full_res))
    return shapes


def init_variables(flownet_spec='S', full_resolution=False, seed=1234):
    """Fixed-seed N(0, sqrt(2/fan_in)) weights, zero biases (SURVEY.md 8d synthetic weights)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for name, shape in variable_shapes(flownet_spec, full_resolution).items():
        if name.endswith('/biases'):
            out[name] = torch.zeros(shape)
        else:
            kh, kw, a, b = shape
            # fan_in in TF's variance_scaling is kh*kw*shape[-2]
            fan_in = kh * kw * a
            out[name] = torch.randn(shape, generator=g) * (2.0 / fan_in) ** 0.5
    return out
