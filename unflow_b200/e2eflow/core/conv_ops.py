"""conv / deconv layers of the FlowNet stacks with a selectable arithmetic mode.

'fp32'    plain cuDNN float32 (what the reference's slim.conv2d computes, flownet.py:174-233);
          no tensor cores.
'3xtf32'  the same contraction on the tensor cores at fp32-level accuracy (the default of bench.py and the
          trainer): every operand is split x = hi + lo (hi = TF32-rounded, lo = exact residual) and
          lo*hi' + hi*lo' + hi*hi' is accumulated by the hand-written wgmma kernels (csrc/tc_conv.cu: forward
          and input gradient, csrc/tc_wgrad.cu: weight gradient, csrc/narrow_conv*.cu: the 2-channel flow
          heads in exact fp32) with the K loop cut into chunks that are summed in fp32 registers: 1.8e-6 of
          max|y| against float64 per layer, and the same 1e-4 flow tolerance against the fp32 oracle as the
          plain fp32 path.  Layers these kernels do not serve (tensors that are not NHWC / 16-byte aligned) fall
          back to cuDNN TF32 convolutions fed the split operands (csrc/split.cu, the round-1 path).
'tf32'    single-pass TF32 (reduced precision; never used for parity or the headline number).
"""
import torch
import torch.nn.functional as F
from torch.nn import grad as nngrad

from ... import _native
from ..._native import check

_MODE = 'fp32'


def set_mode(mode):
    global _MODE
    if mode not in ('fp32', '3xtf32', 'tf32'):
        raise ValueError("conv precision must be 'fp32', '3xtf32' or 'tf32'")
    _MODE = mode
    # the flag is process-global because autograd runs the backward convolutions later
    torch.backends.cudnn.allow_tf32 = mode != 'fp32'
    torch.backends.cuda.matmul.allow_tf32 = False
    return mode


def get_mode():
    return _MODE


LRELU_SLOPE = 0.1   # _leaky_relu: tf.maximum(0.1 * x, x)  (reference flownet.py:84-86)


# ---------------------------------------------------------------------------------------------
# Backward checkpoints: the network marks a few activations ("everything created after this point
# has finished its backward pass once the gradient arrives here"); the data-parallel trainer hangs
# the all-reduce of the corresponding slice of the flat gradient buffer on them, so the reduction
# of the decoder / encoder gradients overlaps the rest of the backward pass (core/train.py).
# ---------------------------------------------------------------------------------------------
_backward_point_cb = None

# ---------------------------------------------------------------------------------------------
# Gradient slots: an activation with several consumers (conv5_1 feeds conv6 AND concat5; a concat buffer
# feeds the next deconv AND a flow head) receives one gradient per consumer, and autograd adds them with a
# generic strided elementwise kernel (0.5 ms per step in the CUPTI table).  The tensor-core input-gradient
# kernels can ADD into an existing buffer in their epilogue, so the first producer of a gradient for an
# activation registers its buffer here and later producers accumulate into it and hand autograd None
# ("no further contribution").  Keys are (forward generation, data pointer, shape): the generation counter
# advances with every forward pass of the network, so buffers of an older graph are never picked up.
# ---------------------------------------------------------------------------------------------
_generation = 0
_grad_slots = {}
_GRAD_SLOTS = __import__('os').environ.get('UNFLOW_GRAD_SLOTS', '1') != '0'


def new_forward_generation():
    """Called at the start of every network forward pass."""
    global _generation
    _generation += 1
    for g in [g for g in _grad_slots if g < _generation - 1]:
        del _grad_slots[g]
    return _generation


def _slot_key(x):
    return (x.data_ptr(), tuple(x.shape))


def grad_slot_get(gen, x, key=None):
    return _grad_slots.get(gen, {}).get(key if key is not None else _slot_key(x)) if _GRAD_SLOTS else None


def grad_slot_put(gen, key_or_tensor, g):
    if _GRAD_SLOTS:
        key = key_or_tensor if isinstance(key_or_tensor, tuple) else _slot_key(key_or_tensor)
        _grad_slots.setdefault(gen, {})[key] = g


def set_backward_point_callback(fn):
    """fn(name) is called from inside the backward pass; None removes it."""
    global _backward_point_cb
    _backward_point_cb = fn


class _BackwardPoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, name):
        ctx.name = name
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        if _backward_point_cb is not None:
            _backward_point_cb(ctx.name)
        return g, None


def backward_point(x, name):
    """Identity; with a callback installed and a differentiable ``x`` it reports when the backward pass
    comes back through this activation."""
    if _backward_point_cb is None or not x.requires_grad:
        return x
    return _BackwardPoint.apply(x, name)


def _bias_act_(y, b):
    """y = leaky_relu(y + b) in place (one pass instead of bias add + activation)."""
    N, C, H, W = y.shape
    assert y.is_contiguous(memory_format=torch.channels_last) and C % 4 == 0
    with torch.cuda.device(y.device):
        check(_native.lib().unflow_bias_lrelu(y.data_ptr(), b.data_ptr(), N * H * W, C, LRELU_SLOPE,
                                              torch.cuda.current_stream().cuda_stream), "bias_lrelu")
    return y


def _bias_grad(g, act):
    """sum over pixels of g * lrelu'(act) (act None: plain sum) -> [C]."""
    N, C, H, W = g.shape
    gb = torch.empty(C, device=g.device, dtype=torch.float32)
    sN, sC, sH, sW = g.stride()
    with torch.cuda.device(g.device):
        check(_native.lib().unflow_bias_grad_lrelu(g.data_ptr(), sN, sC, sH, sW,
                                                   act.data_ptr() if act is not None else None, gb.data_ptr(),
                                                   N, C, H, W, LRELU_SLOPE,
                                                   torch.cuda.current_stream().cuda_stream), "bias_grad_lrelu")
    return gb


def _round4(c):
    return (c + 3) // 4 * 4


def _operand(x, order, concat_batch=False, c_pad=None, n_out=None, pads=(0, 0, 0, 0), act=None):
    """One pass of csrc/split.cu: logical [N,C,H,W] (any strides) -> the dense channels_last TF32
    operand [N_out, 3*C_pad, Hp, Wp] (channel concat) or [3*N_out, C_pad, Hp, Wp] (batch concat)."""
    N, C, H, W = x.shape
    c_pad = _round4(C) if c_pad is None else c_pad
    n_out = N if n_out is None else n_out
    pt, pb, pl, pr = pads
    Hp, Wp = H + pt + pb, W + pl + pr
    out = torch.empty((3 * n_out * Hp * Wp * c_pad,), device=x.device, dtype=torch.float32)
    sN, sC, sH, sW = x.stride()
    from ..ops import kernel_timer
    with torch.cuda.device(x.device), kernel_timer.span("conv_operand", 4 * x.numel() + 4 * out.numel()):
        check(_native.lib().unflow_conv_operand_tf32(
            x.data_ptr(), out.data_ptr(), N, C, H, W, sN, sC, sH, sW, n_out, c_pad, pt, pb, pl, pr,
            1 if concat_batch else 0, order, act.data_ptr() if act is not None else None, LRELU_SLOPE,
            torch.cuda.current_stream().cuda_stream), "conv_operand_tf32")
    if concat_batch:
        return out.view(3 * n_out, Hp, Wp, c_pad).permute(0, 3, 1, 2)
    return out.view(n_out, Hp, Wp, 3 * c_pad).permute(0, 3, 1, 2)


def _conv_input_grad(input_hw, weight, grad_output, stride):
    """Gradient of ``conv2d(x, weight, stride=stride, padding=0)`` w.r.t. ``x`` ([.., input_hw]).

    Written as the transposed convolution it is (output_padding recovers the rows / columns a
    strided conv leaves unused).  ``torch.nn.grad.conv2d_input`` computes the same thing but hands
    cuDNN a stride-0 placeholder for ``x``; ATen then aligns ``grad_output`` to THAT tensor's
    (NCHW) format and back to the weight's NHWC -- two full copies of the 3x-wide gradient operand
    per layer."""
    sh, sw = (stride, stride) if isinstance(stride, int) else stride
    kh, kw = weight.shape[2], weight.shape[3]
    oph = input_hw[0] - ((grad_output.shape[2] - 1) * sh + kh)
    opw = input_hw[1] - ((grad_output.shape[3] - 1) * sw + kw)
    assert 0 <= oph < max(sh, 1) and 0 <= opw < max(sw, 1), (input_hw, grad_output.shape, stride)
    return F.conv_transpose2d(grad_output, weight, None, stride=(sh, sw), padding=0,
                              output_padding=(oph, opw))


def _pad_bias(b, co_p):
    if b is None or b.shape[0] == co_p:
        return b
    return F.pad(b, (0, co_p - b.shape[0]))


class _Conv3x(torch.autograd.Function):
    """conv2d(pad_same(x), w) + b at fp32-level accuracy on the tensor cores (one TF32 cuDNN conv
    over the channel-concatenated hi/lo operands).  ``pads`` = TF SAME (top, bottom, left, right)."""

    @staticmethod
    def forward(ctx, x, w, b, stride, pads, act):
        Co, Ci = w.shape[0], w.shape[1]
        ci_p, co_p = _round4(Ci), _round4(Co)
        fuse = bool(act) and b is not None and co_p == Co
        xs = _operand(x, 0, c_pad=ci_p, pads=pads)               # [N, 3Ci_p, Hp, Wp]  hi,hi,lo
        ws = _operand(w, 1, c_pad=ci_p, n_out=co_p)              # [Co_p, 3Ci_p, k, k] hi,lo,hi
        if fuse:     # conv -> (bias + leaky ReLU) in one in-place pass
            y = _bias_act_(F.conv2d(xs, ws, None, stride=stride, padding=0), b)
            ctx.save_for_backward(x, w, y)
        else:
            assert not act, "fused activation needs a bias and C_out % 4 == 0"
            y = F.conv2d(xs, ws, _pad_bias(b, co_p), stride=stride, padding=0)
            ctx.save_for_backward(x, w)
        ctx.cfg = (stride, pads, b is not None, ci_p, co_p)
        ctx.fuse = fuse
        return y if co_p == Co else y[:, :Co]

    @staticmethod
    def backward(ctx, g):
        if ctx.fuse:
            x, w, a = ctx.saved_tensors
        else:
            (x, w), a = ctx.saved_tensors, None
        stride, pads, has_b, ci_p, co_p = ctx.cfg
        Co, Ci, k = w.shape[0], w.shape[1], w.shape[2]
        N, _, H, W = x.shape
        pt, pb, pl, pr = pads
        gx = gw = gb = None

        def input_grad():
            gs = _operand(g, 0, c_pad=co_p, act=a)                                 # [N, 3Co_p, ..]
            wt = _operand(w, 1, concat_batch=True, c_pad=ci_p, n_out=co_p)        # [3Co_p, Ci_p, k, k]
            gxp = _conv_input_grad((H + pt + pb, W + pl + pr), wt, gs, stride)
            return gxp[:, :Ci, pt:pt + H, pl:pl + W]

        def weight_grad():
            xb = _operand(x, 0, concat_batch=True, c_pad=ci_p, pads=pads)          # [3N, Ci_p, Hp, Wp]
            gb3 = _operand(g, 1, concat_batch=True, c_pad=co_p, act=a)             # [3N, Co_p, ..]
            gwp = nngrad.conv2d_weight(xb, (co_p, ci_p, k, k), gb3, stride=stride, padding=0)
            return gwp[:Co, :Ci], (gwp,)

        if ctx.needs_input_grad[0]:
            gx = input_grad()
        if ctx.needs_input_grad[1]:
            gw = weight_grad()[0]
        if has_b and ctx.needs_input_grad[2]:
            gb = _bias_grad(g, a)
        return gx, gw, gb, None, None, None


class _Deconv3x(torch.autograd.Function):
    """conv_transpose2d(x, w[in,out,4,4], stride=2, padding=1) + b, same scheme."""

    @staticmethod
    def forward(ctx, x, w, b, act):
        Ci, Co = w.shape[0], w.shape[1]
        ci_p, co_p = _round4(Ci), _round4(Co)
        fuse = bool(act) and b is not None and co_p == Co
        xs = _operand(x, 0, c_pad=ci_p)                                           # [N, 3Ci_p, h, w]
        ws = _operand(w, 1, concat_batch=True, c_pad=co_p, n_out=ci_p)            # [3Ci_p, Co_p, 4, 4]
        if fuse:
            y = _bias_act_(F.conv_transpose2d(xs, ws, None, stride=2, padding=1), b)
            ctx.save_for_backward(x, w, y)
        else:
            assert not act, "fused activation needs a bias and C_out % 4 == 0"
            y = F.conv_transpose2d(xs, ws, _pad_bias(b, co_p), stride=2, padding=1)
            ctx.save_for_backward(x, w)
        ctx.cfg = (b is not None, ci_p, co_p)
        ctx.fuse = fuse
        return y if co_p == Co else y[:, :Co]

    @staticmethod
    def backward(ctx, g):
        if ctx.fuse:
            x, w, a = ctx.saved_tensors
        else:
            (x, w), a = ctx.saved_tensors, None
        has_b, ci_p, co_p = ctx.cfg
        Ci, Co = w.shape[0], w.shape[1]
        gx = gw = gb = None

        def input_grad():
            gs = _operand(g, 0, c_pad=co_p, act=a)                                # [N, 3Co_p, 2h, 2w]
            wc = _operand(w, 1, c_pad=co_p, n_out=ci_p)                           # [Ci_p, 3Co_p, 4, 4]
            gxp = F.conv2d(gs, wc, None, stride=2, padding=1)
            return gxp if ci_p == Ci else gxp[:, :Ci]

        def weight_grad():
            # d/dw of conv_transpose == weight gradient of the conv whose input is g and output x
            gb3 = _operand(g, 0, concat_batch=True, c_pad=co_p, act=a)
            xb = _operand(x, 1, concat_batch=True, c_pad=ci_p)
            gwp = nngrad.conv2d_weight(gb3, (ci_p, co_p, 4, 4), xb, stride=2, padding=1)
            return gwp[:Ci, :Co], (gwp,)

        if ctx.needs_input_grad[0]:
            gx = input_grad()
        if ctx.needs_input_grad[1]:
            gw = weight_grad()[0]
        if has_b and ctx.needs_input_grad[2]:
            gb = _bias_grad(g, a)
        return gx, gw, gb, None


# ---------------------------------------------------------------------------------------------
# Hand-written tensor-core path (csrc/tc_conv.cu): wgmma implicit GEMM, 3xTF32 split in shared
# memory, fused bias / leaky ReLU.  Forward and input gradient; the weight gradient still goes
# through the library path below (round-2 work in progress: csrc/tc_wgrad).
# ---------------------------------------------------------------------------------------------
_TC = __import__('os').environ.get('UNFLOW_TC_CONV', '1') != '0'
_TC_WGRAD = __import__('os').environ.get('UNFLOW_TC_WGRAD', '1') != '0'


def _grad_slot(w):
    """The variable's own gradient buffer when the weight-gradient kernel may accumulate into it directly:
    a leaf whose ``.grad`` already exists in the variable's memory order (the Trainer's views into its flat
    gradient buffer, zeroed by the fused Adam kernel).  The split-K kernel ADDS its partial sums with atomics,
    which is exactly autograd's accumulate semantics -- returning None for that input then saves the zero
    fill of a temporary and the ``grad += temporary`` pass over all 39 M parameters."""
    g = w.grad if (w.is_leaf and w.requires_grad) else None
    if g is None or g.shape != w.shape or g.stride() != w.stride() or g.dtype != torch.float32:
        return None
    return g


def _tc_weight_grad(P, G, w, stride, pad_t, pad_l):
    """dL/dw on csrc/tc_wgrad.cu.  Returns the gradient tensor for autograd, or None when it has been
    accumulated into ``w.grad`` in place (see _grad_slot)."""
    from . import tc_conv
    A, B, kh, kw = w.shape
    want = (kh * kw * B, 1, kw * B, B)
    in_order = all(n == 1 or s_ == t for n, s_, t in zip(w.shape, w.stride(), want))
    slot = _grad_slot(w) if in_order else None
    if slot is not None:
        tc_conv.wgrad(P, G, slot, stride=stride, kh=kh, kw=kw, pad_t=pad_t, pad_l=pad_l)
        return None
    gw = torch.zeros((A, kh, kw, B), device=w.device, dtype=torch.float32).permute(0, 3, 1, 2)
    return tc_conv.wgrad(P, G, gw, stride=stride, kh=kh, kw=kw, pad_t=pad_t, pad_l=pad_l)


def _tc_ok(x, stride):
    from . import tc_conv
    return (_TC and _MODE == '3xtf32' and x.is_cuda and tc_conv.supported(x)
            and (stride == 1 or (x.shape[2] % 2 == 0 and x.shape[3] % 2 == 0)))


def _khwc(w):
    """The variable in the memory order [dim0][kh][kw][dim1] the weight-plane kernel reads (how
    FlowNetVariables stores it; derived tensors such as the space-to-depth filter are converted)."""
    A, B, kh, kw = w.shape
    want = (kh * kw * B, 1, kw * B, B)
    if all(n == 1 or s == t for n, s, t in zip(w.shape, w.stride(), want)):
        return w
    return w.detach().contiguous(memory_format=torch.channels_last)


def _lrelu_bwd_bias(g, act, want_bias):
    """One pass over the incoming gradient: gpre = g * lrelu'(act) as a dense NHWC tensor and the bias
    gradient sum_pixels gpre.  ``act`` (the layer's output, possibly a channel slice of a concat buffer)
    None: no activation (gpre is g made dense)."""
    from . import tc_conv
    N, C, H, W = g.shape
    dense = tc_conv.nhwc_geometry(g)
    if act is None and not want_bias and dense is not None and dense[4] % 4 == 0 and g.data_ptr() % 16 == 0:
        return g, None
    ap = 0
    if act is not None:
        ga = tc_conv.nhwc_geometry(act)
        if ga is None:
            act = act.contiguous(memory_format=torch.channels_last)
            ga = tc_conv.nhwc_geometry(act)
        ap = ga[4]
    gp = _round4(C)
    gpre = torch.empty((N, H, W, gp), device=g.device, dtype=torch.float32)[..., :C].permute(0, 3, 1, 2)
    gb = torch.empty(C, device=g.device, dtype=torch.float32)
    sN, sC, sH, sW = g.stride()
    with torch.cuda.device(g.device):
        check(_native.lib().unflow_lrelu_bwd_bias(g.data_ptr(), sN, sC, sH, sW,
                                                  act.data_ptr() if act is not None else None, ap,
                                                  gpre.data_ptr(), gp, gb.data_ptr(), N, C, H, W, LRELU_SLOPE,
                                                  torch.cuda.current_stream().cuda_stream), "lrelu_bwd_bias")
    return gpre, gb


def _dest(out, N, C, H, W, device):
    """Where a tensor-core layer writes its output: the caller's slot (a channel slice of a pre-allocated
    concat buffer -- the epilogue stores straight into it, no concat copy later) or a fresh NHWC tensor.
    Returns (tensor to write, tensor to hand to autograd): the latter is a new tensor object over the same
    memory, so autograd never sees it as a view of the buffer."""
    if out is not None:
        assert tuple(out.shape) == (N, C, H, W), (tuple(out.shape), (N, C, H, W))
        # a NEW tensor over the same memory (own version counter -- ``detach()`` would share the buffer's,
        # and the later in-place fill of a neighbouring slot would make autograd reject the saved output)
        alias = torch.empty(0, device=out.device, dtype=out.dtype).set_(
            out.untyped_storage(), out.storage_offset(), out.shape, out.stride())
        return out, alias
    buf = torch.empty((N, H, W, _round4(C)), device=device, dtype=torch.float32)
    y = buf[..., :C].permute(0, 3, 1, 2)
    return y, y


def _input_grad_into_slot(gen, x, launch):
    """Run an input-gradient kernel for activation ``x``: into the gradient buffer another consumer of ``x``
    already registered (epilogue adds; autograd gets None) or into a fresh NHWC buffer that is registered for
    the consumers still to come.  ``launch(dst, accumulate)``."""
    from . import tc_conv
    N, C, H, W = x.shape
    slot = grad_slot_get(gen, x)
    if slot is not None and tuple(slot.shape) == (N, C, H, W) and tc_conv.supported(slot):
        launch(slot, True)
        return None
    buf = torch.empty((N, H, W, _round4(C)), device=x.device, dtype=torch.float32)
    gx = buf[..., :C].permute(0, 3, 1, 2)
    launch(gx, False)
    grad_slot_put(gen, x, gx)
    return gx


class _ConvTC(torch.autograd.Function):
    """slim.conv2d on the hand-written wgmma kernel: y = act(conv(x, w; stride, TF SAME) + b)."""

    @staticmethod
    def forward(ctx, x, w, b, stride, pads, act, out=None):
        from . import tc_conv
        Co, Ci, k = w.shape[0], w.shape[1], w.shape[2]
        N, _, H, W = x.shape
        pt, pb, pl, pr = pads
        Ho, Wo = (H + pt + pb - k) // stride + 1, (W + pl + pr - k) // stride + 1
        dst, y = _dest(out, N, Co, Ho, Wo, x.device)
        planes = tc_conv.split_weights(_khwc(w))
        tc_conv.run(x, planes, dst, mode=0, stride=stride, kh=k, kw=k, pad_t=pt, pad_l=pl,
                    bias=b, act=bool(act))
        ctx.save_for_backward(x, w, y if act else None)
        ctx.cfg = (stride, tuple(pads), b is not None, bool(act))
        ctx.gen = _generation
        return y

    @staticmethod
    def backward(ctx, g):
        from . import tc_conv
        x, w, a = ctx.saved_tensors
        stride, pads, has_b, act = ctx.cfg
        Co, Ci, k = w.shape[0], w.shape[1], w.shape[2]
        N, _, H, W = x.shape
        pt, pb, pl, pr = pads
        gx = gw = gb = None
        gpre, gb_all = _lrelu_bwd_bias(g, a if act else None, has_b and ctx.needs_input_grad[2])
        if has_b and ctx.needs_input_grad[2]:
            gb = gb_all
        if ctx.needs_input_grad[0]:
            # dx = conv_transpose(gpre, w): rows of the GEMM = C_in, contraction = C_out
            gx = _input_grad_into_slot(ctx.gen, x, lambda dst, acc: tc_conv.run(
                gpre, tc_conv.split_weights(_khwc(w), transpose=True), dst, mode=1,
                stride=stride, kh=k, kw=k, pad_t=pt, pad_l=pl, accumulate=acc))
        if ctx.needs_input_grad[1]:
            if _TC_WGRAD and tc_conv.supported(gpre):
                gw = _tc_weight_grad(gpre, x, w, stride, pt, pl)                   # rows C_out, columns C_in
            else:
                ci_p, co_p = _round4(Ci), _round4(Co)
                xb = _operand(x, 0, concat_batch=True, c_pad=ci_p, pads=pads)      # [3N, Ci_p, Hp, Wp]
                gb3 = _operand(gpre, 1, concat_batch=True, c_pad=co_p)             # [3N, Co_p, ..]
                gw = nngrad.conv2d_weight(xb, (co_p, ci_p, k, k), gb3, stride=stride, padding=0)[:Co, :Ci]
        return gx, gw, gb, None, None, None, None


class _ConvWindow(torch.autograd.Function):
    """The first layers (7x7, stride 2, 3 / 6 / 14 input channels) in the row-window form of
    csrc/tc_conv.cu / tc_wgrad.cu: the kw taps of a filter row are one contiguous window of the
    channel-padded image, so the layer is a convolution with kh taps and an 8*Cp-wide contraction.
    ``w_rw`` is the variable in that form (tc_conv.window_weights, differentiable); the input gets no
    gradient (images / detached inputs)."""

    @staticmethod
    def forward(ctx, x, w_rw, b, kh, stride, pads, act):
        from . import tc_conv
        Co = w_rw.shape[0]
        N, _, H, W = x.shape
        pt, pb, pl, pr = pads
        Ho, Wo = (H + pt + pb - kh) // stride + 1, (W + pl + pr - kh) // stride + 1
        xp = tc_conv.window_input(x, pl, stride, Wo)
        buf = torch.empty((N, Ho, Wo, _round4(Co)), device=x.device, dtype=torch.float32)
        y = buf[..., :Co].permute(0, 3, 1, 2)
        tc_conv.run_window(xp, tc_conv.split_weights(_khwc(w_rw)), y, kh=kh, stride=stride, pad_t=pt, bias=b,
                           act=bool(act))
        ctx.save_for_backward(xp, w_rw, y if act else None)
        ctx.cfg = (kh, stride, pt, b is not None, bool(act))
        return y

    @staticmethod
    def backward(ctx, g):
        from . import tc_conv
        xp, w_rw, a = ctx.saved_tensors
        kh, stride, pt, has_b, act = ctx.cfg
        Co = w_rw.shape[0]
        gw = gb = None
        gpre, gb_all = _lrelu_bwd_bias(g, a if act else None, has_b and ctx.needs_input_grad[2])
        if has_b and ctx.needs_input_grad[2]:
            gb = gb_all
        if ctx.needs_input_grad[1]:
            A, B, k1, k2 = w_rw.shape
            gw = torch.zeros((A, k1, k2, B), device=w_rw.device, dtype=torch.float32).permute(0, 3, 1, 2)
            tc_conv.wgrad_window(gpre, xp, gw, kh=kh, stride=stride, pad_t=pt)
        return None, gw, gb, None, None, None, None


_WINDOW = __import__('os').environ.get('UNFLOW_CONV1_WINDOW', '1') != '0'


def _use_window(x, w, stride):
    return (_WINDOW and _TC and _TC_WGRAD and _MODE == '3xtf32' and x.is_cuda and stride in (2, (2, 2))
            and w.shape[2] == w.shape[3] and 5 <= w.shape[2] <= 8 and w.shape[1] <= 16 and w.shape[0] % 4 == 0
            and not x.requires_grad)


class _DeconvTC(torch.autograd.Function):
    """slim.conv2d_transpose(k=4, stride=2, SAME) on the same kernel (four output-parity classes)."""

    @staticmethod
    def forward(ctx, x, w, b, act, out=None):
        from . import tc_conv
        Ci, Co = w.shape[0], w.shape[1]
        N, _, H, W = x.shape
        dst, y = _dest(out, N, Co, 2 * H, 2 * W, x.device)
        planes = tc_conv.split_weights(_khwc(w), transpose=True)
        tc_conv.run(x, planes, dst, mode=1, stride=2, kh=4, kw=4, pad_t=1, pad_l=1, bias=b, act=bool(act))
        ctx.save_for_backward(x, w, y if act else None)
        ctx.cfg = (b is not None, bool(act))
        ctx.gen = _generation
        return y

    @staticmethod
    def backward(ctx, g):
        from . import tc_conv
        x, w, a = ctx.saved_tensors
        has_b, act = ctx.cfg
        Ci, Co = w.shape[0], w.shape[1]
        N, _, H, W = x.shape
        gx = gw = gb = None
        gpre, gb_all = _lrelu_bwd_bias(g, a if act else None, has_b and ctx.needs_input_grad[2])
        if has_b and ctx.needs_input_grad[2]:
            gb = gb_all
        if ctx.needs_input_grad[0]:
            # dx = conv(gpre, w; stride 2, pad 1): rows = C_in (dim 0 of the IOHW variable), contraction = C_out
            gx = _input_grad_into_slot(ctx.gen, x, lambda dst, acc: tc_conv.run(
                gpre, tc_conv.split_weights(_khwc(w)), dst, mode=0, stride=2, kh=4,
                kw=4, pad_t=1, pad_l=1, accumulate=acc))
        if ctx.needs_input_grad[1]:
            if _TC_WGRAD and tc_conv.supported(gpre):
                gw = _tc_weight_grad(x, gpre, w, 2, 1, 1)                          # rows C_in, columns C_out
            else:
                ci_p, co_p = _round4(Ci), _round4(Co)
                gb3 = _operand(gpre, 0, concat_batch=True, c_pad=co_p)
                xb = _operand(x, 1, concat_batch=True, c_pad=ci_p)
                gw = nngrad.conv2d_weight(gb3, (ci_p, co_p, 4, 4), xb, stride=2, padding=1)[:Ci, :Co]
        return gx, gw, gb, None, None


# The narrow kernels serve every 2-channel 3x3 head: the large ones (flow2 / flow3 of a training batch)
# fill the GPU with 16x32-pixel tiles, the coarse ones (flow4 .. flow6: 8 .. 48 tiles) split the input
# channels over several CTAs per tile (csrc/narrow_conv.cu, csplit).  On the tensor-core kernel a head is
# one 32-wide N block with 2 useful columns and a K of 9 x 1026 walked by a handful of CTAs: 0.5 ms per step.
NARROW_MIN_TILES = 1
_NARROW = __import__('os').environ.get('UNFLOW_NARROW_CONV', '1') != '0'


def _narrow_lib():
    return _native.lib()


def _narrow_tiles(N, H, W):
    return N * ((H + 15) // 16) * ((W + 31) // 32)


def _use_narrow(x, w, stride, pads):
    from . import tc_conv
    return (_NARROW and w.shape[0] == 2 and w.shape[2] == 3 and w.shape[3] == 3 and stride in (1, (1, 1))
            and tuple(pads) == (1, 1, 1, 1) and x.shape[1] % 2 == 0 and x.dtype == torch.float32
            and tc_conv.nhwc_geometry(x) is not None        # NHWC memory, possibly a slice of a concat buffer
            and _narrow_tiles(x.shape[0], x.shape[2], x.shape[3]) >= NARROW_MIN_TILES)


def _pixel_pitch(x):
    from . import tc_conv
    return tc_conv.nhwc_geometry(x)[4]


class _NarrowConv3x3(torch.autograd.Function):
    """The 2-channel flow heads (csrc/narrow_conv.cu): forward and weight gradient in exact fp32 on
    the FMA pipes, reading the wide input once; the input gradient (C_in wide) keeps the
    tensor-core path of ``_Conv3x``."""

    @staticmethod
    def forward(ctx, x, w, b):
        N, C, H, W = x.shape
        wl = w if w.is_contiguous(memory_format=torch.channels_last) else \
            w.contiguous(memory_format=torch.channels_last)
        # 4 floats per pixel: the up-sampling deconv that consumes the flow reads it through a TMA tensor map
        y = torch.empty((N, H, W, 4), device=x.device, dtype=torch.float32)[..., :2].permute(0, 3, 1, 2)
        from ..ops import kernel_timer
        with torch.cuda.device(x.device), kernel_timer.span("narrow_conv_fwd", 4 * x.numel() + 4 * y.numel()):
            check(_narrow_lib().unflow_conv3x3_narrow_fwd(
                x.data_ptr(), _pixel_pitch(x), wl.data_ptr(), b.data_ptr() if b is not None else None, y.data_ptr(),
                4, N, H, W, C, 2, torch.cuda.current_stream().cuda_stream), "conv3x3_narrow_fwd")
        ctx.save_for_backward(x, w)
        ctx.has_b = b is not None
        ctx.gen = _generation
        return y

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        N, C, H, W = x.shape
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            from . import tc_conv
            if _TC and tc_conv.supported(x):
                # input gradient (C_in wide) on the tensor-core kernel: contraction over the 2 flow channels
                gd, _ = _lrelu_bwd_bias(g, None, False)
                gx = _input_grad_into_slot(ctx.gen, x, lambda dst, acc: tc_conv.run(
                    gd, tc_conv.split_weights(_khwc(w), transpose=True), dst, mode=1, stride=1, kh=3, kw=3,
                    pad_t=1, pad_l=1, accumulate=acc))
            else:
                ci_p = _round4(C)
                gs = _operand(g, 0, c_pad=4)                                          # [N, 12, H, W]
                wt = _operand(w, 1, concat_batch=True, c_pad=ci_p, n_out=4)           # [12, Ci_p, 3, 3]
                gx = _conv_input_grad((H + 2, W + 2), wt, gs, 1)[:, :C, 1:1 + H, 1:1 + W]
        if ctx.needs_input_grad[1]:
            lib = _narrow_lib()
            ws = torch.empty(lib.unflow_conv3x3_narrow_wgrad_workspace_bytes(N, H, W, C) // 4,
                             device=x.device, dtype=torch.float32)
            gw = torch.empty((2, 3, 3, C), device=x.device, dtype=torch.float32)
            sN, sC, sH, sW = g.stride()
            from ..ops import kernel_timer
            with torch.cuda.device(x.device), kernel_timer.span("narrow_conv_wgrad", 4 * x.numel() + 4 * g.numel()):
                check(lib.unflow_conv3x3_narrow_wgrad(
                    x.data_ptr(), _pixel_pitch(x), g.data_ptr(), sN, sC, sH, sW, gw.data_ptr(), ws.data_ptr(),
                    N, H, W, C, 2, torch.cuda.current_stream().cuda_stream), "conv3x3_narrow_wgrad")
            gw = gw.permute(0, 3, 1, 2)                                           # [2, C, 3, 3], NHWC-ordered
        if ctx.has_b and ctx.needs_input_grad[2]:
            gb = _bias_grad(g, None)
        return gx, gw, gb


# First layers (7x7, stride 2, 3 / 6 / 14 input channels): with so few channels per filter tap cuDNN
# does not pick its sm100 implicit-GEMM kernels but an indexed sm80 one (measured: 0.8 ms fprop,
# 1.4 ms wgrad + 0.6 ms of layout conversions per step).  Folding the stride into the
# channels -- 2x2 pixel blocks become 4*C channels, the 7x7 filter (zero-extended to 8x8) a 4x4
# filter with stride 1 -- is the same sum with a tensor-core-friendly shape (4*C*3 = 36 channels).
S2D_MAX_CHANNELS = 16
_S2D = __import__('os').environ.get('UNFLOW_CONV1_S2D', '1') != '0'


def _use_space_to_depth(x, w, stride):
    return (_S2D and stride in (2, (2, 2)) and w.shape[2] == w.shape[3] and w.shape[2] % 2 == 1
            and w.shape[2] >= 5 and w.shape[1] <= S2D_MAX_CHANNELS)


def space_to_depth_operands(x, w, pads):
    """``conv2d(pad(x, pads), w, stride=2)`` with an odd k x k filter  ==
    ``conv2d(xs, ws, stride=1)`` with the returned operands: ``xs`` [N, 4C, Ho+m-1, Wo+m-1] holds the
    padded input in 2x2 pixel blocks (channel = (dy, dx, c)), ``ws`` [Co, 4C, m, m] the filter
    zero-extended to (k+1) x (k+1) and regrouped the same way, m = (k+1)/2."""
    N, C, H, W = x.shape
    Co, _, k, _ = w.shape
    m = (k + 1) // 2
    pt, pb, pl, pr = pads
    Ho, Wo = (H + pt + pb - k) // 2 + 1, (W + pl + pr - k) // 2 + 1
    Hb, Wb = Ho + m - 1, Wo + m - 1                           # block rows / cols the filter touches
    xp = F.pad(x, (pl, 2 * Wb - W - pl, pt, 2 * Hb - H - pt))  # extra zero row / col under the 8th tap
    xs = xp.permute(0, 2, 3, 1).reshape(N, Hb, 2, Wb, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(N, Hb, Wb, 4 * C)
    xs = xs.permute(0, 3, 1, 2)                               # NCHW-shaped view of NHWC memory
    ws = F.pad(w, (0, 1, 0, 1)).reshape(Co, C, m, 2, m, 2).permute(0, 3, 5, 1, 2, 4).reshape(Co, 4 * C, m, m)
    return xs, ws


def channels_last_active(x):
    """The tensor-core path computes in NHWC (cuDNN's TF32 kernels are NHWC; NCHW costs a layout
    transform around every conv); the exact-fp32 path keeps the reference's NCHW (cuDNN's fp32
    NHWC kernels measured 18 % slower than NCHW on this network)."""
    return _MODE != 'fp32' and x.is_cuda


def network_input(x_nhwc):
    """NHWC image batch -> the NCHW-shaped tensor the conv stack consumes.  In the tensor-core
    mode this is a free view (NHWC memory == channels_last); in fp32 mode an NCHW copy."""
    x = x_nhwc.permute(0, 3, 1, 2)
    return x if channels_last_active(x_nhwc) else x.contiguous()


def direct_write_ok(x):
    """True when the tensor-core layers are active, i.e. when a caller may hand ``out=`` slots (channel
    slices of pre-allocated concat buffers) to conv2d / conv_transpose2d."""
    return _TC and _MODE == '3xtf32' and x.is_cuda


def conv2d(x, w, b, stride, pads, act=False, out=None):
    """pads = (top, bottom, left, right) TF-SAME padding; act: apply the leaky ReLU.  ``out``: optional
    destination (NCHW-shaped view with NHWC memory); honoured by the tensor-core path -- the result then
    aliases it -- and ignored by the others (the caller's concat copies as before)."""
    if _MODE == '3xtf32' and x.is_cuda:
        if not act and _use_narrow(x, w, stride, pads):
            return _NarrowConv3x3.apply(x, w, b)
        if _use_window(x, w, stride):
            from . import tc_conv
            w_rw = tc_conv.window_weights(w, tc_conv.window_channels(w.shape[1]))
            return _ConvWindow.apply(x, w_rw, b, w.shape[2], 2, tuple(pads), bool(act))
        if _use_space_to_depth(x, w, stride):
            xs, ws = space_to_depth_operands(x, w, pads)
            return conv2d(xs, ws, b, 1, (0, 0, 0, 0), act=act)
        if _tc_ok(x, stride) and w.shape[2] == w.shape[3] and w.shape[2] * w.shape[3] <= 64:
            return _ConvTC.apply(x, w, b, stride, tuple(pads), bool(act), out)
        fuse = act and b is not None and w.shape[0] % 4 == 0
        y = _Conv3x.apply(x, w, b, stride, tuple(pads), fuse)
        return F.leaky_relu(y, LRELU_SLOPE) if (act and not fuse) else y
    pt, pb, pl, pr = pads
    if pt == pb and pl == pr:
        padding = (pt, pl)
    else:
        x = F.pad(x, (pl, pr, pt, pb))
        padding = (0, 0)
    if x.is_cuda and _MODE == 'fp32':
        w = w.contiguous()     # parameters are stored NHWC-ordered; the exact-fp32 path computes in NCHW
    y = F.conv2d(x, w, b, stride=stride, padding=padding)
    return F.leaky_relu(y, LRELU_SLOPE) if act else y


def conv_transpose2d(x, w, b, act=False, out=None):
    if _MODE == '3xtf32' and x.is_cuda:
        if _tc_ok(x, 1):
            return _DeconvTC.apply(x, w, b, bool(act), out)
        fuse = act and b is not None and w.shape[1] % 4 == 0
        y = _Deconv3x.apply(x, w, b, fuse)
        return F.leaky_relu(y, LRELU_SLOPE) if (act and not fuse) else y
    if x.is_cuda and _MODE == 'fp32':
        w = w.contiguous()
    y = F.conv_transpose2d(x, w, b, stride=2, padding=1)
    return F.leaky_relu(y, LRELU_SLOPE) if act else y
