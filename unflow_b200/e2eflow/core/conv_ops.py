"""conv / deconv layers of the FlowNet stacks in one of two arithmetic modes.

'fp32'    plain cuDNN float32 (what the reference's slim.conv2d computes, flownet.py:174-233);
          no tensor cores.
'3xtf32'  the same contraction on the tensor cores at fp32-level accuracy (the default of bench.py; run.py
          and eval.py use it with ``[run] conv_precision = 3xtf32``): every operand is split x = hi + lo
          (hi = TF32-rounded, lo = exact residual) and lo*hi' + hi*lo' + hi*hi' is accumulated by the
          hand-written wgmma kernels (csrc/tc_conv.cu: forward and input gradient, csrc/tc_wgrad.cu: weight
          gradient, csrc/narrow_conv*.cu: the 2-channel flow
          heads in exact fp32) with the K loop cut into chunks that are summed in fp32 registers: 1.8e-6 of
          max|y| against float64 per layer, and the same 1e-4 flow tolerance against the fp32 oracle as the
          plain fp32 path.  Every layer runs on these kernels; an input they cannot read in place is copied
          into a fresh NHWC buffer first (_tc_input).

The mode is process-global.  Importing core/flownet.py sets it from ``UNFLOW_CONV_PRECISION`` (default
'fp32'); run.py then applies ``[run] conv_precision`` when the config has it, and eval.py the key of each
experiment's copied config.
"""
import torch
import torch.nn.functional as F

from ... import _native
from ..._native import check

_MODE = 'fp32'


def set_mode(mode):
    global _MODE
    if mode not in ('fp32', '3xtf32'):
        raise ValueError("conv precision must be 'fp32' or '3xtf32'")
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
    return _grad_slots.get(gen, {}).get(key if key is not None else _slot_key(x))


def grad_slot_put(gen, key_or_tensor, g):
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


# ---------------------------------------------------------------------------------------------
# Hand-written tensor-core path (3xTF32 wgmma implicit GEMM): csrc/tc_conv.cu for the forward (fused
# bias / leaky ReLU) and the input gradient, csrc/tc_wgrad.cu for the weight gradient.
# ---------------------------------------------------------------------------------------------


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


def _tc_input(x, stride=1, pads=(0, 0, 0, 0)):
    """``x`` and its ``pads`` (top, bottom, left, right) as _ConvTC / _DeconvTC take them.

    The kernels read NHWC memory with a 16-byte aligned base and a pixel pitch that is a multiple of 4
    floats, and the input gradient of a stride-2 conv (a transposed launch) needs an even H and W.  Any other
    input is copied into a fresh NHWC buffer of pitch round4(C), one zero row / column longer at the bottom /
    right where H / W is odd at stride 2.  The copy is differentiable: autograd returns dL/dx through it.
    The bottom / right pads shrink by what was appended, so the output extent is that of ``x``; the kernels
    read the appended zeros as they read their own TMA zero fill, so the result is the same.  No FlowNet
    layer takes the copy: the network inputs and the concat buffers are already in this form."""
    from . import tc_conv
    N, C, H, W = x.shape
    eh, ew = (H % 2, W % 2) if stride == 2 else (0, 0)
    if tc_conv.supported(x) and not (eh or ew):
        return x, pads
    buf = torch.zeros((N, H + eh, W + ew, _round4(C)), device=x.device, dtype=torch.float32)
    buf[:, :H, :W, :C] = x.permute(0, 2, 3, 1)
    xt = buf[..., :C].permute(0, 3, 1, 2)
    # The copy is new memory, so no gradient slot can belong to it.  One keyed by its address is left by an
    # earlier, freed tensor of this forward generation (layers called one after another outside a network
    # forward pass, which would start a new generation): drop it, or the backward would add dL/dx into it.
    _grad_slots.get(_generation, {}).pop(_slot_key(xt), None)
    pt, pb, pl, pr = pads
    return xt, (pt, pb - eh, pl, pr - ew)


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
        k = w.shape[2]
        pt, _, pl, _ = pads
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
            gw = _tc_weight_grad(gpre, x, w, stride, pt, pl)                       # rows C_out, columns C_in
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


def _use_window(x, w, stride):
    return (stride in (2, (2, 2)) and w.shape[2] == w.shape[3] and 5 <= w.shape[2] <= 8 and w.shape[1] <= 16
            and w.shape[0] % 4 == 0 and not x.requires_grad)


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
            gw = _tc_weight_grad(x, gpre, w, 2, 1, 1)                              # rows C_in, columns C_out
        return gx, gw, gb, None, None


# The narrow kernels serve every 2-channel 3x3 head: the large ones (flow2 / flow3 of a training batch)
# fill the GPU with 16x32-pixel tiles, the coarse ones (flow4 .. flow6: 8 .. 48 tiles) split the input
# channels over several CTAs per tile (csrc/narrow_conv.cu, csplit).  On the tensor-core kernel a head is
# one 32-wide N block with 2 useful columns and a K of 9 x 1026 walked by a handful of CTAs: 0.5 ms per step.
# The input gradient (a contraction over the 2 flow channels) goes through tc_conv.run, which unflow_tc_conv
# runs on the FMA pipes like every contraction over at most 4 channels (csrc/conv_fma.cu).
def _use_narrow(x, w, stride, pads):
    from . import tc_conv
    return (w.shape[0] == 2 and w.shape[2] == 3 and w.shape[3] == 3 and stride in (1, (1, 1))
            and tuple(pads) == (1, 1, 1, 1) and x.shape[1] % 2 == 0 and x.dtype == torch.float32
            and tc_conv.nhwc_geometry(x) is not None)       # NHWC memory, possibly a slice of a concat buffer


class _NarrowConv3x3(torch.autograd.Function):
    """The 2-channel flow heads (csrc/narrow_conv.cu): forward and weight gradient in exact fp32 on
    the FMA pipes, reading the wide input once at any pixel pitch; the input gradient (C_in wide, a
    contraction over the 2 flow channels) goes through ``tc_conv.run`` and runs on the FMA pipes too
    (csrc/conv_fma.cu)."""

    @staticmethod
    def forward(ctx, x, w, b):
        from . import tc_conv
        N, C, H, W = x.shape
        wl = w if w.is_contiguous(memory_format=torch.channels_last) else \
            w.contiguous(memory_format=torch.channels_last)
        # 4 floats per pixel: the up-sampling deconv that consumes the flow reads it through a TMA tensor map
        y = torch.empty((N, H, W, 4), device=x.device, dtype=torch.float32)[..., :2].permute(0, 3, 1, 2)
        from ..ops import kernel_timer
        with torch.cuda.device(x.device), kernel_timer.span("narrow_conv_fwd", 4 * x.numel() + 4 * y.numel()):
            check(_native.lib().unflow_conv3x3_narrow_fwd(
                x.data_ptr(), tc_conv.nhwc_geometry(x)[4], wl.data_ptr(), b.data_ptr() if b is not None else None,
                y.data_ptr(), 4, N, H, W, C, 2, torch.cuda.current_stream().cuda_stream), "conv3x3_narrow_fwd")
        ctx.save_for_backward(x, w)
        ctx.has_b = b is not None
        ctx.gen = _generation
        return y

    @staticmethod
    def backward(ctx, g):
        from . import tc_conv
        x, w = ctx.saved_tensors
        N, C, H, W = x.shape
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            # contraction over the 2 flow channels; the launch reads only the gradient, so x's pitch does not
            # matter: dL/dx goes to a fresh round4-pitched buffer or a registered gradient slot
            gd, _ = _lrelu_bwd_bias(g, None, False)
            gx = _input_grad_into_slot(ctx.gen, x, lambda dst, acc: tc_conv.run(
                gd, tc_conv.split_weights(_khwc(w), transpose=True), dst, mode=1, stride=1, kh=3, kw=3,
                pad_t=1, pad_l=1, accumulate=acc))
        if ctx.needs_input_grad[1]:
            lib = _native.lib()
            ws = torch.empty(lib.unflow_conv3x3_narrow_wgrad_workspace_bytes(N, H, W, C) // 4,
                             device=x.device, dtype=torch.float32)
            gw = torch.empty((2, 3, 3, C), device=x.device, dtype=torch.float32)
            sN, sC, sH, sW = g.stride()
            from ..ops import kernel_timer
            with torch.cuda.device(x.device), kernel_timer.span("narrow_conv_wgrad", 4 * x.numel() + 4 * g.numel()):
                check(lib.unflow_conv3x3_narrow_wgrad(
                    x.data_ptr(), tc_conv.nhwc_geometry(x)[4], g.data_ptr(), sN, sC, sH, sW, gw.data_ptr(),
                    ws.data_ptr(), N, H, W, C, 2, torch.cuda.current_stream().cuda_stream), "conv3x3_narrow_wgrad")
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


def _use_space_to_depth(x, w, stride):
    return (stride in (2, (2, 2)) and w.shape[2] == w.shape[3] and w.shape[2] % 2 == 1
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


def tc_active(x):
    """True when the layers fed ``x`` run on the tensor-core kernels (3xTF32 mode, CUDA tensors).  They
    compute in NHWC: the network input is then a free view of the NHWC images, concats go into NHWC
    buffers, and callers may hand ``out=`` slots (channel slices of pre-allocated concat buffers) to
    conv2d / conv_transpose2d.  The exact-fp32 path keeps the reference's NCHW (cuDNN's fp32 NHWC kernels
    measured 18 % slower than NCHW on this network)."""
    return _MODE == '3xtf32' and x.is_cuda


def network_input(x_nhwc):
    """NHWC image batch -> the NCHW-shaped tensor the conv stack consumes.  In the tensor-core
    mode this is a free view (NHWC memory == channels_last); in fp32 mode an NCHW copy."""
    x = x_nhwc.permute(0, 3, 1, 2)
    return x if tc_active(x_nhwc) else x.contiguous()


def conv2d(x, w, b, stride, pads, act=False, out=None):
    """pads = (top, bottom, left, right) TF-SAME padding; act: apply the leaky ReLU.  ``out``: optional
    destination (NCHW-shaped view with NHWC memory); honoured by the tensor-core path -- the result then
    aliases it -- and ignored by the others (the caller's concat copies as before)."""
    if tc_active(x):
        if not act and _use_narrow(x, w, stride, pads):
            return _NarrowConv3x3.apply(x, w, b)
        if _use_window(x, w, stride):
            from . import tc_conv
            w_rw = tc_conv.window_weights(w, tc_conv.window_channels(w.shape[1]))
            return _ConvWindow.apply(x, w_rw, b, w.shape[2], 2, tuple(pads), bool(act))
        if _use_space_to_depth(x, w, stride):
            xs, ws = space_to_depth_operands(x, w, pads)
            return conv2d(xs, ws, b, 1, (0, 0, 0, 0), act=act)
        kh, kw = w.shape[2], w.shape[3]
        if kh != kw or kh * kw > 64 or kh < stride:
            # (k < stride: the input gradient's transposed launch would have output parity classes without a tap)
            raise ValueError("the tensor-core conv takes square k x k filters with stride <= k <= 8, not %dx%d at "
                             "stride %d" % (kh, kw, stride))
        x, pads = _tc_input(x, stride, pads)
        return _ConvTC.apply(x, w, b, stride, tuple(pads), bool(act), out)
    pt, pb, pl, pr = pads
    if pt == pb and pl == pr:
        padding = (pt, pl)
    else:
        x = F.pad(x, (pl, pr, pt, pb))
        padding = (0, 0)
    if x.is_cuda:
        w = w.contiguous()     # parameters are stored NHWC-ordered; the exact-fp32 path computes in NCHW
    y = F.conv2d(x, w, b, stride=stride, padding=padding)
    return F.leaky_relu(y, LRELU_SLOPE) if act else y


def conv_transpose2d(x, w, b, act=False, out=None):
    if tc_active(x):
        x, _ = _tc_input(x)
        return _DeconvTC.apply(x, w, b, bool(act), out)
    if x.is_cuda:
        w = w.contiguous()
    y = F.conv_transpose2d(x, w, b, stride=2, padding=1)
    return F.leaky_relu(y, LRELU_SLOPE) if act else y
