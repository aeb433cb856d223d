"""Float64 references of the non-tensor-core kernels (include/unflow.h), with their error scales.

Every reference here is the operation's definition evaluated in float64 from the float32 operands the kernel read,
on the device of its operands.  Each comes with A, the same evaluation on absolute values (every difference becomes
a sum of magnitudes), so that a kernel is checked elementwise as |got - ref| <= TAU * A: an error cannot hide behind
cancellation or behind a large element elsewhere.  Used by tests/test_gpu_step_launches.py (one training step,
every launch) and tests/test_gpu_float64_kernels.py (the shapes and edges the step does not reach); pinned on the
CPU to the reference's golden outputs, the oracle and brute definitions by tests/test_float64_refs_cpu.py.
"""
import math

import torch
import torch.nn.functional as F

from oracle import losses as olosses
from oracle.image_warp import image_warp as oimage_warp


# ---- device pointers as tensors --------------------------------------------------------------------------------
class _DeviceArray:
    def __init__(self, ptr, shape, strides, typestr, itemsize):
        self.__cuda_array_interface__ = dict(
            shape=tuple(int(s) for s in shape), typestr=typestr, data=(int(ptr), False), version=3,
            strides=None if strides is None else tuple(int(s) * itemsize for s in strides))


def view(ptr, shape, strides=None, dtype=torch.float32):
    """The device memory at `ptr` as a tensor (strides in elements; None = dense)."""
    typestr, size = {torch.float32: ("<f4", 4), torch.uint8: ("|u1", 1)}[dtype]
    return torch.as_tensor(_DeviceArray(ptr, shape, strides, typestr, size), device="cuda")


def worst_ratio(got, ref, A):
    """max |got - ref| / A; an error where A == 0 counts as infinite."""
    err = (got.double() - ref).abs()
    if not err.numel():
        return 0.0
    return float(torch.where(err == 0, torch.zeros_like(err), err / A.clamp_min(1e-300)).max())


# ---- correlation (reference ops/correlation_op.cu.cc; NCHW) -------------------------------------------------------
def corr_geometry(H, W, ks, md, pad, s1, s2):
    kr = (ks - 1) // 2
    border = md + kr
    ngr = md // s2
    oh = math.ceil((H + 2 * pad - 2 * border) / s1)
    ow = math.ceil((W + 2 * pad - 2 * border) / s1)
    return ngr, 2 * ngr + 1, oh, ow


def correlation(in0, in1, ks, md, pad, s1, s2, skip_row=None):
    """out[b, (p+ngr)*D + o+ngr, y, x] = sum_{c,j,i} in0p[c, y*s1+md+j, x*s1+md+i] in1p[c, .. + s2*p, .. + s2*o]
    / (ks*ks*C), zero padded by `pad`.  `skip_row`: leave displacement row p out (a wrong kernel, for the
    negative control)."""
    B, C, H, W = in0.shape
    ngr, D, oh, ow = corr_geometry(H, W, ks, md, pad, s1, s2)
    p0, p1 = F.pad(in0, [pad] * 4), F.pad(in1, [pad] * 4)
    outs = []
    for p in range(-ngr, ngr + 1):
        for o in range(-ngr, ngr + 1):
            acc = in0.new_zeros(B, oh, ow)
            if p != skip_row:
                for j in range(ks):
                    for i in range(ks):
                        y0, x0 = md + j, md + i
                        a = p0[:, :, y0:y0 + s1 * (oh - 1) + 1:s1, x0:x0 + s1 * (ow - 1) + 1:s1]
                        y1, x1 = y0 + s2 * p, x0 + s2 * o
                        b = p1[:, :, y1:y1 + s1 * (oh - 1) + 1:s1, x1:x1 + s1 * (ow - 1) + 1:s1]
                        acc = acc + (a * b).sum(1)
            outs.append(acc / (ks * ks * C))
    return torch.stack(outs, 1)


@torch.enable_grad()        # also inside a backward pass, where autograd is off
def correlation_grads(gout, in0, in1, attrs, skip_row=None):
    """(g0, g1) of sum(gout * correlation(in0, in1)) in float64 by autograd, and their A (|gout|, |in|)."""
    def vjp(g, a, b):
        a, b = a.detach().requires_grad_(True), b.detach().requires_grad_(True)
        return torch.autograd.grad((correlation(a, b, *attrs, skip_row=skip_row) * g).sum(), (a, b))
    g0, g1 = vjp(gout, in0, in1)
    A0, A1 = vjp(gout.abs(), in0.abs(), in1.abs())
    return g0, g1, A0, A1


def fold_reverse(grev, s2, ngr):
    """The gradient of corr(in1, in0) re-indexed onto corr(in0, in1)'s displacements:
    out[(p,o)](y, x) = grev[(-p,-o)](y + s2*p, x + s2*o), zero where that pixel leaves the image."""
    B, DD, H, W = grev.shape
    D = 2 * ngr + 1
    m = s2 * ngr
    gp = F.pad(grev, [m] * 4).view(B, D, D, H + 2 * m, W + 2 * m)
    out = torch.empty_like(grev).view(B, D, D, H, W)
    for pi in range(D):
        for oi in range(D):
            p, o = pi - ngr, oi - ngr
            out[:, pi, oi] = gp[:, D - 1 - pi, D - 1 - oi, m + s2 * p:m + s2 * p + H, m + s2 * o:m + s2 * o + W]
    return out.view(B, DD, H, W)


# ---- downsample, warps ----------------------------------------------------------------------------------------------
def downsample(x, s):
    """[B,H,W,C] block mean."""
    B, H, W, C = x.shape
    return x.view(B, H // s, s, W // s, s, C).mean((2, 4))


def _gather(img, yy, xx):
    """img [B,H,W,C] at integer pixel maps yy, xx [B,h,w] -> [B,h,w,C]."""
    B, H, W, C = img.shape
    idx = (yy * W + xx).reshape(B, -1, 1).expand(-1, -1, C)
    return img.reshape(B, H * W, C).gather(1, idx).reshape(*yy.shape, C)


def _fp32_sum(grid, f):
    """grid + f rounded to fp32 as the kernels compute it, differentiable w.r.t. f (float64)."""
    s = (grid.float() + f.detach().float()).double()
    return f + (s - f).detach()


def _fp32_frac(f, fl):
    """f - floor(f) rounded to fp32, differentiable w.r.t. f (float64).  image_warp defines its bilinear weights
    by this fp32 difference (reference image_warp.py:26-27): a flow a hair below an integer has a fraction within
    an ulp of 1, whose rounding is a large relative error of the other side's weight 1 - fraction."""
    s = (f.detach().float() - fl.float()).double()
    return (f - fl) + (s - (f - fl)).detach()


def warp_taps(flow, mode, floor_from=None):
    """Tap pixels and bilinear weights of one gather: mode 0 = BackwardWarp (zero outside), 1 = image_warp
    (clamped taps), 2 = spatial transformer (absolute coordinates, weights from the clamped taps).  Returns
    [(yy, xx, weight, valid)] for the taps (y0,x0) (y1,x0) (y0,x1) (y1,x1); weights differentiable w.r.t. flow.
    `floor_from` (mode 1): the flow whose floor() picks the taps, e.g. the fp32 flow a kernel warped with; the
    weights still come from `flow`, so the float64 derivative is taken on the kernel's side of an integer."""
    B, H, W, _ = flow.shape
    u, v = flow[..., 0], flow[..., 1]
    gx = torch.arange(W, device=flow.device).view(1, 1, W)
    gy = torch.arange(H, device=flow.device).view(1, H, 1)
    if mode == 2:
        x, y = u, v
    else:
        # the kernel forms the sample position in fp32: take its floor from the same rounded sum (a derivative
        # is discontinuous where the floor changes), with d position / d flow = 1
        x, y = _fp32_sum(gx, u), _fp32_sum(gy, v)
    if mode == 1:
        src = flow if floor_from is None else floor_from.to(flow.dtype)
        fu, fv = torch.floor(src[..., 0]).detach(), torch.floor(src[..., 1]).detach()
        xw, yw = _fp32_frac(u, fu), _fp32_frac(v, fv)
        x0, y0 = gx + fu.long(), gy + fv.long()
    else:
        x0, y0 = torch.floor(x).detach().long(), torch.floor(y).detach().long()
        xw, yw = x - x0, y - y0
    x1, y1 = x0 + 1, y0 + 1
    if mode == 0:
        vx0, vx1 = (x0 >= 0) & (x0 < W), (x1 >= 0) & (x1 < W)
        vy0, vy1 = (y0 >= 0) & (y0 < H), (y1 >= 0) & (y1 < H)
        cx0, cx1, cy0, cy1 = x0.clamp(0, W - 1), x1.clamp(0, W - 1), y0.clamp(0, H - 1), y1.clamp(0, H - 1)
        wl, wt = 1 - xw, 1 - yw
        return [(cy0, cx0, wl * wt, vx0 & vy0), (cy1, cx0, wl * yw, vx0 & vy1),
                (cy0, cx1, xw * wt, vx1 & vy0), (cy1, cx1, xw * yw, vx1 & vy1)]
    cx0, cx1, cy0, cy1 = x0.clamp(0, W - 1), x1.clamp(0, W - 1), y0.clamp(0, H - 1), y1.clamp(0, H - 1)
    if mode == 2:
        wl, xr, wt, yb = cx1 - x, x - cx0, cy1 - y, y - cy0
    else:
        wl, xr, wt, yb = 1 - xw, xw, 1 - yw, yw
    ones = torch.ones_like(cx0, dtype=torch.bool)
    return [(cy0, cx0, wl * wt, ones), (cy1, cx0, wl * yb, ones), (cy0, cx1, xr * wt, ones), (cy1, cx1, xr * yb, ones)]


def warp(img, flow, mode, skip_tap=None, floor_from=None):
    """The bilinear gather of unflow_backward_warp_fwd in float64 (differentiable w.r.t. img and flow).
    `skip_tap`: leave tap t of warp_taps out (a wrong kernel, for the negative control); `floor_from`: see
    warp_taps."""
    out = 0
    for t, (yy, xx, wgt, valid) in enumerate(warp_taps(flow, mode, floor_from)):
        if t != skip_tap:
            out = out + (wgt * valid)[..., None] * _gather(img, yy, xx)
    return out


def warp_abs(img, flow, mode):
    """A of warp(): sum over the taps of |weight| * |tap|."""
    out = 0
    for yy, xx, wgt, valid in warp_taps(flow.detach(), mode):
        out = out + (wgt.abs() * valid)[..., None] * _gather(img.abs(), yy, xx)
    return out


@torch.enable_grad()        # also inside a backward pass, where autograd is off
def warp_grads(grad, img, flow, mode, skip_tap=None):
    """(dimage, dflow) of sum(grad * warp(img, flow)) by float64 autograd, and their A (of the full warp)."""
    i, f = img.detach().requires_grad_(True), flow.detach().requires_grad_(True)
    dimg, dflow = torch.autograd.grad((warp(i, f, mode, skip_tap) * grad).sum(), (i, f))
    B, H, W, C = img.shape
    f = flow.detach()
    taps = warp_taps(f, mode)
    x = f[..., 0] if mode == 1 else _fp32_sum(torch.arange(W, device=f.device).view(1, 1, W), f[..., 0])
    y = f[..., 1] if mode == 1 else _fp32_sum(torch.arange(H, device=f.device).view(1, H, 1), f[..., 1])
    xw, yw = x - torch.floor(x), y - torch.floor(y)
    ga = grad.abs()
    Ai = torch.zeros_like(img)
    Af = torch.zeros_like(flow)
    # tap t's weight moves with u by +-(its row fraction) and with v by +-(its column fraction)
    for t, (yy, xx, wgt, valid) in enumerate(taps):
        Ai.view(B, H * W, C).scatter_add_(1, (yy * W + xx).reshape(B, -1, 1).expand(-1, -1, C),
                                          ((wgt.abs() * valid)[..., None] * ga).reshape(B, -1, C))
        tap = (_gather(img.abs(), yy, xx) * ga).sum(-1) * valid
        Af[..., 0] += tap * (yw if t in (1, 3) else 1 - yw)
        Af[..., 1] += tap * (xw if t in (2, 3) else 1 - xw)
    return dimg, dflow, Ai, Af


# ---- forward warp (reference ops/forward_warp_op.cu.cc) --------------------------------------------------------------
def forward_warp_splats(flow, k=4):
    """The splats of ForwardWarp: every source pixel adds exp(-((nx-tx)^2 + (ny-ty)^2) / 2) to the pixels of
    the window [floor(t - 4), floor(t + 4)] around its target t = pos + flow, clipped to the image.  Yields
    (target index [B, H*W], weight, nx - tx, ny - ty), weights zero outside the window; differentiable."""
    B, H, W, _ = flow.shape
    gx = torch.arange(W, device=flow.device).view(1, 1, W)
    gy = torch.arange(H, device=flow.device).view(1, H, 1)
    tx, ty = _fp32_sum(gx, flow[..., 0]), _fp32_sum(gy, flow[..., 1])
    bx, by = torch.floor(tx.detach() - k).long(), torch.floor(ty.detach() - k).long()
    for j in range(2 * k + 1):
        ny = by + j
        vy = (ny >= 0) & (ny < H) & (ny <= torch.floor(ty.detach() + k).long())
        for i in range(2 * k + 1):
            nx = bx + i
            ok = vy & (nx >= 0) & (nx < W) & (nx <= torch.floor(tx.detach() + k).long())
            dx, dy = nx - tx, ny - ty
            wgt = torch.exp(-(dx ** 2 + dy ** 2) / 2) * ok
            idx = (ny.clamp(0, H - 1) * W + nx.clamp(0, W - 1)).reshape(B, -1)
            yield idx, wgt.reshape(B, -1), dx.reshape(B, -1), dy.reshape(B, -1)


def forward_warp(flow):
    """[B,H,W,1] splat map of ForwardWarp in float64, and the number of splats each pixel received."""
    B, H, W, _ = flow.shape
    out, count = flow.new_zeros(B, H * W), flow.new_zeros(B, H * W)
    for idx, wgt, _, _ in forward_warp_splats(flow):
        out = out.scatter_add(1, idx, wgt)
        count = count.scatter_add(1, idx, (wgt > 0).double())
    return out.view(B, H, W, 1), count.view(B, H, W, 1)


@torch.enable_grad()        # also inside a backward pass, where autograd is off
def forward_warp_grads(grad, flow):
    """dflow of sum(grad * forward_warp(flow)) by float64 autograd, and its A: sum over the window of
    |grad(n)| * weight * (|nx - tx|, |ny - ty|)."""
    B, H, W, _ = flow.shape
    f = flow.detach().requires_grad_(True)
    dflow, = torch.autograd.grad((forward_warp(f)[0] * grad).sum(), f)
    A = torch.zeros(B, H * W, 2, device=flow.device, dtype=torch.float64)
    ga = grad.abs().reshape(B, H * W)
    for idx, wgt, dx, dy in forward_warp_splats(flow.detach()):
        gw = ga.gather(1, idx) * wgt
        A[..., 0] += gw * dx.abs()
        A[..., 1] += gw * dy.abs()
    return dflow, A.view(B, H, W, 2)


# ---- the fused level loss (csrc/level_loss.cu; reference losses.py:16-122,206-366) ---------------------------------
EPS2, ALPHA = 1e-6, 0.45
FB_OCC_OFFSET = 0.5         # the fb occlusion test |f + w(g)|^2 > 0.01 (|f|^2 + |w(g)|^2) + 0.5 (losses.py:59-63)
TERMS = ['sym', 'occ', 'photo', 'grad', 'smooth_1st', 'smooth_2nd', 'fb', 'ternary']


def charb(x):
    return (x * x + EPS2) ** ALPHA


def charb_d(x):
    return 2 * ALPHA * x * (x * x + EPS2) ** (ALPHA - 1)


def charb_d_scale(x, xabs):
    """A of c'(x) when x carries a rounding error of order 2^-24 * xabs: |c'(x)| + K(x) * xabs, where
    K(x) = 2*alpha*(x^2 + eps^2)^(alpha - 1) bounds |c''| near x.  Without the second part a flow difference
    that cancels to ~0 in fp32 would count as an infinite relative error."""
    K = 2 * ALPHA * (x * x + EPS2) ** (ALPHA - 1)
    return K * (x.abs() + xabs)


def gray255(im):
    return (im[..., 0] * 0.2989 + im[..., 1] * 0.5870 + im[..., 2] * 0.1140) * 255


def census(g, R, clamp=False):
    """[B,h,w] grey -> [B,h,w,P*P] soft census t(g(n) - g(c)), zero padded (reference conv2d SAME);
    clamp=True replicates the border instead (a wrong kernel, for the negative control)."""
    B, h, w = g.shape
    if clamp:
        gp = F.pad(g[:, None], [R] * 4, mode="replicate")[:, 0]
    else:
        gp = F.pad(g, [R] * 4)
    out = []
    for dy in range(-R, R + 1):
        for dx in range(-R, R + 1):
            s = gp[:, R + dy:R + dy + h, R + dx:R + dx + w] - g
            out.append(s / torch.sqrt(0.81 + s * s))
    return torch.stack(out, -1)


def _span(n, need):
    return (1, n - 1) if need else (0, n)


SECOND_ORDER = [(0, 1), (1, 0), (1, 1), (1, -1)]        # x, y, diag1 (q-w-1 / q+w+1), diag2 (q-w+1 / q+w-1)


def _second_order_deltas(f):
    """[(delta [B,Y,X,2], a, c, centre, (y0, y1, x0, x1), (ey, ex))] of the four 2nd-order filters, centres
    where the filter's mask is 1."""
    B, h, w, _ = f.shape
    out = []
    for ey, ex in SECOND_ORDER:
        y0, y1 = _span(h, ey != 0)
        x0, x1 = _span(w, ex != 0)
        if y1 <= y0 or x1 <= x0:
            continue
        a = f[:, y0 - ey:y1 - ey, x0 - ex:x1 - ex]
        c = f[:, y0 + ey:y1 + ey, x0 + ex:x1 + ex]
        ctr = f[:, y0:y1, x0:x1]
        out.append(((a + c) - 2 * ctr, a, c, ctr, (y0, y1, x0, x1), (ey, ex)))
    return out


def _first_order_deltas(f):
    B, h, w, _ = f.shape
    return [(f[:, :, :-1] - f[:, :, 1:], (0, 1)), (f[:, :-1] - f[:, 1:], (1, 0))]


class LevelInputs:
    """The operands of one level-loss call as float64 tensors (flows [B,h,w,2], masks [B,h,w])."""

    def __init__(self, im1, im2, ffw, fbw, border, fwarp_fw, fwarp_bw, occl, R, bits):
        d = lambda t: None if t is None else t.detach().double()
        self.im1, self.im2, self.ffw, self.fbw = d(im1), d(im2), d(ffw), d(fbw)
        self.border = d(border)
        self.fwarp_fw, self.fwarp_bw = d(fwarp_fw), d(fwarp_bw)
        self.occl, self.R, self.bits = occl, R, bits
        self.B, self.h, self.w = im1.shape[:3]

    def want(self, name):
        return bool(self.bits >> TERMS.index(name) & 1)


def masks_f32(ffw, fbw, border, occl, fwarp_fw, fwarp_bw):
    """mask_fw, mask_bw [B,h,w] by the mask formulas of oracle/losses.py compute_losses, op by op in float32
    (one rounding per op, no contraction: what the kernel evaluates with __fmul_rn / __fadd_rn), on the flows'
    device."""
    ffw_in = ffw
    ffw, fbw = ffw.detach().float().cpu(), fbw.detach().float().cpu()
    if border is None:
        mfw, mbw = olosses.create_outgoing_mask(ffw), olosses.create_outgoing_mask(fbw)
    else:
        mfw = mbw = border.detach().float().cpu().expand(ffw.shape[0], -1, -1, -1)
    if occl == 1:
        fbw_w, ffw_w = oimage_warp(fbw, ffw), oimage_warp(ffw, fbw)
        occ = []
        for f, gw in ((ffw, fbw_w), (fbw, ffw_w)):
            mag = olosses.length_sq(f) + olosses.length_sq(gw)
            occ.append((olosses.length_sq(f + gw) > 0.01 * mag + FB_OCC_OFFSET).float())
        mfw, mbw = mfw * (1 - occ[0]), mbw * (1 - occ[1])
    elif occl == 2:
        mfw = mfw * (1 - (fwarp_bw.float().cpu() < 0.8).float())
        mbw = mbw * (1 - (fwarp_fw.float().cpu() < 0.8).float())
    dev = ffw_in.device
    return mfw[..., 0].to(dev), mbw[..., 0].to(dev)


def level_losses(L, ffw, fbw, mfw, mbw, variant=None):
    """The 8 loss terms (TERMS order; unrequested ones 0) in float64 with the masks held fixed, differentiable
    w.r.t. ffw and fbw.  variant: None = the definition; 'detach_fb' stops the gradient of the fb term into
    the other flow (through image_warp(flow_bw, flow_fw)); 'clamp_census' replicates the image border in the
    census window; 'margin' shrinks the census transform mask to R - 1 (wrong kernels, negative controls).
    The Sobel 'grad' term has no kernel and no reference here: its bit raises."""
    if L.want('grad'):
        raise ValueError("level_losses: the 'grad' term is not evaluated")
    B, h, w, R = L.B, L.h, L.w, L.R
    n1 = float(B * h * w)
    out = [ffw.new_zeros(())] * 8
    add = lambda k, v: out.__setitem__(TERMS.index(k), out[TERMS.index(k)] + v)
    for A, Bim, f, g, m, fwo in ((L.im1, L.im2, ffw, fbw, mfw, L.fwarp_bw), (L.im2, L.im1, fbw, ffw, mbw, L.fwarp_fw)):
        occ = 1 - m
        if L.want('occ'):
            add('occ', charb(occ).sum() / n1)
        if L.want('sym'):
            add('sym', charb(occ - (fwo[..., 0] < 0.8).double()).sum() / n1)
        if L.want('fb'):
            gw = warp(g.detach() if variant == 'detach_fb' else g, f, 1)
            fd = f + gw
            add('fb', (m[..., None] * charb(fd)).sum() / (2 * n1))
        if L.want('photo') or L.want('ternary'):
            Bw = warp(Bim, f, 1)
        if L.want('photo'):
            add('photo', (m[..., None] * charb((A - Bw) * 255)).sum() / (3 * n1))
        if L.want('smooth_1st'):
            add('smooth_1st', sum(charb(d).sum() for d, _ in _first_order_deltas(f)) / (2 * n1))
        if L.want('smooth_2nd'):
            add('smooth_2nd', sum(charb(d[0]).sum() for d in _second_order_deltas(f)) / (4 * n1))
        if L.want('ternary'):
            t1 = census(gray255(A), R, clamp=variant == 'clamp_census')
            t2 = census(gray255(Bw), R, clamp=variant == 'clamp_census')
            dd = (t1 - t2) ** 2
            dist = (dd / (0.1 + dd)).sum(-1)
            r = R - 1 if variant == 'margin' else R
            tm = torch.zeros(h, w, device=m.device, dtype=m.dtype)
            tm[r:h - r, r:w - r] = 1
            add('ternary', (m * tm * charb(dist)).sum() / n1)
    return torch.stack(out)


@torch.enable_grad()        # also inside a backward pass, where autograd is off
def level_loss_grads(L, mfw, mbw, gl, variant=None):
    """(dflow_fw, dflow_bw) of sum(gl * level_losses) by float64 autograd."""
    f = L.ffw.clone().requires_grad_(True)
    b = L.fbw.clone().requires_grad_(True)
    loss = (level_losses(L, f, b, mfw, mbw, variant) * gl.double()).sum()
    if not loss.requires_grad:          # only the mask terms (occ, sym): no gradient
        return torch.zeros_like(f), torch.zeros_like(b)
    gf, gb = torch.autograd.grad(loss, (f, b), allow_unused=True)
    return (gf if gf is not None else torch.zeros_like(f)), (gb if gb is not None else torch.zeros_like(b))


def _dwarp_abs(img_abs, taps, xw, yw):
    """|d warp / d(u, v)| with every tap difference as a sum: ((|Ic|+|Ia|)(1-yw) + (|Id|+|Ib|)yw, ...)."""
    (ya, xa, _, _), (yb, xb, _, _), (yc, xc, _, _), (yd, xd, _, _) = taps
    Ia, Ib, Ic, Id = (_gather(img_abs, y, x) for y, x in ((ya, xa), (yb, xb), (yc, xc), (yd, xd)))
    xw, yw = xw[..., None], yw[..., None]
    return (Ic + Ia) * (1 - yw) + (Id + Ib) * yw, (Ib + Ia) * (1 - xw) + (Id + Ic) * xw


def level_loss_grad_scale(L, mfw, mbw, gl):
    """A of level_loss_grads, elementwise: the sum over every contribution that reaches a flow element of its
    absolute magnitude, differences taken as sums of magnitudes and c'(x) as charb_d_scale.  (fb: the direct
    term plus the scatter through the four taps of the other direction; census: u * |dgB/du| *
    sum_n (|W(n)| + |W(q)|) |phi|; smoothness: sum |coef| |c'(delta)| over the valid stencils.)"""
    B, h, w, R = L.B, L.h, L.w, L.R
    n1 = float(B * h * w)
    gl = gl.double().abs()
    u = {k: float(gl[TERMS.index(k)]) / d for k, d in
         (('photo', 3 * n1), ('fb', 2 * n1), ('smooth_1st', 2 * n1), ('smooth_2nd', 4 * n1), ('ternary', n1))}
    Af, Ab = torch.zeros_like(L.ffw), torch.zeros_like(L.fbw)
    wgt = torch.tensor([0.2989, 0.5870, 0.1140], device=L.ffw.device, dtype=torch.float64)
    for A, Bim, f, g, m, Aout, Aother in ((L.im1, L.im2, L.ffw, L.fbw, mfw, Af, Ab),
                                          (L.im2, L.im1, L.fbw, L.ffw, mbw, Ab, Af)):
        taps = warp_taps(f, 1)
        xw, yw = f[..., 0] - torch.floor(f[..., 0]), f[..., 1] - torch.floor(f[..., 1])
        if L.want('fb'):
            gw, gwa = warp(g, f, 1), warp_abs(g, f, 1)
            fd = f + gw
            Kf = u['fb'] * m[..., None] * charb_d_scale(fd, f.abs() + gwa)       # [B,h,w,2]
            dgu, dgv = _dwarp_abs(g.abs(), taps, xw, yw)                          # [B,h,w,2] each
            Aout[..., 0] += Kf[..., 0] * (1 + dgu[..., 0]) + Kf[..., 1] * dgu[..., 1]
            Aout[..., 1] += Kf[..., 1] * (1 + dgv[..., 1]) + Kf[..., 0] * dgv[..., 0]
            for yy, xx, wt, _ in taps:
                Aother.view(B, h * w, 2).scatter_add_(1, (yy * w + xx).reshape(B, -1, 1).expand(-1, -1, 2),
                                                      (wt[..., None] * Kf).reshape(B, -1, 2))
        dB = torch.zeros(B, h, w, 3, device=f.device, dtype=torch.float64)
        if L.want('photo'):
            Bw, Bwa = warp(Bim, f, 1), warp_abs(Bim, f, 1)
            dB += u['photo'] * m[..., None] * 255 * charb_d_scale((A - Bw) * 255, 255 * (A.abs() + Bwa))
        if L.want('ternary'):
            Bw = warp(Bim, f, 1)
            gA, gB = gray255(A), gray255(Bw)
            t1, t2 = census(gA, R), census(gB, R)
            dd = (t1 - t2) ** 2
            dist = (dd / (0.1 + dd)).sum(-1)
            tm = torch.zeros(h, w, device=f.device, dtype=torch.float64)
            tm[R:h - R, R:w - R] = 1
            Wq = (m * tm * charb_d(dist)).abs()
            pad = lambda t: F.pad(t, [R] * 4)
            gAp, gBp, Wp = pad(gA), pad(gB), pad(Wq)
            acc = torch.zeros_like(gA)
            for dy in range(-R, R + 1):
                for dx in range(-R, R + 1):
                    sl = lambda t: t[:, R + dy:R + dy + h, R + dx:R + dx + w]
                    s1, s2 = gA - sl(gAp), gB - sl(gBp)
                    ta, tb = s1 / torch.sqrt(0.81 + s1 * s1), s2 / torch.sqrt(0.81 + s2 * s2)
                    d = (ta - tb) ** 2
                    phi = 0.1 / (0.1 + d) ** 2 * 2 * (ta.abs() + tb.abs()) * 0.81 / (0.81 + s2 * s2) ** 1.5
                    acc += (sl(Wp) + Wq) * phi
            dB += u['ternary'] * acc[..., None] * 255 * wgt
        if L.want('photo') or L.want('ternary'):
            dwu, dwv = _dwarp_abs(Bim.abs(), taps, xw, yw)
            Aout[..., 0] += (dB * dwu).sum(-1)
            Aout[..., 1] += (dB * dwv).sum(-1)
        if L.want('smooth_1st'):
            for d, (ey, ex) in _first_order_deltas(f):
                a_ = f[:, :h - ey, :w - ex]
                c_ = f[:, ey:, ex:]
                k = u['smooth_1st'] * charb_d_scale(d, a_.abs() + c_.abs())
                Aout[:, :h - ey, :w - ex] += k
                Aout[:, ey:, ex:] += k
        if L.want('smooth_2nd'):
            for d, a_, c_, ctr, (y0, y1, x0, x1), (ey, ex) in _second_order_deltas(f):
                k = u['smooth_2nd'] * charb_d_scale(d, a_.abs() + c_.abs() + 2 * ctr.abs())
                Aout[:, y0 - ey:y1 - ey, x0 - ex:x1 - ex] += k
                Aout[:, y0 + ey:y1 + ey, x0 + ex:x1 + ex] += k
                Aout[:, y0:y1, x0:x1] += 2 * k
    return Af, Ab


# ---- the fused supervised flow loss (csrc/supervised_loss.cu; reference supervised.py:45-57) ---------------------
@torch.enable_grad()        # also inside a backward pass, where autograd is off
def supervised_loss_grads(flow, gt, mask, scale=20.0):
    """float64 loss, d loss / d flow, and the elementwise error budget of the float32 kernel's dflow.  The upscale
    is the oracle's restatement of TF's legacy resize_bilinear, not the product's."""
    from oracle import tf_compat
    f32 = 2.0 ** -24
    H, W = gt.shape[1:3]
    f = flow.detach().double().requires_grad_(True)
    v = tf_compat.resize_bilinear_legacy(f, (H, W)) * scale
    x = v - gt.double()
    m = torch.ones_like(x[..., :1]) if mask is None else mask.double()
    n = float(x.numel())
    loss = (m * (x * x + EPS2) ** ALPHA).sum() / n
    dflow, = torch.autograd.grad(loss, f, retain_graph=True)
    with torch.no_grad():
        q = x * x + EPS2
        c = 2 * ALPHA * x * q ** (ALPHA - 1)                         # d/dx of the penalty
        dc = 2 * ALPHA * q ** (ALPHA - 1) + 4 * ALPHA * (ALPHA - 1) * x * x * q ** (ALPHA - 2)
        # float32: |x| carries ~8 ulp of |v| + |gt| (the lerps, the scale, the difference); the penalty's
        # derivative ~1e-5 relative (exp2 / log2 approximations, the gather's fixed-order sum)
        per_px = m * (1e-5 * c.abs() + dc.abs() * 8 * f32 * (v.abs() + gt.double().abs()))
    budget, = torch.autograd.grad(v, f, grad_outputs=per_px * scale / n)
    return loss.detach(), dflow, budget.abs()


# ---- the networks' leaky-ReLU kinks (tests/test_gpu_float64_network.py, tests/test_gpu_float64_objective.py) ----
def record_kink_sides(monkeypatch):
    """Record, per layer scope and in call order, which side of the leaky-ReLU kink every element of the product's
    activations fell on (y > 0).  Returns {scope: [bool masks]}."""
    from unflow_b200.e2eflow.core import flownet as pfl
    sides = {}
    real_conv, real_deconv = pfl._Scope.conv, pfl._Scope.deconv

    def conv(self, x, name, stride=1, act=True, out=None):
        y = real_conv(self, x, name, stride, act, out)
        if act:
            sides.setdefault(self.p + name, []).append(y.detach() > 0)
        return y

    def deconv(self, x, name, act=True, out=None):
        y = real_deconv(self, x, name, act, out)
        if act:
            sides.setdefault(self.p + name, []).append(y.detach() > 0)
        return y
    monkeypatch.setattr(pfl._Scope, "conv", conv)
    monkeypatch.setattr(pfl._Scope, "deconv", deconv)
    return sides


def follow_kink_sides(monkeypatch, sides):
    """The oracle's leaky ReLU with the product's side of the kink: where fp32 and float64 disagree on the sign of
    a pre-activation within rounding of zero, the slope (1 or 0.1) is the one the product took.  Without this a
    handful of such elements on the 5x18-pixel levels moves a weight gradient by 1e-2.  The product's calls over
    one 2B batch (both directions, both images) cover the oracle's two calls over B, in the same order."""
    from oracle import flownet as oflownet
    cat = {k: torch.cat(v, 0) for k, v in sides.items()}
    used = dict.fromkeys(cat, 0)

    def act(x, scope):
        i, n = used[scope], x.shape[0]
        m = cat[scope][i:i + n]
        assert m.shape == x.shape, (scope, tuple(m.shape), tuple(x.shape))
        used[scope] = i + n
        return torch.where(m, x, 0.1 * x)
    monkeypatch.setattr(oflownet, "leaky_relu", act)
    return used, cat


def errors(got, ref):
    """(relative L2 error, max error over max |ref|) of a float32 result against its float64 reference."""
    d = got.double() - ref
    return (float(d.norm() / ref.norm().clamp_min(1e-300)),
            float(d.abs().max() / ref.abs().max().clamp_min(1e-300)))
