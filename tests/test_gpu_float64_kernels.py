"""The non-tensor-core kernels against float64 at the shapes and edges one training step does not reach.

Same references and bound as tests/test_gpu_step_launches.py: |got - ref| <= TAU * A elementwise, A = the same
float64 evaluation on absolute values (tests/float64_refs.py), with that file's TAU per kernel family.

  level loss   w not a multiple of 32, h not a multiple of 8, levels smaller than one tile, h or w < 2R + 1 (the
               census transform mask is all zero, the smoothness terms are not), h = 1 and w = 1; flows that
               push all four taps outside the image, integer and half-integer flows, flows landing exactly on
               x = 0 / x = w - 1 with border_mask = None (the <= / >= edges of the outgoing mask); the fractional
               border masks of the loss pyramid and a U(0, 1) mask; occlusion '', 'fb', 'disocc'; every term
               alone and all together; B = 1 and 4.
  correlation  the generic kernel (kernel_size 3, stride_1 2, pad != max_displacement, odd H, W % 4 != 0), the
               tiled backward's run-time radius (even r < 10), C not a multiple of the 128-channel slab.
  warps        BORDER_ZERO / BORDER_CLAMP at 4x384x1280x3 and 2-channel flows at 96x320, forward, dflow and the
               dimage scatter; BORDER_CLAMP with a flow a hair below an integer; BORDER_STN forward.
  forward warp forward and backward at 96x320, at a small flow scale and at one where many splats leave.
  Adam         the four entry points at step 1 and 7, with and without the l2 mask.

Negative controls show that the bounds catch plausible wrong kernels: the level-loss gradient against a
reference that detaches the fb term's path into the other flow, and against one whose census transform mask
margin is R - 1; the correlation backward against a reference that drops one displacement row.  (A census window
that clamps at the image border instead of zero padding is not observable: the transform mask zeroes every
centre whose window leaves the image.  The test asserts exactly that.)  Measured on an H100 SXM 80 GB at a 400 W
power limit: the level-loss gradient is checked at 1.4e-5 in the control case, the detached fb path reaches 6.9e-3
(115 x TAU_LOSS) and the narrow margin 0.62; the correlation gradient is checked at 1.5e-7 and a dropped
displacement row reaches 0.38 (1e5 x TAU_SUM).  The file takes about 5 s of GPU time.
"""
import numpy as np
import pytest
import torch

import float64_refs as R
from oracle import losses as olosses
from test_gpu_step_launches import (TAU_ADAM, TAU_LOSS, TAU_SUM, adam_reference, l2_bits, level_loss_bwd_ratios,
                                    level_loss_fwd_ratios)

pytestmark = pytest.mark.gpu

GL = [0.9, 12.4, 0.7, 0.0, 1.3, 3.0, 0.2, 1.0]          # d total / d term (sym, occ, photo, -, s1, s2, fb, tern)
ALL = ['sym', 'occ', 'photo', 'smooth_1st', 'smooth_2nd', 'fb', 'ternary']


def _lib():
    from unflow_b200 import _native
    return _native.lib()


def _st():
    return torch.cuda.current_stream().cuda_stream


def make_flows(B, h, w, kind, seed):
    g = torch.Generator().manual_seed(seed)
    f = (torch.rand(B, h, w, 2, generator=g) * 2 - 1) * 3
    gx = torch.arange(w, dtype=torch.float32).view(1, 1, w)
    gy = torch.arange(h, dtype=torch.float32).view(1, h, 1)
    if kind == "far":            # all four taps outside, on every side in turn (clamped: zero derivative)
        side = torch.randint(0, 4, (B, h, w), generator=g)
        f[..., 0] = torch.where(side == 0, -(w + 5.5), torch.where(side == 1, w + 5.5, f[..., 0]))
        f[..., 1] = torch.where(side == 2, -(h + 5.5), torch.where(side == 3, h + 5.5, f[..., 1]))
    elif kind == "integer":
        f = f.round()
    elif kind == "half":
        f = f.round() + 0.5
    elif kind == "edges":        # land exactly on x = 0, x = w - 1, y = 0 or y = h - 1
        side = torch.randint(0, 5, (B, h, w), generator=g)
        f[..., 0] = torch.where(side == 0, -gx, torch.where(side == 1, (w - 1) - gx, f[..., 0]))
        f[..., 1] = torch.where(side == 2, -gy, torch.where(side == 3, (h - 1) - gy, f[..., 1]))
    return f


def make_border(B, h, w, kind, seed):
    if kind is None:
        return None
    if kind == "binary":
        return olosses.create_border_mask(torch.zeros(B, h, w, 1), 0.1)
    if kind == "pyramid":        # the loss pyramid's level-0 mask: the full-size border mask averaged over 4x4
        full = olosses.create_border_mask(torch.zeros(B, 4 * h, 4 * w, 1), 0.1)
        return full.view(B, h, 4, w, 4, 1).mean((2, 4))
    return torch.rand(B, h, w, 1, generator=torch.Generator().manual_seed(seed))


def run_level(B, h, w, flows="smooth", border=None, occl=1, Rr=2, terms=ALL, seed=0):
    """One level_loss fwd + bwd call on the kernels -> (call description dict, losses, gl, dflow_fw, dflow_bw)."""
    from unflow_b200.e2eflow import ops
    from unflow_b200.e2eflow.core.fused_loss import _bits
    lib = _lib()
    g = torch.Generator().manual_seed(seed + 1)
    im1, im2 = torch.rand(B, h, w, 3, generator=g).cuda(), torch.rand(B, h, w, 3, generator=g).cuda()
    ffw = make_flows(B, h, w, flows, seed + 2).cuda()
    fbw = make_flows(B, h, w, flows, seed + 3).cuda()
    bm = make_border(B, h, w, border, seed + 4)
    bm = bm.cuda().contiguous() if bm is not None else None
    bits = _bits(terms)
    fwf = fwb = None
    if occl == 2 or 'sym' in terms:
        fwf, fwb = ops.forward_warp(ffw), ops.forward_warp(fbw)
    d = dict(im1=im1, im2=im2, ffw=ffw, fbw=fbw, border=bm, fwarp_fw=fwf, fwarp_bw=fwb, B=B, h=h, w=w, occl=occl,
             R=Rr, bits=bits)
    p = lambda t: t.data_ptr() if t is not None else None
    losses = torch.empty(8, device="cuda")
    saved = torch.empty(4 * B * h * w, device="cuda")
    ws = torch.empty(int(lib.unflow_level_loss_workspace_bytes(B, h, w)), device="cuda", dtype=torch.uint8)
    assert lib.unflow_level_loss_fwd(p(im1), p(im2), p(ffw), p(fbw), p(bm), p(fwf), p(fwb), p(losses), p(saved),
                                     None, p(ws), B, h, w, occl, Rr, bits, _st()) == 0
    gl = torch.tensor(GL, device="cuda")
    dfw, dbw = torch.empty_like(ffw), torch.empty_like(fbw)
    assert lib.unflow_level_loss_bwd(p(gl), p(im1), p(im2), p(ffw), p(fbw), p(bm), p(fwf), p(fwb), p(saved),
                                     p(dfw), p(dbw), B, h, w, occl, Rr, bits, _st()) == 0
    torch.cuda.synchronize()
    return d, losses, gl, dfw, dbw


LEVEL_CASES = [
    # B, h, w, flows, border, occl, R, terms
    (1, 6, 20, "smooth", "binary", 1, 3, ALL),
    (4, 13, 45, "smooth", "pyramid", 1, 3, ALL),
    (2, 24, 80, "smooth", "pyramid", 1, 2, ['occ', 'fb', 'ternary', 'smooth_2nd']),
    (2, 17, 35, "smooth", "random", 0, 2, ALL),
    (2, 16, 33, "smooth", "random", 2, 1, ALL),
    (1, 1, 9, "smooth", None, 1, 1, ALL),
    (1, 7, 1, "smooth", None, 1, 1, ALL),
    (2, 5, 40, "smooth", None, 1, 3, ALL),
    (2, 40, 6, "smooth", "random", 2, 3, ALL),
    (2, 12, 36, "far", None, 1, 2, ALL),
    (2, 12, 36, "far", "random", 0, 2, ALL),
    (2, 12, 36, "integer", None, 1, 2, ALL),
    (2, 12, 36, "half", "binary", 2, 2, ALL),
    (2, 12, 36, "edges", None, 1, 2, ALL),
    (2, 12, 36, "edges", None, 0, 3, ALL),
] + [(1, 10, 37, "smooth", "random", 1, 2, [t]) for t in ALL] + \
    [(4, 9, 70, "smooth", "pyramid", 2, 3, [t]) for t in ('sym', 'photo', 'fb', 'ternary')]


@pytest.mark.parametrize("B,h,w,flows,border,occl,Rr,terms", LEVEL_CASES)
def test_level_loss_vs_float64(B, h, w, flows, border, occl, Rr, terms):
    d, losses, gl, dfw, dbw = run_level(B, h, w, flows, border, occl, Rr, terms, seed=B * 1000 + h * 37 + w)
    lib = _lib()
    fwd = level_loss_fwd_ratios(lib, d, losses)
    rf, rb = level_loss_bwd_ratios(lib, d, gl, dfw, dbw)
    print("\nlosses %s  dflow_fw %.3e  dflow_bw %.3e" % (["%s %.2e" % r for r in fwd], rf, rb))
    assert all(r <= TAU_LOSS for _, r in fwd), fwd
    assert rf <= TAU_LOSS and rb <= TAU_LOSS, (rf, rb)


@pytest.mark.parametrize("variant,margin", [("detach_fb", 10), ("margin", 100)])
def test_level_loss_bound_catches_a_wrong_gradient(variant, margin):
    """Negative controls: the kernel's gradient checked against a reference without the fb scatter into the other
    flow, or with the census transform mask one pixel too narrow, must break TAU by a wide margin."""
    d, losses, gl, dfw, dbw = run_level(2, 24, 40, "smooth", None, 1, 3, ALL, seed=5)
    good = max(level_loss_bwd_ratios(_lib(), d, gl, dfw, dbw))
    bad = max(level_loss_bwd_ratios(_lib(), d, gl, dfw, dbw, variant=variant))
    print("\n%s: correct reference %.3e, wrong reference %.3e" % (variant, good, bad))
    assert good <= TAU_LOSS
    assert bad > margin * TAU_LOSS, bad


def test_level_loss_census_padding_is_not_observable():
    d, losses, gl, dfw, dbw = run_level(2, 24, 40, "smooth", None, 1, 3, ALL, seed=5)
    assert max(level_loss_bwd_ratios(_lib(), d, gl, dfw, dbw, variant="clamp_census")) <= TAU_LOSS


# ---- correlation -----------------------------------------------------------------------------------------------------
def _corr_case(shape, attrs, seed, bidir, skip_row=None):
    from unflow_b200.e2eflow import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(*shape, device="cuda", generator=g).requires_grad_(True)
    b = torch.randn(*shape, device="cuda", generator=g).requires_grad_(True)
    kw = dict(zip(("kernel_size", "max_displacement", "pad", "stride_1", "stride_2"), attrs))
    outs = ops.correlation_bidir(a, b, **kw) if bidir else (ops.correlation(a, b, **kw),)
    grads = [torch.randn(o.shape, device="cuda", generator=g) for o in outs]
    sum((o * gg).sum() for o, gg in zip(outs, grads)).backward()
    a64, b64 = a.detach().double(), b.detach().double()
    ratios = [R.worst_ratio(outs[0], R.correlation(a64, b64, *attrs), R.correlation(a64.abs(), b64.abs(), *attrs))]
    if bidir:
        ratios.append(R.worst_ratio(outs[1], R.correlation(b64, a64, *attrs),
                                    R.correlation(b64.abs(), a64.abs(), *attrs)))
    # d/da of sum(g0 * corr(a, b)) + sum(g1 * corr(b, a))
    ga, gb, Aa, Ab = R.correlation_grads(grads[0].double(), a64, b64, attrs, skip_row)
    if bidir:
        gb2, ga2, Ab2, Aa2 = R.correlation_grads(grads[1].double(), b64, a64, attrs, skip_row)
        ga, gb, Aa, Ab = ga + ga2, gb + gb2, Aa + Aa2, Ab + Ab2
    return ratios, R.worst_ratio(a.grad, ga, Aa), R.worst_ratio(b.grad, gb, Ab)


@pytest.mark.parametrize("shape,attrs", [((2, 5, 11, 14), (3, 4, 5, 2, 2)), ((1, 7, 9, 10), (3, 2, 3, 1, 1)),
                                         ((2, 3, 13, 18), (1, 4, 2, 1, 2))])
def test_correlation_generic_kernel_vs_float64(shape, attrs):
    from unflow_b200 import _native
    assert _native.lib().unflow_correlation_fwd_path(shape[1], shape[2], shape[3], *attrs) == 0
    fwd, ra, rb = _corr_case(shape, attrs, 3, False)
    print("\nfwd %s  g0 %.3e  g1 %.3e" % (fwd, ra, rb))
    assert max(fwd + [ra, rb]) <= TAU_SUM


@pytest.mark.parametrize("shape,md", [((2, 64, 48, 160), 8), ((2, 64, 48, 160), 16), ((2, 200, 48, 160), 20),
                                      ((1, 130, 20, 36), 4)])
def test_correlation_tiled_kernels_vs_float64(shape, md):
    """Forward of both volumes, fold and backward of the tiled kernels: the run-time radius path (even
    r = md / 2 < 10) and channel counts that leave a partial 128-channel slab."""
    attrs = (1, md, md, 1, 2)
    fwd, ra, rb = _corr_case(shape, attrs, 4, True)
    print("\nfwd %s  g0 %.3e  g1 %.3e" % (fwd, ra, rb))
    assert max(fwd + [ra, rb]) <= TAU_SUM


def test_correlation_bound_catches_a_dropped_displacement_row():
    _, good_a, good_b = _corr_case((1, 16, 12, 40), (1, 8, 8, 1, 2), 5, True)
    _, bad_a, bad_b = _corr_case((1, 16, 12, 40), (1, 8, 8, 1, 2), 5, True, skip_row=1)
    print("\ncorrect %.3e / %.3e, row dropped %.3e / %.3e" % (good_a, good_b, bad_a, bad_b))
    assert max(good_a, good_b) <= TAU_SUM
    assert min(bad_a, bad_b) > 1000 * TAU_SUM


# ---- warps ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(4, 384, 1280, 3), (4, 96, 320, 2)])
@pytest.mark.parametrize("mode", [0, 1])
def test_warp_vs_float64(shape, mode):
    from unflow_b200 import _native
    B, H, W, C = shape
    lib = _native.lib()
    g = torch.Generator(device="cuda").manual_seed(H + C)
    img = torch.rand(B, H, W, C, device="cuda", generator=g)
    flow = make_flows(B, H, W, "edges", 11).cuda() * 1.0
    cat = torch.randint(0, 6, (B, H, W), device="cuda", generator=g)
    flow[..., 0] = torch.where(cat == 0, flow[..., 0] + 3 * W, torch.where(cat == 1, flow[..., 0] - 3 * W, flow[..., 0]))
    flow[..., 1] = torch.where(cat == 2, flow[..., 1].round(), flow[..., 1])
    out = torch.empty_like(img)
    assert lib.unflow_backward_warp_fwd(img.data_ptr(), flow.data_ptr(), out.data_ptr(), B, H, W, C, mode, _st()) == 0
    grad = torch.randn(B, H, W, C, device="cuda", generator=g)
    dflow, dimg = torch.empty_like(flow), torch.zeros_like(img)
    assert lib.unflow_backward_warp_bwd(grad.data_ptr(), img.data_ptr(), flow.data_ptr(), dflow.data_ptr(),
                                        dimg.data_ptr(), B, H, W, C, mode, _st()) == 0
    torch.cuda.synchronize()
    i64, f64 = img.double(), flow.double()
    rf = R.worst_ratio(out, R.warp(i64, f64, mode), R.warp_abs(i64, f64, mode))
    di, df, Ai, Af = R.warp_grads(grad.double(), i64, f64, mode)
    ri, rfl = R.worst_ratio(dimg, di, Ai), R.worst_ratio(dflow, df, Af)
    print("\nout %.3e  dimage %.3e  dflow %.3e" % (rf, ri, rfl))
    assert max(rf, ri, rfl) <= TAU_SUM


def test_image_warp_fraction_just_below_an_integer():
    """image_warp with u = -1.5 * 2^-24 beside a zero tap: the fp32 fraction u - floor(u) = 1 - 1.5 * 2^-24 rounds
    to 1 - 2^-23, so the left tap weighs 2^-23 instead of 1.5 * 2^-24.  The kernel does what the reference op does;
    a float64 reference with the exact fraction is off by 1/3 of A here (a stacked network's image_warp in the
    CSS step reached 4.6e-6 of A that way, over TAU_SUM).  float64_refs takes the fraction from the fp32 rounding."""
    from unflow_b200 import _native
    B, H, W, C = 1, 2, 8, 3
    lib = _native.lib()
    img = (torch.arange(W, device="cuda") % 2 == 0).float().view(1, 1, W, 1).expand(B, H, W, C).contiguous()
    flow = torch.zeros(B, H, W, 2, device="cuda")
    flow[..., 0] = -1.5 * 2.0 ** -24
    out, grad = torch.empty_like(img), torch.ones_like(img)
    dflow, dimg = torch.empty_like(flow), torch.zeros_like(img)
    assert lib.unflow_backward_warp_fwd(img.data_ptr(), flow.data_ptr(), out.data_ptr(), B, H, W, C, 1, _st()) == 0
    assert lib.unflow_backward_warp_bwd(grad.data_ptr(), img.data_ptr(), flow.data_ptr(), dflow.data_ptr(),
                                        dimg.data_ptr(), B, H, W, C, 1, _st()) == 0
    torch.cuda.synchronize()
    i64, f64 = img.double(), flow.double()
    ratios = [R.worst_ratio(out, R.warp(i64, f64, 1), R.warp_abs(i64, f64, 1))]
    di, df, Ai, Af = R.warp_grads(grad.double(), i64, f64, 1)
    ratios += [R.worst_ratio(dimg, di, Ai), R.worst_ratio(dflow, df, Af)]
    exact = R.worst_ratio(out[:, :, 1::2], torch.full_like(out[:, :, 1::2], 1.5 * 2.0 ** -24, dtype=torch.float64),
                          torch.full_like(out[:, :, 1::2], 1.5 * 2.0 ** -24, dtype=torch.float64))
    print("\nout %.3e  dimage %.3e  dflow %.3e; against the exact fraction %.3e" % (*ratios, exact))
    assert max(ratios) <= TAU_SUM
    assert exact > 0.3


def test_spatial_transformer_sampler_vs_float64():
    from unflow_b200 import _native
    B, H, W, C = 2, 96, 320, 3
    g = torch.Generator(device="cuda").manual_seed(2)
    img = torch.rand(B, H, W, C, device="cuda", generator=g)
    coords = torch.stack([torch.rand(B, H, W, device="cuda", generator=g) * (W + 40) - 20,
                          torch.rand(B, H, W, device="cuda", generator=g) * (H + 40) - 20], -1)
    coords[:, ::7, :, 0] = W - 1.0
    coords[:, :, ::5, 1] = coords[:, :, ::5, 1].round()
    out = torch.empty_like(img)
    assert _native.lib().unflow_backward_warp_fwd(img.data_ptr(), coords.data_ptr(), out.data_ptr(), B, H, W, C, 2,
                                                  _st()) == 0
    torch.cuda.synchronize()
    r = R.worst_ratio(out, R.warp(img.double(), coords.double(), 2), R.warp_abs(img.double(), coords.double(), 2))
    print("\nout %.3e" % r)
    assert r <= TAU_SUM


@pytest.mark.parametrize("scale", [3.0, 40.0])
def test_forward_warp_vs_float64(scale):
    """Splat map and its flow gradient.  The in-tile splats are fixed point (each weight rounded to 2^-24), so the
    forward's A adds 2^-24 per splat received to the map value."""
    from unflow_b200 import _native
    B, H, W = 4, 96, 320
    lib = _native.lib()
    g = torch.Generator(device="cuda").manual_seed(int(scale))
    flow = (torch.rand(B, H, W, 2, device="cuda", generator=g) * 2 - 1) * scale
    out = torch.empty(B, H, W, 1, device="cuda")
    assert lib.unflow_forward_warp_fwd(flow.data_ptr(), out.data_ptr(), B, H, W, _st()) == 0
    grad = torch.randn(B, H, W, 1, device="cuda", generator=g)
    dflow = torch.empty_like(flow)
    assert lib.unflow_forward_warp_bwd(grad.data_ptr(), flow.data_ptr(), dflow.data_ptr(), B, H, W, _st()) == 0
    torch.cuda.synchronize()
    ref, count = R.forward_warp(flow.double())
    rf = R.worst_ratio(out, ref, ref + count * 2.0 ** -24 / TAU_SUM)
    df, A = R.forward_warp_grads(grad.double(), flow.double())
    rg = R.worst_ratio(dflow, df, A)
    print("\nout %.3e  dflow %.3e  (pixels receiving nothing: %.1f %%)" % (rf, rg, 100 * float((count == 0).double().mean())))
    assert rf <= TAU_SUM and rg <= TAU_SUM


# ---- Adam ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("step", [1, 7])
@pytest.mark.parametrize("entry", ["adam_step", "adam_step_l2", "adam_step_dev", "adam_step_dev_l2"])
def test_adam_entry_points_vs_float64(entry, step):
    from unflow_b200 import _native
    lib = _native.lib()
    n = 4 * 3001
    g = torch.Generator(device="cuda").manual_seed(step)
    p = torch.randn(n, device="cuda", generator=g) * 0.05
    gr = torch.randn(n, device="cuda", generator=g) * 1e-3
    m = torch.randn(n, device="cuda", generator=g) * 1e-4
    v = torch.rand(n, device="cuda", generator=g) * 1e-6
    mask = torch.randint(0, 16, (n // 4,), device="cuda", generator=g, dtype=torch.uint8)
    # the hyper-parameters are fp32 in the ABI: the reference takes the same fp32 values (1 - 0.999f is not 0.001)
    lr, b1, b2, eps, gs, l2 = (float(np.float32(x)) for x in (1e-4, 0.9, 0.999, 1e-8, 0.5, 4e-4))
    l2m = l2_bits(mask.data_ptr(), n) if entry.endswith("l2") else torch.zeros(n, device="cuda", dtype=torch.float64)
    (p1, m1, v1), (Ap, Am, Av) = adam_reference(p.double(), gr.double(), m.double(), v.double(), lr, b1, b2, eps, gs,
                                                 float(step), l2m, l2 if entry.endswith("l2") else 0.0)
    ptrs = (p.data_ptr(), gr.data_ptr(), m.data_ptr(), v.data_ptr(), n)
    hyper = torch.tensor([lr, b1, b2, eps, gs, float(step)], device="cuda")
    fn = getattr(lib, "unflow_" + entry)
    if entry == "adam_step":
        rc = fn(*ptrs, lr, b1, b2, eps, step, gs, 1, _st())
    elif entry == "adam_step_l2":
        rc = fn(*ptrs, lr, b1, b2, eps, step, gs, 1, mask.data_ptr(), l2, _st())
    elif entry == "adam_step_dev":
        rc = fn(*ptrs, hyper.data_ptr(), 1, _st())
    else:
        rc = fn(*ptrs, hyper.data_ptr(), 1, mask.data_ptr(), l2, _st())
    assert rc == 0
    torch.cuda.synchronize()
    ratios = [R.worst_ratio(p, p1, Ap), R.worst_ratio(m, m1, Am), R.worst_ratio(v, v1, Av)]
    print("\nparam %.3e  m %.3e  v %.3e" % tuple(ratios))
    assert max(ratios) <= TAU_ADAM
    assert not bool(gr.any())
    if "dev" in entry:
        assert float(hyper[5]) == step + 1
