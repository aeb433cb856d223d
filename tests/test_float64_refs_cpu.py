"""The float64 references of the GPU checks, pinned on the CPU to sources that do not derive from them.

Every float64 check of a kernel (tests/test_gpu_step_launches.py, test_gpu_float64_kernels.py, the variant, batch,
supervised, tensor-core, objective, network and data-parallel files) measures it with tests/float64_refs.py, the
ref_* convolutions of test_gpu_tc_step_launches.py and adam_reference / tf32_rna / l2_bits of
test_gpu_step_launches.py.  A reference that shares a misreading with its kernel passes all of them, so each one is
held here to at least one independent source: the reference CUDA kernels' outputs (tests/golden/
reference_kernels.npz), the reference's own Python run (tests/golden/reference_run.npz), the oracle's
restatements (oracle/losses.py, oracle/tf_compat.py, oracle/supervised.py) and the loop definitions of
oracle/brute.py, or a definition written out here (TF's Adam rule, the TF32 bit rounding, pixel loops).
Each error scale A (|got - ref| <= TAU * A in the GPU files) is held to A >= |ref|, to A == |ref| where the
operation is linear in non-negative operands, and to the tightness measured below, so a loosened A fails.

Worst deviation of each pin, as |reference - source| / max |source| (float32 sources) or relative (float64):
  correlation            reference kernels corr0..2: out 2.2e-7, d0 / d1 4.7e-7 (corr1, ks 3); brute (ks 3, s1 2,
                         s2 2, pad 3 != md 4): 4.8e-17
  fold_reverse           symmetry of corr(in1, in0): bitwise; adjoint identity to 1e-12
  downsample             reference kernels down2 / down4: 1.3e-7; brute: 0
  warp mode 0            reference kernels bwarp out 9.7e-8, dflow 1.3e-7; brute zero-padded warp: 0
  warp mode 1            reference run warp_out 1.4e-7, warp_dim 6.7e-8, warp_dflow 1.1e-6; brute clamped warp: 0;
                         the fp32 fraction bit for bit, a flow 2^-30 below 0 takes the pixel itself
  warp mode 2            reference run spatial transformer: 3.2e-7
  forward_warp           reference kernels fwarp out 2.5e-7, dflow 3.0e-7; brute 7.9e-16
  census, gray255        oracle ternary_transform / rgb_to_grayscale, R = 1, 2, 3: 0 / 0
  masks_f32              border, outgoing: bitwise; fb and disocc: bitwise to the oracle's compute_losses masks, and
                         fb to the reference's occ_fw / occ_bw outside the band between its occlusion() threshold
                         (unwarped |f_bw|^2) and compute_losses' (warped)
  level_losses           every term of the reference's compute_losses, occlusion fb / '' / disocc: 1.8e-7 relative
  level_loss_grads       the reference's flow gradients (its Sobel term from the oracle): 1.7e-6 of A = 0.029 TAU_LOSS;
                         gradcheck on a 1x5x6 level passes
  supervised_loss_grads  oracle charbonnier_loss of its resize and a pixel loop from TF's resize definition: < 1e-12
  ref_conv / ref_wgrad   tf_compat SAME convs (7x7 / 5x5 / 3x3 s2, 3x3 s1, k4 s2 deconvs): 0; pixel loops, autograd
                         (ref_wgrad, ref_wgrad_window) and ref_conv for the window forms: < 1e-12
  adam_reference         TF's AdamOptimizer rule with the oracle's L2 gradient, steps 1, 2, 1000: 0
  tf32_rna, l2_bits      bitwise, incl. ties, carries, +-0, subnormals, inf and NaN; bitwise to train.l2_mask_bytes

Tightness of the error scales (sum A / sum |ref| on the seeded inputs; A == |ref| where it must be):
  warp_grads dflow 5.8 (mode 1), forward_warp_grads 3.9, charb_d_scale with a 1e-3 operand error 1.008,
  level_loss_grad_scale 2760 / 3343 / 2974 (golden level fb / '' / disocc: near a zero charbonnier argument the
  scale is K(x) |operands|, K ~ 1800), adam_reference param 1.0.  Each is asserted within 1.2x of these.

Negative controls (each misreading monkeypatched into the reference; margin = its deviation / the pin's bound):
  correlation / (C) instead of / (ks^2 C): 8e12 (visible only at ks 3)     skip_row: 7e11
  ref_conv mode 1 offset off by one: 1.8e12                               skip_tap (each tap, modes 0 / 1 / 2): >= 7.7e4
  census margin R - 1 ('margin'): 1.0e4                                   census clamp_census: 2e12
  SECOND_ORDER's second diagonal flipped: 67                              smooth_2nd normaliser 4 -> 2: 5.0e4
  fb threshold 0.5 -> 0.05: 828 mask bits                                 detach_fb: 62, and gradcheck fails
  Adam's eps inside the sqrt: 6.6e8                                       tf32_rna truncating: 2029 of 4120 inputs
The level loss is blind to 'clamp_census' (its transform mask keeps every census window inside the image), as
tests/test_gpu_float64_kernels.py states of the kernel; census() itself fails its pin with it.  The whole file
takes about 30 s.
"""
import math
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import float64_refs as R
import synth
from oracle import brute
from oracle import losses as olosses
from oracle import tf_compat
from oracle.flownet import FLOW_SCALE
from oracle.image_warp import image_warp as oimage_warp
from oracle.unsupervised import regularization_loss
from test_gpu_step_launches import _lrelu_d, adam_reference, l2_bits, tf32_rna
from test_gpu_tc_step_launches import ref_conv, ref_conv_window, ref_wgrad, ref_wgrad_window

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_reference_kernels as MK  # noqa: E402

K = np.load(os.path.join(HERE, "golden", "reference_kernels.npz"))
G = synth.ReferenceRun(os.path.join(HERE, "golden", "reference_run.npz"))
WEIGHTS = dict(ternary=1.0, smooth_2nd=3.0, fb=0.2, occ=12.4, photo=0.5, grad=0.25, smooth_1st=0.75, sym=0.3)
LEVEL_CASES = [('fb', 1, True, 3), ('none', 0, False, 1), ('disocc', 2, True, 2)]   # tag, occl, border, R

TOL_F32 = 1e-5          # against a float32 source: of its largest magnitude (as tests/test_reference_kernels.py)
TOL_F64 = 1e-12         # against a float64 source: relative
TAU_LOSS = 6e-5         # the level-loss kernels' bound, |got - ref| <= TAU_LOSS * A (tests/test_gpu_step_launches.py)
TOL_LOSS = 2e-5         # a loss term of the reference's float32 run: relative (tests/test_oracle_vs_reference_run.py)

# ---- which reference each pin claims --------------------------------------------------------------------------
PINNED = set()
# the error scales A that must come with a pin of their own ("A:" + the function that returns or defines it)
A_SCALES = ["A:correlation", "A:correlation_grads", "A:downsample", "A:warp_abs", "A:warp_grads",
            "A:forward_warp_grads", "A:charb_d_scale", "A:level_loss_grad_scale", "A:ref_conv", "A:ref_wgrad",
            "A:adam_reference"]
# public callables of float64_refs that are not references of an operation
NOT_REFERENCES = {
    "view": "device pointers as tensors; CUDA only, used by tests/test_gpu_float64_refs.py",
    "record_kink_sides": "records the product network's leaky-ReLU sides; no value of its own",
    "follow_kink_sides": "replays them into the oracle network; no value of its own",
}


def pins(*names):
    def mark(fn):
        PINNED.update(names)
        return fn
    return mark


def dev(got, want, scale=None):
    """max |got - want| / scale (default: max |want|)."""
    got, want = torch.as_tensor(got).double(), torch.as_tensor(want).double()
    s = float(want.abs().max()) if scale is None else float(scale)
    return float((got - want).abs().max()) / max(s, 1e-300)


def rel(got, want):
    """max |got - want| / |want| elementwise (0 / 0 = 0)."""
    got, want = torch.as_tensor(got).double(), torch.as_tensor(want).double()
    err = (got - want).abs()
    return float(torch.where(err == 0, torch.zeros_like(err), err / want.abs().clamp_min(1e-300)).max())


def sample_dev(t, key):
    """t against the reference kernel output `key` of reference_kernels.npz, at its stored positions."""
    assert tuple(t.shape) == tuple(int(v) for v in K[key + "_shape"]), key
    got = t.detach().double().reshape(-1).numpy()[K[key + "_idx"]]
    return float(np.abs(got - K[key + "_val"]).max() / K[key + "_absmax"])


def bounds(A, ref):
    """A >= |ref| elementwise within 1e-12 relative."""
    return bool((ref.abs() <= A * (1 + 1e-12) + 1e-300).all())


def tight(A, ref):
    return float(A.sum() / ref.abs().sum())


def g64(key):
    return torch.from_numpy(np.asarray(G[key])).double()


# ---- correlation, fold_reverse ----------------------------------------------------------------------------------
def _attrs(a):
    return (a["kernel_size"], a["max_displacement"], a["pad"], a["stride_1"], a["stride_2"])


def corr_pin(cases=(0, 1, 2), **kw):
    """Worst deviation of correlation / correlation_grads from the reference kernels' samples and from
    brute.correlation (ks 3, s1 2, s2 2, pad 3 != md 4).  corr2 (256 channels, d = 20) takes its gradients on the
    channels of 16 sampled positions: the correlation is a sum over channels divided by ks^2 C, so the gradient of
    a channel subset S is correlation_grads on S times |S| / C."""
    out = {}
    for i in cases:
        B, C, H, W, attrs = MK.CORR_CASES[i]
        g, a, b = MK.corr_inputs(B, C, H, W)
        at = _attrs(attrs)
        a, b = a.double(), b.double()
        ref = R.correlation(a, b, *at, **kw)
        out["corr%d out" % i] = sample_dev(ref, "corr%d_out" % i)
        go = torch.randn(ref.shape, generator=g).double()
        if C <= 32:
            g0, g1, _, _ = R.correlation_grads(go, a, b, at, **kw)
            out["corr%d d0" % i] = sample_dev(g0, "corr%d_d0" % i)
            out["corr%d d1" % i] = sample_dev(g1, "corr%d_d1" % i)
            continue
        for key, k in (("d0", 0), ("d1", 1)):
            idx = K["corr%d_%s_idx" % (i, key)]
            chan = (idx // (H * W)) % C
            S = sorted(set(chan.tolist()))[:16]
            gs = R.correlation_grads(go, a[:, S], b[:, S], at, **kw)[k] * (len(S) / C)
            full = torch.zeros(B, C, H, W, dtype=torch.float64)
            full[:, S] = gs
            sel = np.isin(chan, S)
            got = full.reshape(-1).numpy()[idx[sel]]
            out["corr%d %s" % (i, key)] = float(np.abs(got - K["corr%d_%s_val" % (i, key)][sel]).max()
                                                / K["corr%d_%s_absmax" % (i, key)])
    gen = torch.Generator().manual_seed(5)
    a, b = torch.randn(1, 5, 12, 16, generator=gen).double(), torch.randn(1, 5, 12, 16, generator=gen).double()
    want = brute.correlation(a.numpy(), b.numpy(), kernel_size=3, max_displacement=4, pad=3, stride_1=2, stride_2=2)
    out["brute"] = dev(R.correlation(a, b, 3, 4, 3, 2, 2, **kw), torch.from_numpy(want)) * TOL_F32 / TOL_F64
    return out


@pins("correlation", "correlation_grads", "corr_geometry")
def test_correlation_against_the_reference_kernels_and_brute():
    out = corr_pin()
    assert max(out.values()) <= TOL_F32, out
    for i, (B, C, H, W, attrs) in enumerate(MK.CORR_CASES):
        ngr, D, oh, ow = R.corr_geometry(H, W, *_attrs(attrs))
        assert (B, D * D, oh, ow) == tuple(int(v) for v in K["corr%d_out_shape" % i])


@pins("A:correlation", "A:correlation_grads")
def test_correlation_error_scales():
    gen = torch.Generator().manual_seed(6)
    at = (3, 4, 3, 2, 2)
    a, b = torch.randn(2, 4, 12, 16, generator=gen).double(), torch.randn(2, 4, 12, 16, generator=gen).double()
    ref = R.correlation(a, b, *at)
    go = torch.randn(ref.shape, generator=gen).double()
    assert bounds(R.correlation(a.abs(), b.abs(), *at), ref)
    g0, g1, A0, A1 = R.correlation_grads(go, a, b, at)
    assert bounds(A0, g0) and bounds(A1, g1)
    a, b, go = a.abs(), b.abs(), go.abs()
    assert rel(R.correlation(a, b, *at), R.correlation(a, b, *at).abs()) == 0
    g0, g1, A0, A1 = R.correlation_grads(go, a, b, at)
    assert rel(A0, g0) <= 1e-12 and rel(A1, g1) <= 1e-12


def test_negative_controls_of_the_correlation_pin(monkeypatch):
    """1 / C instead of 1 / (ks^2 C) shows only where ks > 1: corr1 and the brute case."""
    real = R.correlation
    monkeypatch.setattr(R, "correlation", lambda a, b, ks, *r, **kw: real(a, b, ks, *r, **kw) * ks * ks)
    assert max(corr_pin(cases=(1,)).values()) > 1e5 * TOL_F32
    monkeypatch.setattr(R, "correlation", real)
    assert max(corr_pin(cases=(0, 1), skip_row=0).values()) > 1e5 * TOL_F32


@pins("fold_reverse")
def test_fold_reverse_is_the_symmetry_of_the_correlation_and_self_adjoint():
    """corr(b, a)[-p, -o](y + s2 p, x + s2 o) = corr(a, b)[p, o](y, x): fold_reverse(corr(in1, in0)) equals
    corr(in0, in1) where the shifted pixel is inside and is 0 elsewhere; <fold_reverse(g), c> = <g, unfold(c)>."""
    gen = torch.Generator().manual_seed(7)
    ks, md, pad, s1, s2 = 1, 4, 4, 1, 2
    a, b = torch.randn(2, 3, 9, 11, generator=gen).double(), torch.randn(2, 3, 9, 11, generator=gen).double()
    ngr, D, oh, ow = R.corr_geometry(9, 11, ks, md, pad, s1, s2)
    c01, c10 = R.correlation(a, b, ks, md, pad, s1, s2), R.correlation(b, a, ks, md, pad, s1, s2)
    got = R.fold_reverse(c10, s2, ngr).view(2, D, D, oh, ow)
    want = c01.view(2, D, D, oh, ow)

    def unfold(c):          # the pixel loop: unfold(c)[(q, r)](y, x) = c[(-q, -r)](y + s2 q, x + s2 r), 0 outside
        c = c.view(2, D, D, oh, ow)
        u = torch.zeros_like(c)
        for q in range(-ngr, ngr + 1):
            for r in range(-ngr, ngr + 1):
                for y in range(oh):
                    for x in range(ow):
                        yy, xx = y + s2 * q, x + s2 * r
                        if 0 <= yy < oh and 0 <= xx < ow:
                            u[:, q + ngr, r + ngr, y, x] = c[:, ngr - q, ngr - r, yy, xx]
        return u.view(2, D * D, oh, ow)
    inside = unfold(torch.ones_like(c10)).view(2, D, D, oh, ow) != 0
    assert torch.equal(got[inside], want[inside]) and not bool(got[~inside].any())
    assert 0 < int(inside.sum()) < inside.numel()
    g, c = torch.randn(c10.shape, generator=gen).double(), torch.randn(c10.shape, generator=gen).double()
    lhs, rhs = float((R.fold_reverse(g, s2, ngr) * c).sum()), float((g * unfold(c)).sum())
    assert abs(lhs - rhs) <= 1e-12 * float((g.abs() * unfold(c.abs())).sum())


# ---- downsample, warps, forward warp ----------------------------------------------------------------------------
def warp_golden():
    """The inputs of reference_kernels' warp / forward warp / downsample samples, drawn as the generator did."""
    g, im, fl = MK.warp_inputs()
    go_b = torch.randn(tuple(int(v) for v in K["bwarp_out_shape"]), generator=g)
    go_f = torch.randn(tuple(int(v) for v in K["fwarp_out_shape"]), generator=g)
    x = torch.rand(2, 16, 24, 3, generator=g)
    return im.double(), fl.double(), go_b.double(), go_f.double(), x.double()


def quantised(t):
    """Flows on a 2^-10 grid: pixel + flow is exact in fp32, so the fp32-rounded positions of the references are
    the exact ones of the brute definitions."""
    return torch.round(t * 1024) / 1024


@pins("downsample", "A:downsample")
def test_downsample_against_the_reference_kernels_and_brute():
    x = warp_golden()[4]
    for s in (2, 4):
        assert sample_dev(R.downsample(x, s), "down%d_out" % s) <= TOL_F32
        assert dev(R.downsample(x, s), torch.from_numpy(brute.downsample(x.numpy(), s))) <= TOL_F64
        assert rel(R.downsample(x.abs(), s), R.downsample(x, s).abs()) == 0         # x >= 0: A == |ref|
        xs = x - 0.5
        assert bounds(R.downsample(xs.abs(), s), R.downsample(xs, s))


def warp_pins(**kw):
    im, fl, go_b, _, _ = warp_golden()
    out = {"bwarp out": sample_dev(R.warp(im, fl, 0, **kw), "bwarp_out"),
           "bwarp dflow": sample_dev(R.warp_grads(go_b, im, fl, 0, **kw)[1], "bwarp_dflow")}
    fq = quantised(fl)
    out["brute zero"] = dev(R.warp(im, fq, 0, **kw), torch.from_numpy(brute.backward_warp_zero(im.numpy(), fq.numpy())))
    out["brute zero"] *= TOL_F32 / TOL_F64
    im1, ffw = g64("L_im1"), g64("L_ffw")
    gsel = torch.linspace(-1, 1, im1.numel(), dtype=torch.float32).reshape(im1.shape).double()
    out["warp_out"] = dev(R.warp(im1, ffw, 1, **kw), g64("warp_out"))
    dimg, dflow, _, _ = R.warp_grads(gsel, im1, ffw, 1, **kw)
    out["warp_dim"], out["warp_dflow"] = dev(dimg, g64("warp_dim")), dev(dflow, g64("warp_dflow"))
    fq = quantised(ffw * 3)
    want = torch.from_numpy(brute.backward_warp_clamp(im1.numpy(), fq.numpy()))
    out["brute clamp"] = dev(R.warp(im1, fq, 1, **kw), want) * TOL_F32 / TOL_F64
    out["transformer"] = dev(stn_warp(**kw), g64("aug_transformer"))
    return out


def stn_coords():
    """The spatial transformer's sample positions of reference_run's aug_* case (fp32, as its _meshgrid and
    _interpolate form them), embedded in a [B, H, W, 2] field of the input's size (mode 2 clamps to it)."""
    U, theta = g64("aug_im1"), torch.from_numpy(np.asarray(G["aug_theta"])).reshape(-1, 2, 3)
    B, H, W, _ = U.shape
    oh, ow = 20, 30
    x_t = torch.linspace(-1.0, 1.0, ow).view(1, ow).expand(oh, ow)
    y_t = torch.linspace(-1.0, 1.0, oh).view(oh, 1).expand(oh, ow)
    grid = torch.stack([x_t.reshape(-1), y_t.reshape(-1), torch.ones(oh * ow)], 0)
    T = theta @ grid
    coords = torch.zeros(B, H, W, 2, dtype=torch.float64)
    coords[:, :oh, :ow, 0] = ((T[:, 0] + 1.0) * float(W) / 2.0).view(B, oh, ow).double()
    coords[:, :oh, :ow, 1] = ((T[:, 1] + 1.0) * float(H) / 2.0).view(B, oh, ow).double()
    return U, coords


def stn_warp(**kw):
    U, coords = stn_coords()
    return R.warp(U, coords, 2, **kw)[:, :20, :30]


@pins("warp", "warp_taps", "warp_grads")
def test_warps_against_the_reference_kernels_run_and_brute():
    out = warp_pins()
    assert max(out.values()) <= TOL_F32, out


def test_negative_controls_of_the_warp_pins():
    for t in range(4):
        out = warp_pins(skip_tap=t)
        for key in ("bwarp out", "brute zero", "warp_out", "brute clamp", "transformer"):
            assert out[key] > 1e4 * TOL_F32, (t, key, out[key])


@pins("_fp32_frac", "_fp32_sum")
def test_fp32_fraction_bit_for_bit_and_a_flow_a_hair_below_an_integer():
    """image_warp's weights come from the fp32 difference f - floor(f): bit for bit, derivative 1.  A flow u a hair
    below 0 has the fp32 fraction 1, so the warp takes the pixel itself, not 2^-30 of its left neighbour."""
    f32 = np.array([np.nextafter(np.float32(k), np.float32(-np.inf)) for k in range(-3, 4)] +
                   [-2.0 ** -30, 2.0 ** -30, 0.5, -0.5, 123.456, -7.999], dtype=np.float32)
    f32 = np.concatenate([f32, np.random.default_rng(1).normal(0, 8, 64).astype(np.float32)])
    f = torch.from_numpy(f32).double().requires_grad_(True)
    fl = torch.floor(f.detach())
    got = R._fp32_frac(f, fl)
    want = torch.from_numpy((f32 - np.floor(f32)).astype(np.float32)).double()
    assert torch.equal(got.detach(), want)
    assert torch.equal(torch.autograd.grad(got.sum(), f)[0], torch.ones_like(f))
    s = R._fp32_sum(torch.arange(f.numel()), f)
    assert torch.equal(s.detach(), (torch.arange(f.numel()).float() + f.detach().float()).double())
    img = torch.rand(1, 3, 5, 2, dtype=torch.float64)
    flow = torch.zeros(1, 3, 5, 2, dtype=torch.float64)
    flow[..., 0] = -2.0 ** -30
    assert torch.equal(R.warp(img, flow, 1), img)
    assert not torch.equal(torch.from_numpy(brute.backward_warp_clamp(img.numpy(), flow.numpy()))[:, :, 1:], img[:, :, 1:])


@pins("A:warp_abs", "warp_abs", "A:warp_grads")
def test_warp_error_scales():
    """A == |ref| for non-negative images and upstream gradients (every bilinear weight is >= 0 with in-image
    positions); dflow's A is >= |dflow|, 2.4x it in sum on the reference run's level."""
    im1, ffw = g64("L_im1"), g64("L_ffw")
    gen = torch.Generator().manual_seed(8)
    grad = torch.randn(im1.shape, generator=gen).double()
    _, coords = stn_coords()
    stn_img = g64("aug_im1")
    for img, flow, mode in ((im1, ffw, 0), (im1, ffw, 1), (stn_img, coords.clamp(0, 23), 2)):
        g = grad if mode != 2 else torch.randn(img.shape, generator=gen).double()
        ref = R.warp(img - 0.5, flow, mode)
        assert bounds(R.warp_abs(img - 0.5, flow, mode), ref)
        assert rel(R.warp_abs(img, flow, mode), R.warp(img, flow, mode)) <= 1e-15
        dimg, dflow, Ai, Af = R.warp_grads(g, img - 0.5, flow, mode)
        assert bounds(Ai, dimg) and bounds(Af, dflow), mode
        dimg, _, Ai, _ = R.warp_grads(g.abs(), img, flow, mode)
        assert rel(Ai, dimg) <= 1e-12, mode
        if mode == 1:
            assert tight(Af, dflow) < 1.2 * 5.8, tight(Af, dflow)


@pins("forward_warp", "forward_warp_splats", "forward_warp_grads", "A:forward_warp_grads")
def test_forward_warp_against_the_reference_kernels_and_brute():
    _, fl, _, go_f, _ = warp_golden()
    out, count = R.forward_warp(fl)
    assert sample_dev(out, "fwarp_out") <= TOL_F32
    dflow, A = R.forward_warp_grads(go_f, fl)
    assert sample_dev(dflow, "fwarp_dflow") <= TOL_F32
    assert bounds(A, dflow) and tight(A, dflow) < 1.2 * 3.9, tight(A, dflow)
    fq = quantised(fl)
    assert dev(R.forward_warp(fq)[0], torch.from_numpy(brute.forward_warp(fq.numpy()))) <= TOL_F64
    assert torch.equal(count > 0, out > 0)


# ---- census, masks, level losses ----------------------------------------------------------------------------------
@pins("census", "gray255")
def test_census_against_the_oracle_ternary_transform():
    gen = torch.Generator().manual_seed(9)
    im = torch.rand(2, 9, 11, 3, generator=gen).double()
    assert dev(R.gray255(im), tf_compat.rgb_to_grayscale(im)[..., 0] * 255) == 0
    for r in (1, 2, 3):
        want = olosses.ternary_transform(im, r)
        assert dev(R.census(R.gray255(im), r), want) <= TOL_F64, r
        assert dev(R.census(R.gray255(im), r, clamp=True), want) > 1e-2, r         # clamp_census


def golden_level(tag, occl, use_border, r, bits=None):
    im1, im2, ffw, fbw = (g64(k) for k in ("L_im1", "L_im2", "L_ffw", "L_fbw"))
    border = g64("border_mask") if use_border else None
    fw_fw = torch.from_numpy(brute.forward_warp(ffw.numpy()))
    fw_bw = torch.from_numpy(brute.forward_warp(fbw.numpy()))
    if bits is None:
        bits = sum(1 << k for k, name in enumerate(R.TERMS) if name != 'grad')
    L = R.LevelInputs(im1, im2, ffw, fbw, border, fw_fw, fw_bw, occl, r, bits)
    mfw, mbw = R.masks_f32(ffw, fbw, border, occl, fw_fw, fw_bw)
    return L, mfw.double(), mbw.double()


def oracle_masks(tag, mode, use_border):
    im1, im2, ffw, fbw = (torch.from_numpy(np.asarray(G[k])) for k in ("L_im1", "L_im2", "L_ffw", "L_fbw"))
    border = torch.from_numpy(np.asarray(G["border_mask"])) if use_border else None
    aux = olosses.compute_losses(im1, im2, ffw, fbw, border_mask=border, mask_occlusion=mode)['_aux']
    return aux['mask_fw'][..., 0], aux['mask_bw'][..., 0]


def masks_pin():
    """Number of mask bits of masks_f32 that differ from the oracle's compute_losses (occlusion fb)."""
    _, mfw, mbw = golden_level('fb', 1, True, 3)
    ofw, obw = oracle_masks('fb', 'fb', True)
    return int((mfw.float() != ofw).sum() + (mbw.float() != obw).sum())


@pins("masks_f32")
def test_masks_bit_exact_against_the_reference_run():
    ffw, fbw = torch.from_numpy(np.asarray(G["L_ffw"])), torch.from_numpy(np.asarray(G["L_fbw"]))
    border = torch.from_numpy(np.asarray(G["border_mask"]))
    mfw, mbw = R.masks_f32(ffw, fbw, border, 0, None, None)
    assert torch.equal(mfw, border[..., 0]) and torch.equal(mbw, border[..., 0])
    assert mfw.device == ffw.device
    mfw, _ = R.masks_f32(ffw * 4, fbw, None, 0, None, None)
    assert torch.equal(mfw, torch.from_numpy(np.asarray(G["outgoing_mask"]))[..., 0])
    assert masks_pin() == 0
    # the reference's occlusion() thresholds on the unwarped |f_bw|^2 (losses.py:125-134), compute_losses on the
    # warped one: the masks agree bit for bit except where |f + w(g)|^2 lies between the two thresholds
    ones = torch.ones_like(border)
    m = R.masks_f32(ffw, fbw, ones, 1, None, None)
    for k, (f, g) in enumerate(((ffw, fbw), (fbw, ffw))):
        occ = torch.from_numpy(np.asarray(G["occ_fw" if k == 0 else "occ_bw"]))[..., 0]
        gw = oimage_warp(g, f)
        d = olosses.length_sq(f + gw)[..., 0]
        t_warped = (0.01 * (olosses.length_sq(f) + olosses.length_sq(gw)) + 0.5)[..., 0]
        t_plain = (0.01 * (olosses.length_sq(ffw) + olosses.length_sq(fbw)) + 0.5)[..., 0]
        band = (d > torch.minimum(t_warped, t_plain)) & (d <= torch.maximum(t_warped, t_plain))
        assert torch.equal((1 - m[k])[~band], occ[~band]), k
        assert 0 < float(occ.mean()) < 1
    # disocc: the mask of each direction clears where the other direction's splat map is below 0.8
    fw_fw, fw_bw = (torch.from_numpy(brute.forward_warp(f.double().numpy())).float() for f in (ffw, fbw))
    mfw, mbw = R.masks_f32(ffw, fbw, border, 2, fw_fw, fw_bw)
    assert torch.equal(mfw, border[..., 0] * (fw_bw[..., 0] >= 0.8).float())
    assert torch.equal(mbw, border[..., 0] * (fw_fw[..., 0] >= 0.8).float())
    ofw, obw = oracle_masks('disocc', 'disocc', True)
    assert torch.equal(mfw, ofw) and torch.equal(mbw, obw)


def test_negative_control_of_the_mask_pin(monkeypatch):
    monkeypatch.setattr(R, "FB_OCC_OFFSET", 0.05)
    assert masks_pin() > 10


def level_pin():
    """Worst relative deviation of level_losses from the reference's compute_losses terms, all three modes."""
    worst = {}
    for tag, occl, use_border, r in LEVEL_CASES:
        L, mfw, mbw = golden_level(tag, occl, use_border, r)
        got = R.level_losses(L, L.ffw, L.fbw, mfw, mbw)
        for k, name in enumerate(R.TERMS):
            if name != 'grad':
                worst[tag + " " + name] = rel(got[k], float(G['cl_%s_%s' % (tag, name)]))
    return worst


@pins("level_losses", "LevelInputs", "charb")
def test_level_losses_against_the_reference_compute_losses():
    worst = level_pin()
    assert max(worst.values()) <= TOL_LOSS, worst
    L, mfw, mbw = golden_level('fb', 1, True, 3, bits=(1 << len(R.TERMS)) - 1)
    with pytest.raises(ValueError):
        R.level_losses(L, L.ffw, L.fbw, mfw, mbw)
    x = torch.linspace(-3, 3, 101, dtype=torch.float64)
    assert dev(R.charb(x), torch.tensor([brute.charbonnier(v) * 1 for v in x.tolist()])) <= TOL_F64


def _mutant_level_losses(monkeypatch, scale):
    real = R.level_losses

    def mutant(*a, **kw):
        return real(*a, **kw) * scale
    monkeypatch.setattr(R, "level_losses", mutant)


def test_negative_controls_of_the_level_loss_pin(monkeypatch):
    s = torch.ones(len(R.TERMS), dtype=torch.float64)
    s[R.TERMS.index('smooth_2nd')] = 2.0                               # smooth_2nd divided by 2 n, not 4 n
    with monkeypatch.context() as m:
        _mutant_level_losses(m, s)
        assert level_pin()['fb smooth_2nd'] > 1e4 * TOL_LOSS
    with monkeypatch.context() as m:
        m.setattr(R, "SECOND_ORDER", [(0, 1), (1, 0), (1, 1), (1, 1)])
        assert level_pin()['fb smooth_2nd'] > 10 * TOL_LOSS
    real = R.level_losses
    with monkeypatch.context() as m:
        m.setattr(R, "level_losses", lambda *a, **kw: real(*a, variant='margin'))
        assert level_pin()['fb ternary'] > 1e3 * TOL_LOSS
        # 'clamp_census' is not observable here: the transform mask keeps every census window inside the image
        # (tests/test_gpu_float64_kernels.py says the same of the kernel); census() itself fails its pin with it
        m.setattr(R, "level_losses", lambda *a, **kw: real(*a, variant='clamp_census'))
        assert max(level_pin().values()) <= TOL_LOSS


def sobel_grads(L, mfw, mbw, w):
    """The flow gradient of w * the Sobel term of the reference's compute_losses (oracle/losses.gradient_loss,
    float64): the golden gradients include it, level_losses does not evaluate it."""
    with torch.enable_grad():
        f, b = L.ffw.clone().requires_grad_(True), L.fbw.clone().requires_grad_(True)
        loss = (olosses.gradient_loss(L.im1, oimage_warp(L.im2, f), mfw[..., None]) +
                olosses.gradient_loss(L.im2, oimage_warp(L.im1, b), mbw[..., None])) * w
        return torch.autograd.grad(loss, (f, b))


def golden_gl():
    return torch.tensor([0.0 if name == 'grad' else WEIGHTS[name] for name in R.TERMS], dtype=torch.float64)


def grad_pin(variant=None):
    """Worst |got - want| / A of the weighted flow gradients against the reference's float32 run, all three modes,
    A = level_loss_grad_scale.  The reference's float32 gradients carry the rounding a float32 kernel does (a
    charbonnier derivative near 0 moves by ~1e-4 of max |grad| when its argument rounds), so they are held to the
    kernels' own bound, TAU_LOSS * A."""
    worst = 0.0
    for tag, occl, use_border, r in LEVEL_CASES:
        L, mfw, mbw = golden_level(tag, occl, use_border, r)
        gl = golden_gl()
        gf, gb = R.level_loss_grads(L, mfw, mbw, gl, variant)
        Af, Ab = R.level_loss_grad_scale(L, mfw, mbw, gl)
        sf, sb = sobel_grads(L, mfw, mbw, WEIGHTS['grad'])
        for got, A, key in ((gf + sf, Af, 'dfw'), (gb + sb, Ab, 'dbw')):
            want = g64('cl_%s_%s' % (tag, key))
            worst = max(worst, R.worst_ratio(want, got, A + sf.abs() if key == 'dfw' else A + sb.abs()))
    return worst


def small_level(seed=10):
    """A 1x5x6 level whose flows stay 0.25 away from integers (so finite differences do not cross a floor())."""
    gen = torch.Generator().manual_seed(seed)
    B, h, w = 1, 5, 6
    im1, im2 = torch.rand(B, h, w, 3, generator=gen).double(), torch.rand(B, h, w, 3, generator=gen).double()
    fl = lambda: (torch.randint(-2, 3, (B, h, w, 2), generator=gen) + 0.25 +
                  0.5 * torch.rand(B, h, w, 2, generator=gen)).double()
    ffw, fbw = fl(), fl()
    border = (torch.rand(B, h, w, 1, generator=gen) > 0.2).double()
    fw = torch.ones(B, h, w, 1, dtype=torch.float64)
    bits = sum(1 << k for k, name in enumerate(R.TERMS) if name != 'grad')
    L = R.LevelInputs(im1, im2, ffw, fbw, border, fw, fw, 1, 1, bits)
    return L, border[..., 0], torch.roll(border[..., 0], 1, 2)


def gradcheck_level(monkeypatch, variant=None):
    monkeypatch.setattr(R, "_fp32_frac", lambda f, fl: f - fl)          # the fp32 roundings are steps for
    monkeypatch.setattr(R, "_fp32_sum", lambda g, f: g + f)             # finite differences
    L, mfw, mbw = small_level()
    gl = torch.tensor([0.3, 12.4, 0.5, 0.0, 0.75, 3.0, 0.2, 1.0], dtype=torch.float64)

    class LossFn(torch.autograd.Function):
        """level_losses' value with level_loss_grads as its derivative."""
        @staticmethod
        def forward(ctx, f, b):
            ctx.save_for_backward(f, b)
            return (R.level_losses(L, f, b, mfw, mbw) * gl).sum()

        @staticmethod
        def backward(ctx, g):
            f, b = ctx.saved_tensors
            Lf = R.LevelInputs(L.im1, L.im2, f, b, L.border, L.fwarp_fw, L.fwarp_bw, L.occl, L.R, L.bits)
            gf, gb = R.level_loss_grads(Lf, mfw, mbw, gl, variant)
            return g * gf, g * gb
    f, b = L.ffw.clone().requires_grad_(True), L.fbw.clone().requires_grad_(True)
    return torch.autograd.gradcheck(LossFn.apply, (f, b), raise_exception=False)


@pins("level_loss_grads")
def test_level_loss_grads_against_the_reference_gradients_and_finite_differences(monkeypatch):
    assert grad_pin() <= TAU_LOSS
    assert gradcheck_level(monkeypatch)


def test_negative_control_of_the_level_loss_gradient_pins(monkeypatch):
    assert grad_pin('detach_fb') > 10 * TAU_LOSS
    assert not gradcheck_level(monkeypatch, 'detach_fb')


@pins("A:level_loss_grad_scale", "level_loss_grad_scale", "_dwarp_abs", "_second_order_deltas",
      "_first_order_deltas", "_span")
def test_level_loss_grad_scale_bounds_every_term():
    """Each term alone (the other weights 0) stays under its own scale, and the sum over the terms of |grad| under
    the scale of all of them; sum A / sum |grad| of the golden levels stays within 1.2x of 2760 / 3343 / 2974."""
    for (tag, occl, use_border, r), measured in zip(LEVEL_CASES, (2760, 3343, 2974)):
        L, mfw, mbw = golden_level(tag, occl, use_border, r)
        gl = golden_gl()
        Af, Ab = R.level_loss_grad_scale(L, mfw, mbw, gl)
        sf, sb = torch.zeros_like(Af), torch.zeros_like(Ab)
        for name in ('photo', 'fb', 'smooth_1st', 'smooth_2nd', 'ternary'):
            one = torch.zeros_like(gl)
            one[R.TERMS.index(name)] = gl[R.TERMS.index(name)]
            gf, gb = R.level_loss_grads(L, mfw, mbw, one)
            af, ab = R.level_loss_grad_scale(L, mfw, mbw, one)
            assert bounds(af, gf) and bounds(ab, gb), (tag, name)
            sf, sb = sf + gf.abs(), sb + gb.abs()
        assert bounds(Af, sf) and bounds(Ab, sb), tag
        gf, gb = R.level_loss_grads(L, mfw, mbw, gl)
        t = tight(torch.cat([Af, Ab]), torch.cat([gf, gb]))
        assert t < 1.2 * measured, (tag, t)


@pins("charb_d", "A:charb_d_scale", "charb_d_scale")
def test_charbonnier_derivative_and_its_scale():
    x = torch.linspace(-2, 2, 401, dtype=torch.float64).requires_grad_(True)
    d, = torch.autograd.grad(R.charb(x).sum(), x)
    x = x.detach()
    assert rel(R.charb_d(x), d) <= 1e-13
    assert rel(R.charb_d_scale(x, torch.zeros_like(x)), R.charb_d(x).abs()) <= 1e-15
    # with an operand error e <= 1e-3 |x|-scale, |c'(x + e) - c'(x)| stays within 2^-10 of the scale per unit of e
    e = 1e-3
    assert bool(((R.charb_d(x + e) - R.charb_d(x)).abs() <= R.charb_d_scale(x, torch.full_like(x, e)) * 1.0 + 1e-3).all())
    assert tight(R.charb_d_scale(x, torch.full_like(x, 1e-3)), R.charb_d(x)) < 1.2 * 1.008


# ---- the supervised loss --------------------------------------------------------------------------------------------
def brute_supervised(flow, gt, mask, scale):
    """Loss and dflow by a pixel loop from TF's legacy resize definition: src = dst * (in / out) in fp32, taps
    floor(src) and min(ceil(src), in - 1), weight src - floor(src)."""
    B, h, w, _ = flow.shape
    H, W = gt.shape[1:3]
    fy, fx = np.float32(h) / np.float32(H), np.float32(w) / np.float32(W)
    fl, g, m = flow.numpy(), gt.numpy(), mask.numpy()
    n = B * H * W * 2
    loss, d = 0.0, np.zeros_like(fl)
    for b in range(B):
        for Y in range(H):
            sy = np.float32(Y) * np.float32(fy)
            y0, y1, ly = int(math.floor(sy)), min(int(math.ceil(sy)), h - 1), float(sy - np.float32(math.floor(sy)))
            for X in range(W):
                sx = np.float32(X) * np.float32(fx)
                x0, x1, lx = int(math.floor(sx)), min(int(math.ceil(sx)), w - 1), float(sx - np.float32(math.floor(sx)))
                taps = ((y0, x0, (1 - ly) * (1 - lx)), (y0, x1, (1 - ly) * lx), (y1, x0, ly * (1 - lx)),
                        (y1, x1, ly * lx))
                for c in range(2):
                    v = scale * sum(wt * fl[b, yy, xx, c] for yy, xx, wt in taps)
                    x = v - g[b, Y, X, c]
                    loss += m[b, Y, X, 0] * (x * x + 1e-6) ** 0.45 / n
                    dc = m[b, Y, X, 0] * 0.9 * x * (x * x + 1e-6) ** -0.55 / n
                    for yy, xx, wt in taps:
                        d[b, yy, xx, c] += dc * scale * wt
    return loss, torch.from_numpy(d)


@pins("supervised_loss_grads")
def test_supervised_loss_against_the_oracle_term_and_a_pixel_loop():
    gen = torch.Generator().manual_seed(11)
    flow = torch.randn(2, 3, 5, 2, generator=gen) * 2
    gt = torch.randn(2, 12, 20, 2, generator=gen) * 20
    mask = (torch.rand(2, 12, 20, 1, generator=gen) > 0.3).float()
    loss, dflow, budget = R.supervised_loss_grads(flow, gt, mask)
    f = flow.double().requires_grad_(True)
    want = olosses.charbonnier_loss(tf_compat.resize_bilinear_legacy(f, (12, 20)) * FLOW_SCALE * 4 - gt.double(),
                                    mask.double())
    dwant, = torch.autograd.grad(want, f)
    assert rel(loss, want.detach()) <= TOL_F64 and dev(dflow, dwant) <= TOL_F64
    bl, bd = brute_supervised(flow.double(), gt.double(), mask.double(), 20.0)
    assert rel(loss, torch.tensor(bl)) <= TOL_F64 and dev(dflow, bd) <= TOL_F64
    assert bool((budget >= 0).all()) and float(budget.max()) < 1e-3 * float(dflow.abs().max())


# ---- the tensor-core convolutions ------------------------------------------------------------------------------------
FLOWNET_CONVS = [(3, 8, 7, 2), (8, 12, 5, 2), (12, 16, 3, 2), (16, 16, 3, 1)]       # Cin, Cout, k, stride


def conv_pin(**_):
    """Worst relative deviation of ref_conv from tf_compat's SAME convs and k4 s2 deconvs."""
    gen = torch.Generator().manual_seed(12)
    worst = 0.0
    for Cin, Cout, k, s in FLOWNET_CONVS:
        for H, W in ((11, 14), (12, 9)):
            x = torch.randn(2, Cin, H, W, generator=gen).double()
            w = torch.randn(Cout, Cin, k, k, generator=gen).double()
            pt, _ = tf_compat.same_pad(H, k, s)
            pl, _ = tf_compat.same_pad(W, k, s)
            want = tf_compat.conv2d_same(x, w, None, s)
            wt = w.permute(2, 3, 0, 1).reshape(k * k, Cout, Cin)
            got = ref_conv(x, wt, 0, s, k, k, pt, pl, *want.shape[2:])
            worst = max(worst, dev(got, want))
    for Cin, Cout, h, w_ in ((8, 2, 5, 6), (2, 2, 3, 7), (16, 8, 4, 4)):
        x = torch.randn(2, Cin, h, w_, generator=gen).double()
        w = torch.randn(Cin, Cout, 4, 4, generator=gen).double()
        want = tf_compat.conv2d_transpose_same(x, w, None)
        wt = w.permute(2, 3, 1, 0).reshape(16, Cout, Cin)
        worst = max(worst, dev(ref_conv(x, wt, 1, 2, 4, 4, 1, 1, 2 * h, 2 * w_), want))
    return worst


def loop_conv(x, wt, mode, stride, kh, kw, pad_t, pad_l, Hout, Wout, n, co, oy, ox):
    """One output of ref_conv by its index definition (include/unflow.h)."""
    N, Cin, H, W = x.shape
    acc = 0.0
    for ky in range(kh):
        for kx in range(kw):
            for ci in range(Cin):
                if mode == 0:
                    iy, ix = stride * oy - pad_t + ky, stride * ox - pad_l + kx
                    if 0 <= iy < H and 0 <= ix < W:
                        acc += float(x[n, ci, iy, ix]) * float(wt[ky * kw + kx, co, ci])
                else:
                    for iy in range(H):
                        for ix in range(W):
                            if stride * iy - pad_t + ky == oy and stride * ix - pad_l + kx == ox:
                                acc += float(x[n, ci, iy, ix]) * float(wt[ky * kw + kx, co, ci])
    return acc


@pins("ref_conv", "ref_wgrad", "ref_conv_window", "ref_wgrad_window", "A:ref_conv", "A:ref_wgrad")
def test_tensor_core_references_against_tf_convs_pixel_loops_and_autograd():
    assert conv_pin() <= TOL_F64
    gen = torch.Generator().manual_seed(13)
    for mode, (Cin, Cout, k, s, pt, H, W, Ho, Wo) in ((0, (3, 4, 7, 2, 3, 9, 10, 5, 5)), (0, (4, 5, 3, 1, 1, 6, 7, 6, 7)),
                                                      (1, (4, 3, 4, 2, 1, 4, 5, 8, 10))):
        x = torch.randn(2, Cin, H, W, generator=gen).double()
        wt = torch.randn(k * k, Cout, Cin, generator=gen).double().requires_grad_(True)
        y = ref_conv(x, wt, mode, s, k, k, pt, pt, Ho, Wo)
        for n, co, oy, ox in ((0, 0, 0, 0), (1, Cout - 1, Ho - 1, Wo - 1), (0, 1, Ho // 2, 1), (1, 2, 1, Wo // 2)):
            want = loop_conv(x, wt.detach(), mode, s, k, k, pt, pt, Ho, Wo, n, co, oy, ox)
            assert abs(float(y[n, co, oy, ox]) - want) <= 1e-12 * max(1.0, abs(want)), (mode, n, co, oy, ox)
        P = torch.randn(y.shape, generator=gen).double()
        dw, = torch.autograd.grad((y * P).sum(), wt)
        dw = dw.reshape(k, k, Cout, Cin)
        if mode == 0:
            assert dev(ref_wgrad(P, x, s, k, k, pt, pt), dw.permute(2, 3, 0, 1)) <= TOL_F64
        else:
            assert dev(ref_wgrad(x, P, s, k, k, pt, pt), dw.permute(3, 2, 0, 1)) <= TOL_F64
        wt = wt.detach()
        assert bounds(ref_conv(x.abs(), wt.abs(), mode, s, k, k, pt, pt, Ho, Wo), y)
        assert rel(ref_conv(x.abs(), wt.abs(), mode, s, k, k, pt, pt, Ho, Wo),
                   ref_conv(x.abs(), wt.abs(), mode, s, k, k, pt, pt, Ho, Wo).abs()) == 0
        if mode == 0:
            A = ref_wgrad(P.abs(), x.abs(), s, k, k, pt, pt)
            assert bounds(A, ref_wgrad(P, x, s, k, k, pt, pt)) and rel(A, A.abs()) == 0
    # the window forms: output column ox reads the 8 pixels from stride * ox, i.e. ref_conv with a kh x 8 kernel
    for N, H, Wp, Cp, Cout, kh, s, pt, Ho, Wo in ((2, 9, 20, 4, 6, 7, 2, 3, 5, 7), (1, 6, 12, 8, 3, 3, 1, 1, 6, 5)):
        xp = torch.randn(N, H, Wp, Cp, generator=gen).double()
        wt = torch.randn(kh, Cout, 8 * Cp, generator=gen).double().requires_grad_(True)
        y = ref_conv_window(xp, wt, s, kh, pt, Ho, Wo)
        wt2 = wt.detach().reshape(kh, Cout, 8, Cp).permute(0, 2, 1, 3).reshape(kh * 8, Cout, Cp)
        assert dev(y, ref_conv(xp.permute(0, 3, 1, 2), wt2, 0, s, kh, 8, pt, 0, Ho, Wo)) <= TOL_F64
        P = torch.randn(y.shape, generator=gen).double()
        dw, = torch.autograd.grad((y * P).sum(), wt)
        assert dev(ref_wgrad_window(P, xp, s, kh, pt), dw.permute(1, 2, 0)[..., None]) <= TOL_F64


def test_negative_control_of_the_conv_pin(monkeypatch):
    import test_gpu_tc_step_launches as TC
    real = TC.ref_conv

    def off_by_one(x, wt, mode, stride, kh, kw, pad_t, pad_l, Hout, Wout):       # o = stride*i - pad + k + 1
        return real(x, wt, mode, stride, kh, kw, pad_t - (mode == 1), pad_l - (mode == 1), Hout, Wout)
    monkeypatch.setitem(globals(), "ref_conv", off_by_one)
    assert conv_pin() > 1e3 * TOL_F64


# ---- Adam, TF32, the L2 mask, the leaky-ReLU derivative -----------------------------------------------------------
def tf_adam(p, g, m, v, lr, b1, b2, eps, gs, t, l2m, l2):
    """tf.train.AdamOptimizer's update (its documentation): t <- t + 1, lr_t = lr sqrt(1 - b2^t) / (1 - b1^t),
    m <- b1 m + (1 - b1) g, v <- b2 v + (1 - b2) g^2, p <- p - lr_t m / (sqrt(v) + eps), on the gradient of
    grad_scale * loss + the L2 term of the regularised weights (oracle/unsupervised.regularization_loss), element
    by element in Python floats."""
    preg = (p * l2m).clone().requires_grad_(True)
    dl2, = torch.autograd.grad(regularization_loss({'w/weights': preg}, scale=l2), preg)
    lr_t = lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t)
    out = ([], [], [])
    for i in range(p.numel()):
        gi = gs * float(g[i]) + float(dl2[i])
        mi = b1 * float(m[i]) + (1 - b1) * gi
        vi = b2 * float(v[i]) + (1 - b2) * gi * gi
        out[0].append(float(p[i]) - lr_t * mi / (math.sqrt(vi) + eps))
        out[1].append(mi)
        out[2].append(vi)
    return tuple(torch.tensor(o, dtype=torch.float64) for o in out)


def adam_pin(fn):
    gen = torch.Generator().manual_seed(14)
    n = 64
    p = torch.randn(n, generator=gen).double() * 0.05
    g = torch.randn(n, generator=gen).double() * 1e-3
    m = torch.randn(n, generator=gen).double() * 1e-4
    v = torch.rand(n, generator=gen).double() * 1e-6
    l2m = (torch.rand(n, generator=gen) > 0.5).double()
    lr, b1, b2, eps, gs, l2 = (float(np.float32(x)) for x in (1e-4, 0.9, 0.999, 1e-8, 0.5, 4e-4))
    worst = 0.0
    for t in (1, 2, 1000):
        (p1, m1, v1), (Ap, Am, Av) = fn(p, g, m, v, lr, b1, b2, eps, gs, float(t), l2m, l2)
        wp, wm, wv = tf_adam(p, g, m, v, lr, b1, b2, eps, gs, t, l2m, l2)
        worst = max(worst, dev(p1, wp, float(Ap.max())), dev(m1, wm, float(Am.max())), dev(v1, wv, float(Av.max())))
        assert bounds(Ap, p1) and bounds(Am, m1) and bounds(Av, v1)
    return worst


@pins("adam_reference", "A:adam_reference")
def test_adam_reference_against_tf_adam():
    assert adam_pin(adam_reference) <= TOL_F64
    gen = torch.Generator().manual_seed(15)
    p, g, m, v = (torch.rand(32, generator=gen).double() * s for s in (0.05, 1e-3, 1e-4, 1e-6))
    (p1, m1, v1), (Ap, Am, Av) = adam_reference(p, g, m, v, 1e-4, 0.9, 0.999, 1e-8, 0.5, 3.0, torch.ones(32), 4e-4)
    assert rel(Am, m1) <= 1e-15 and rel(Av, v1) <= 1e-15              # non-negative operands: A == |ref|
    assert tight(Ap, p1) < 1.01


def test_negative_control_of_the_adam_pin():
    def eps_in_sqrt(p, g, m, v, lr, b1, b2, eps, gs, t, l2m, l2):
        (p1, m1, v1), A = adam_reference(p, g, m, v, lr, b1, b2, eps, gs, t, l2m, l2)
        lr_t = lr * (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
        return (p - lr_t * m1 / (v1 + eps).sqrt(), m1, v1), A
    assert adam_pin(eps_in_sqrt) > 1e3 * TOL_F64


def tf32_bits(u):
    """TF32 rounding by its bit definition: keep sign, exponent and the top 10 mantissa bits; round the 13 dropped
    bits to nearest, a tie (exactly 0x1000) away from zero; a carry may run into the exponent (up to inf).  Inf
    stays inf; a NaN stays a NaN."""
    u = int(u) & 0xFFFFFFFF
    if (u >> 23) & 0xFF == 0xFF:
        return u if u & 0x7FFFFF == 0 else None                 # None: any NaN
    dropped, kept = u & 0x1FFF, u & ~0x1FFF & 0xFFFFFFFF
    if dropped > 0x1000 or dropped == 0x1000:
        kept += 0x2000
    return kept


def tf32_cases():
    edge = [0x3F801000, 0x3F803000, 0x3F800FFF, 0x3F801001, 0xBF801000, 0x3F7FF000, 0x3F7FEFFF, 0x00000000,
            0x80000000, 0x00000001, 0x00001000, 0x00000FFF, 0x007FF000, 0x807FF000, 0x00400000, 0x7F7FFFFF,
            0x7F7FEFFF, 0xFF7FF000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x7FFFFFFF, 0xFFFFFFFF, 0x7F800001]
    rnd = np.random.default_rng(2).integers(0, 2 ** 32, 4096, dtype=np.uint64).tolist()
    return np.array(edge + rnd, dtype=np.uint64).astype(np.uint32)


def tf32_pin(fn):
    """Number of inputs whose fn(x) differs from the bit definition (NaN for NaN counts as equal)."""
    u = tf32_cases()
    got = fn(torch.from_numpy(u.view(np.int32).copy()).view(torch.float32)).view(torch.int32).numpy().view(np.uint32)
    bad = 0
    for a, b in zip(u.tolist(), got.tolist()):
        want = tf32_bits(a)
        bad += (((b >> 23) & 0xFF != 0xFF or b & 0x7FFFFF == 0) if want is None else b != want)
    return bad


@pins("tf32_rna")
def test_tf32_rna_against_the_bit_definition():
    assert tf32_pin(tf32_rna) == 0


def test_negative_control_of_the_tf32_pin():
    assert tf32_pin(lambda w: (w.view(torch.int32) & ~0x1FFF).view(torch.float32)) > 1000


@pins("l2_bits")
def test_l2_bits_against_the_trainer_mask():
    from unflow_b200.e2eflow.core.train import l2_mask_bytes
    n = 48
    isw, packed = l2_mask_bytes(n, [0, 5, 7, 20, 33], [5, 2, 13, 13, 15], [True, False, True, True, False])
    assert 0 < int(isw.sum()) < n
    assert torch.equal(l2_bits(packed, n), isw.double())


@pins("_lrelu_d")
def test_leaky_relu_derivative():
    pre = torch.linspace(-2, 2, 41, dtype=torch.float64).requires_grad_(True)
    act = F.leaky_relu(pre, 0.1)
    d, = torch.autograd.grad(act.sum(), pre)
    assert torch.equal(_lrelu_d(act.detach(), 0.1), d)


@pins("worst_ratio", "errors")
def test_the_ratio_helpers():
    ref = torch.tensor([1.0, 2.0, 0.0, 0.0], dtype=torch.float64)
    A = torch.tensor([1.0, 4.0, 0.0, 0.0], dtype=torch.float64)
    assert R.worst_ratio(torch.tensor([1.5, 2.0, 0.0, 0.0]), ref, A) == 0.5
    assert R.worst_ratio(torch.tensor([1.0, 2.0, 0.0, 1e-30]), ref, A) > 1e200
    assert R.errors(torch.tensor([1.0, 2.5]), torch.tensor([1.0, 2.0], dtype=torch.float64)) == (0.5 / 5 ** 0.5, 0.25)


# ---- every reference has a pin ----------------------------------------------------------------------------------------
def test_every_reference_and_error_scale_is_pinned():
    import inspect
    names = {n for n, v in vars(R).items() if (inspect.isfunction(v) or inspect.isclass(v))
             and v.__module__ == R.__name__ and not n.startswith("_")}
    helpers = {"ref_conv", "ref_wgrad", "ref_conv_window", "ref_wgrad_window", "adam_reference", "tf32_rna",
               "l2_bits", "_lrelu_d"}
    import test_gpu_tc_step_launches as TC
    assert {n for n in vars(TC) if n.startswith("ref_")} <= helpers
    want = (names - set(NOT_REFERENCES)) | helpers | set(A_SCALES)
    missing = sorted(want - PINNED)
    assert not missing, "references without a pin: %s" % missing
    assert set(NOT_REFERENCES) <= names
