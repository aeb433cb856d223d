"""Every non-tensor-core launch of one FlowNetC training step, checked against float64 at the step's own shapes.

Two eager steps as bench.py runs them (batch 4 at 384x1280, 3xTF32, default options), one plain and one with
the training-time augmentation (the BORDER_STN sampler, an affine-warped border mask that takes any value in
[0, 1]).  The library handle is replaced by a proxy for the step: every call of an entry point goes through a
checker that views the call's device pointers as tensors (shapes and strides from its integer arguments),
snapshots what the call overwrites, runs it, synchronises and compares the result elementwise with a float64
evaluation of include/unflow.h on the same operands: |got - ref| <= TAU * A, A = the same evaluation on
absolute values (tests/float64_refs.py).  The tensor-core entry points pass through (their shadow check is
tests/test_gpu_tc_step_launches.py), host-only queries are recorded, and an entry point the step calls without
a checker fails the test (tests/native_entry_points.py classifies them all; the sets each step calls are pinned).

The level loss: the masks are discrete, so they are not recomputed in float64.  The checker re-issues the call
into scratch buffers with masks_out set, asserts its 8 losses are bitwise equal to the step's (determinism) and
its masks bit-equal to an op-by-op float32 evaluation of oracle/losses.py's mask formulas, then evaluates every
continuous quantity in float64 with those masks held fixed.  The gradient reference is float64 autograd of
that forward with grad_losses as the upstream vector; its A is tests/float64_refs.level_loss_grad_scale.

Error models and TAU (one value per kernel family, 3x the worst ratio measured on an H100 SXM 80 GB at a 400 W
power limit over both steps and tests/test_gpu_float64_kernels.py):
  TAU_SUM  fp32 sums of products (correlation, downsample, narrow 3x3 conv, bias gradients, warps, forward warp):
           a few units of 2^-24 per accumulation level.  Worst 1.26e-6 (the step's downsample / correlation
           launches; 1.08e-6 in the forward-warp gradient), TAU 4e-6.
  TAU_LOSS the level loss: __log2f / exp2f / rsqrtf / __fdividef (~2^-22 each) and the atomic order of the
           backward scatter.  Losses at most 3.7e-7 of their value; gradients worst 2.0e-5 (census term of a
           9x70 level, R = 3), 1.9e-5 in the augmented step; TAU 6e-5.
  TAU_ADAM the Adam update: powf / sqrtf / division in fp32.  Worst 6.7e-7 (2.8e-7 in the step), TAU 2e-6.
Copies (relayout, weight split) are bit-exact; correlation_fold_grad is one fp32 rounding (2^-24 * A, measured
exactly 2^-24).  The plain step makes 114 checked launches, the augmented one 119; the file takes about 12 s of
GPU time (the two float64 steps 3 s each, the rest model set-up).
"""
import time

import pytest
import torch
import torch.nn.functional as F

import float64_refs as R
import native_entry_points as EP
from test_gpu_tc_step_launches import ref_conv, ref_wgrad

pytestmark = pytest.mark.gpu

TAU_SUM = 4e-6
TAU_LOSS = 6e-5
TAU_ADAM = 2e-6
TAU_FOLD = 2.0 ** -24


def _round4(c):
    return (c + 3) // 4 * 4


def tf32_rna(w):
    """fp32 -> the nearest TF32 value (10 mantissa bits, ties away from zero: cvt.rna.tf32.f32), as fp32.  A NaN
    stays a NaN (the carry out of a large payload would wrap it to a signed zero)."""
    b = w.view(torch.int32)
    return torch.where(torch.isnan(w), w, ((b + 0x1000) & ~0x1FFF).view(torch.float32))


# ---- checkers: check(args, call) runs the real call via call() and returns a list of (label, shape, ratio, tau) ----
def _corr_args(a):
    B, C, H, W, ks, md, pad, s1, s2 = a
    return (B, C, H, W), (ks, md, pad, s1, s2)


def check_corr_fwd_bidir(a, call):
    (B, C, H, W), attrs = _corr_args(a[4:13])
    ngr, D, oh, ow = R.corr_geometry(H, W, *attrs)
    call()
    in0, in1 = R.view(a[0], (B, C, H, W)).double(), R.view(a[1], (B, C, H, W)).double()
    out, rev = R.view(a[2], (B, D * D, oh, ow)), R.view(a[3], (B, D * D, oh, ow))
    shape = "%dx%dx%dx%d d%d" % (B, C, H, W, attrs[1])
    r = []
    for name, got, x, y in (("out", out, in0, in1), ("out_rev", rev, in1, in0)):
        r.append((name, shape, R.worst_ratio(got, R.correlation(x, y, *attrs), R.correlation(x.abs(), y.abs(), *attrs)),
                  TAU_SUM))
    return r


def check_corr_fold(a, call):
    (B, C, H, W), attrs = _corr_args(a[3:12])
    ngr, D, oh, ow = R.corr_geometry(H, W, *attrs)
    g = R.view(a[0], (B, D * D, oh, ow)).double()
    grev = R.view(a[1], (B, D * D, oh, ow)).double()
    call()
    got = R.view(a[2], (B, D * D, oh, ow))
    folded = R.fold_reverse(grev, attrs[4], ngr)
    return [("gout_eff", "%dx%dx%dx%d" % (B, D * D, oh, ow), R.worst_ratio(got, g + folded, g.abs() + folded.abs()),
             TAU_FOLD)]


def check_corr_bwd(a, call):
    (B, C, H, W), attrs = _corr_args(a[5:14])
    ngr, D, oh, ow = R.corr_geometry(H, W, *attrs)
    gout = R.view(a[0], (B, D * D, oh, ow)).double()
    in0, in1 = R.view(a[1], (B, C, H, W)).double(), R.view(a[2], (B, C, H, W)).double()
    call()
    g0, g1, A0, A1 = R.correlation_grads(gout, in0, in1, attrs)
    shape = "%dx%dx%dx%d d%d" % (B, C, H, W, attrs[1])
    return [("g0", shape, R.worst_ratio(R.view(a[3], (B, C, H, W)), g0, A0), TAU_SUM),
            ("g1", shape, R.worst_ratio(R.view(a[4], (B, C, H, W)), g1, A1), TAU_SUM)]


def check_p2i(a, call):
    src_p, src_batch, dst_p, dst_batch, pitch, B, C, P, acc = a[:9]
    src = R.view(src_p, (B, C, P), (src_batch, P, 1)).clone()
    dst = R.view(dst_p, (B, P, C), (dst_batch, pitch, 1))
    span = R.view(dst_p, (B, P - 1, pitch), (dst_batch, pitch, 1)) if P > 1 else None
    old = dst.clone()
    old_span = span.clone() if span is not None else None
    call()
    want = old + src.permute(0, 2, 1) if acc else src.permute(0, 2, 1)
    ok = torch.equal(dst, want)
    if span is not None:
        slack = torch.ones(pitch, dtype=torch.bool, device="cuda")
        slack[:C] = False
        # bit patterns: the pitch padding of a fresh buffer is uninitialised and may hold NaNs
        bits = lambda t: t.view(torch.int32)[..., slack]
        ok = ok and torch.equal(bits(span), bits(old_span))
    return [("acc" if acc else "copy", "%dx%dx%d p%d" % (B, C, P, pitch), 0.0 if ok else float("inf"), 0.0)]


def check_i2p(a, call):
    src_p, src_batch, pitch, dst_p, dst_batch, B, C, P = a[:8]
    call()
    src = R.view(src_p, (B, P, C), (src_batch, pitch, 1))
    dst = R.view(dst_p, (B, C, P), (dst_batch, P, 1))
    return [("copy", "%dx%dx%d p%d" % (B, C, P, pitch), 0.0 if torch.equal(dst, src.permute(0, 2, 1)) else
             float("inf"), 0.0)]


def check_downsample(a, call):
    img_p, out_p, B, H, W, C, s = a[:7]
    call()
    x = R.view(img_p, (B, H, W, C)).double()
    got = R.view(out_p, (B, H // s, W // s, C))
    return [("out", "%dx%dx%dx%d /%d" % (B, H, W, C, s), R.worst_ratio(got, R.downsample(x, s),
                                                                      R.downsample(x.abs(), s)), TAU_SUM)]


def check_backward_warp_fwd(a, call):
    img_p, flow_p, out_p, B, H, W, C, mode = a[:8]
    call()
    img = R.view(img_p, (B, H, W, C)).double()
    flow = R.view(flow_p, (B, H, W, 2)).double()
    got = R.view(out_p, (B, H, W, C))
    return [("mode%d" % mode, "%dx%dx%dx%d" % (B, H, W, C),
             R.worst_ratio(got, R.warp(img, flow, mode), R.warp_abs(img, flow, mode)), TAU_SUM)]


def check_narrow_fwd(a, call):
    x_p, xp, w_p, b_p, y_p, yp, N, H, W, C, Co = a[:11]
    call()
    x = R.view(x_p, (N, H, W, C), (H * W * xp, W * xp, xp, 1)).double().permute(0, 3, 1, 2)
    w = R.view(w_p, (Co, 3, 3, C)).double()
    wt = w.permute(1, 2, 0, 3).reshape(9, Co, C)
    ref = ref_conv(x, wt, 0, 1, 3, 3, 1, 1, H, W)
    A = ref_conv(x.abs(), wt.abs(), 0, 1, 3, 3, 1, 1, H, W)
    if b_p:
        b = R.view(b_p, (Co,)).double().view(1, Co, 1, 1)
        ref, A = ref + b, A + b.abs()
    got = R.view(y_p, (N, H, W, Co), (H * W * yp, W * yp, yp, 1)).permute(0, 3, 1, 2)
    return [("y", "%dx%dx%dx%d" % (N, C, H, W), R.worst_ratio(got, ref, A), TAU_SUM)]


def check_narrow_wgrad(a, call):
    x_p, xp, g_p, sN, sC, sH, sW, gw_p, ws_p, N, H, W, C, Co = a[:14]
    call()
    x = R.view(x_p, (N, H, W, C), (H * W * xp, W * xp, xp, 1)).double().permute(0, 3, 1, 2)
    g = R.view(g_p, (N, Co, H, W), (sN, sC, sH, sW)).double()
    ref = ref_wgrad(g, x, 1, 3, 3, 1, 1).permute(0, 2, 3, 1)          # [Co, 3, 3, C]
    A = ref_wgrad(g.abs(), x.abs(), 1, 3, 3, 1, 1).permute(0, 2, 3, 1)
    return [("gw", "%dx%dx%dx%d" % (N, C, H, W), R.worst_ratio(R.view(gw_p, (Co, 3, 3, C)), ref, A), TAU_SUM)]


def _lrelu_d(act, slope):
    return torch.where(act > 0, torch.ones_like(act), torch.full_like(act, slope))


def check_bias_lrelu(a, call):
    y_p, b_p, pixels, C, slope = a[:5]
    y = R.view(y_p, (pixels, C))
    old = y.double()
    call()
    b = R.view(b_p, (C,)).double()
    pre = old + b
    return [("y", "%dx%d" % (pixels, C), R.worst_ratio(y, F.leaky_relu(pre, slope), old.abs() + b.abs()), TAU_SUM)]


def check_bias_grad_lrelu(a, call):
    g_p, sN, sC, sH, sW, act_p, gb_p, N, C, H, W, slope = a[:12]
    call()
    g = R.view(g_p, (N, C, H, W), (sN, sC, sH, sW)).double()
    d = _lrelu_d(R.view(act_p, (N, H, W, C)).double().permute(0, 3, 1, 2), slope) if act_p else 1.0
    ref, A = (g * d).sum((0, 2, 3)), (g.abs() * d).sum((0, 2, 3))
    return [("gb", "%dx%dx%dx%d" % (N, C, H, W), R.worst_ratio(R.view(gb_p, (C,)), ref, A), TAU_SUM)]


def check_lrelu_bwd_bias(a, call):
    g_p, sN, sC, sH, sW, act_p, ap, gpre_p, gp, gb_p, N, C, H, W, slope = a[:15]
    call()
    g = R.view(g_p, (N, C, H, W), (sN, sC, sH, sW)).double()
    d = _lrelu_d(R.view(act_p, (N, H, W, C), (H * W * ap, W * ap, ap, 1)).double().permute(0, 3, 1, 2),
                 slope) if act_p else 1.0
    shape = "%dx%dx%dx%d" % (N, C, H, W)
    out = [("gb", shape, R.worst_ratio(R.view(gb_p, (C,)), (g * d).sum((0, 2, 3)), (g.abs() * d).sum((0, 2, 3))),
            TAU_SUM)]
    if gpre_p:
        gpre = R.view(gpre_p, (N, H, W, C), (H * W * gp, W * gp, gp, 1)).permute(0, 3, 1, 2)
        out.append(("gpre", shape, R.worst_ratio(gpre, g * d, (g * d).abs()), TAU_SUM))
    return out


def check_wsplit(a, call):
    w_p, hi_p, lo_p, taps, Rr, C, s_t, s_r, s_c = a[:9]
    call()
    w = R.view(w_p, (taps, Rr, C), (s_t, s_r, s_c))
    Cp = _round4(C)
    hi, lo = R.view(hi_p, (taps, Rr, Cp)), R.view(lo_p, (taps, Rr, Cp))
    ok = (torch.equal(hi[..., :C], tf32_rna(w.contiguous())) and torch.equal(hi[..., :C] + lo[..., :C], w)
          and torch.equal(lo[..., :C], w - hi[..., :C]) and not bool(hi[..., C:].any()) and not bool(lo[..., C:].any()))
    return [("hi/lo", "%dx%dx%d" % (taps, Rr, C), 0.0 if ok else float("inf"), 0.0)]


def adam_reference(p, g, m, v, lr, b1, b2, eps, gs, t, l2m, l2):
    """The TF Adam rule in float64 (include/unflow.h): -> (p', m', v') and their A."""
    lr_t = lr * (1 - b2 ** t) ** 0.5 / (1 - b1 ** t)
    gr = g * gs + l2m * l2 * p
    gr_a = (g * gs).abs() + l2m * l2 * p.abs()
    m1 = b1 * m + (1 - b1) * gr
    v1 = b2 * v + (1 - b2) * gr * gr
    step = lr_t * m1 / (v1.sqrt() + eps)
    Am = b1 * m.abs() + (1 - b1) * gr_a
    Av = b2 * v.abs() + (1 - b2) * gr_a * gr_a
    Ap = p.abs() + lr_t * Am / (v1.sqrt() + eps)
    return (p - step, m1, v1), (Ap, Am, Av)


def l2_bits(mask, n):
    """The adam kernel's L2 mask (uint8 [n / 4], bit k of byte i = element 4 * i + k) as float64 flags [n]."""
    mk = mask.long()
    return torch.stack([(mk >> k) & 1 for k in range(4)], 1).reshape(n).double()


def check_adam_l2(a, call):
    p_p, g_p, m_p, v_p, n, lr, b1, b2, eps, step, gs, zero_grad, mask_p, l2 = a[:14]
    bufs = [R.view(x, (n,)) for x in (p_p, g_p, m_p, v_p)]
    p, g, m, v = (b.double() for b in bufs)
    call()
    f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))        # the ABI passes fp32 hyper-parameters
    l2m = l2_bits(R.view(mask_p, (n // 4,), dtype=torch.uint8), n) if mask_p else torch.zeros_like(p)
    (p1, m1, v1), (Ap, Am, Av) = adam_reference(p, g, m, v, f32(lr), f32(b1), f32(b2), f32(eps), f32(gs),
                                                 float(step), l2m, f32(l2))
    shape = "n=%d step %d" % (n, step)
    ok = not zero_grad or not bool(bufs[1].any())
    return [("param", shape, R.worst_ratio(bufs[0], p1, Ap), TAU_ADAM),
            ("m", shape, R.worst_ratio(bufs[2], m1, Am), TAU_ADAM),
            ("v", shape, R.worst_ratio(bufs[3], v1, Av), TAU_ADAM),
            ("grads zeroed", shape, 0.0 if ok else float("inf"), 0.0)]


# ---- the level loss ----------------------------------------------------------------------------------------------
def _level_views(a, bwd):
    if bwd:
        gl_p, im1, im2, ffw, fbw, border, fwf, fwb, saved, dfw, dbw, B, h, w, occl, Rr, bits = a[:17]
    else:
        im1, im2, ffw, fbw, border, fwf, fwb, losses, saved, masks, ws, B, h, w, occl, Rr, bits = a[:17]
    v = lambda p, c: R.view(p, (B, h, w, c)) if p else None
    return dict(im1=v(im1, 3), im2=v(im2, 3), ffw=v(ffw, 2), fbw=v(fbw, 2), border=v(border, 1),
                fwarp_fw=v(fwf, 1), fwarp_bw=v(fwb, 1), B=B, h=h, w=w, occl=occl, R=Rr, bits=bits)


def reissue_level_fwd(lib, d, want_saved):
    """The same level_loss_fwd call into scratch buffers, with masks_out -> (losses, masks [2,B,h,w], saved)."""
    B, h, w = d["B"], d["h"], d["w"]
    losses = torch.empty(8, device="cuda")
    masks = torch.empty(2, B, h, w, device="cuda")
    saved = torch.empty(4 * B * h * w, device="cuda") if want_saved else None
    ws = torch.empty(int(lib.unflow_level_loss_workspace_bytes(B, h, w)), device="cuda", dtype=torch.uint8)
    p = lambda t: t.data_ptr() if t is not None else None
    rc = lib.unflow_level_loss_fwd(p(d["im1"]), p(d["im2"]), p(d["ffw"]), p(d["fbw"]), p(d["border"]),
                                   p(d["fwarp_fw"]), p(d["fwarp_bw"]), losses.data_ptr(), p(saved), masks.data_ptr(),
                                   ws.data_ptr(), B, h, w, d["occl"], d["R"], d["bits"],
                                   torch.cuda.current_stream().cuda_stream)
    assert rc == 0
    torch.cuda.synchronize()
    return losses, masks, saved


def level_inputs(d):
    return R.LevelInputs(d["im1"], d["im2"], d["ffw"], d["fbw"], d["border"], d["fwarp_fw"], d["fwarp_bw"],
                         d["occl"], d["R"], d["bits"])


def fixed_masks(lib, d):
    """The kernel's masks, asserted bit-equal to the float32 oracle formulas, as float64 [B,h,w] each."""
    _, masks, _ = reissue_level_fwd(lib, d, False)
    want = R.masks_f32(d["ffw"], d["fbw"], d["border"], d["occl"], d["fwarp_fw"], d["fwarp_bw"])
    for k in range(2):
        assert torch.equal(masks[k], want[k]), "level_loss mask %d differs from the float32 oracle formulas" % k
    return masks[0].double(), masks[1].double()


def level_loss_fwd_ratios(lib, d, got_losses):
    """[(term, ratio)] of one level_loss_fwd result against float64 (A = the term's value: sums of
    non-negative elements); asserts the re-issued call is bitwise equal."""
    again, _, _ = reissue_level_fwd(lib, d, False)
    assert torch.equal(again, got_losses), "level_loss_fwd is not bitwise repeatable"
    mfw, mbw = fixed_masks(lib, d)
    L = level_inputs(d)
    ref = R.level_losses(L, L.ffw, L.fbw, mfw, mbw)
    out = []
    for k, name in enumerate(R.TERMS):
        if L.want(name):
            out.append((name, R.worst_ratio(got_losses[k:k + 1], ref[k:k + 1], ref[k:k + 1].abs())))
        else:
            assert float(got_losses[k]) == 0.0, name
    return out


def level_loss_bwd_ratios(lib, d, gl, dfw, dbw, variant=None):
    """(ratio dflow_fw, ratio dflow_bw) of one level_loss_bwd result against float64 autograd."""
    mfw, mbw = fixed_masks(lib, d)
    L = level_inputs(d)
    gf, gb = R.level_loss_grads(L, mfw, mbw, gl, variant)
    Af, Ab = R.level_loss_grad_scale(L, mfw, mbw, gl)
    return R.worst_ratio(dfw, gf, Af), R.worst_ratio(dbw, gb, Ab)


def _lib():
    """The library itself, also while the step's proxy stands in for it (re-issued calls are not checked)."""
    from unflow_b200 import _native
    lib = _native.lib()
    return lib._real if isinstance(lib, LibProxy) else lib


def check_level_fwd(a, call):
    d = _level_views(a, False)
    call()
    losses = R.view(a[7], (8,)).clone()
    shape = "%dx%dx%d r%d occl%d" % (d["B"], d["h"], d["w"], d["R"], d["occl"])
    return [(name, shape, r, TAU_LOSS) for name, r in level_loss_fwd_ratios(_lib(), d, losses)]


def check_level_bwd(a, call):
    d = _level_views(a, True)
    B, h, w = d["B"], d["h"], d["w"]
    gl = R.view(a[0], (8,)).clone()
    saved_in = R.view(a[8], (4 * B * h * w,)).clone() if a[8] else None
    call()
    if saved_in is not None:
        _, _, saved = reissue_level_fwd(_lib(), d, True)
        assert torch.equal(saved, saved_in), "the saved planes differ from a re-issued forward"
    dfw, dbw = R.view(a[9], (B, h, w, 2)), R.view(a[10], (B, h, w, 2))
    rf, rb = level_loss_bwd_ratios(_lib(), d, gl, dfw, dbw)
    shape = "%dx%dx%d r%d occl%d" % (B, h, w, d["R"], d["occl"])
    return [("dflow_fw", shape, rf, TAU_LOSS), ("dflow_bw", shape, rb, TAU_LOSS)]


CHECKERS = {
    "unflow_correlation_fwd_bidir": check_corr_fwd_bidir,
    "unflow_correlation_fold_grad": check_corr_fold,
    "unflow_correlation_bwd": check_corr_bwd,
    "unflow_planar_to_interleaved": check_p2i,
    "unflow_interleaved_to_planar": check_i2p,
    "unflow_downsample": check_downsample,
    "unflow_level_loss_fwd": check_level_fwd,
    "unflow_level_loss_bwd": check_level_bwd,
    "unflow_conv3x3_narrow_fwd": check_narrow_fwd,
    "unflow_conv3x3_narrow_wgrad": check_narrow_wgrad,
    "unflow_lrelu_bwd_bias": check_lrelu_bwd_bias,
    "unflow_bias_grad_lrelu": check_bias_grad_lrelu,
    "unflow_bias_lrelu": check_bias_lrelu,
    "unflow_tc_wsplit": check_wsplit,
    "unflow_adam_step_l2": check_adam_l2,
    "unflow_backward_warp_fwd": check_backward_warp_fwd,
}


class LibProxy:
    """Stands in for the ctypes library handle: each entry point goes through its checker in `checkers`."""

    def __init__(self, real, checkers=CHECKERS):
        self._real = real
        self.checkers = checkers
        self.rows = []            # (launch #, entry point, label, shape, ratio, tau)
        self.calls = set()
        self.unchecked = []
        self.launches = 0

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if not name.startswith("unflow_"):
            return fn

        def wrapped(*args):
            self.calls.add(name)
            if name in EP.HOST_ONLY or name in EP.TC_DELEGATED:
                return fn(*args)
            chk = self.checkers.get(name)
            if chk is None:
                self.unchecked.append(name)
                return fn(*args)
            rc = []
            i = self.launches
            self.launches += 1
            results = chk(args, lambda: (rc.append(fn(*args)), torch.cuda.synchronize()))
            assert rc and rc[0] == 0, "%s returned %s" % (name, rc)
            for label, shape, ratio, tau in results:
                self.rows.append((i, name[len("unflow_"):], label, shape, ratio, tau))
            return rc[0]
        return wrapped

    def table(self):
        lines = ["%4s %-24s %-22s %-26s %-11s %s" % ("#", "entry point", "output", "shape", "|err|/A", "TAU")]
        for i, name, label, shape, ratio, tau in self.rows:
            lines.append("%4d %-24s %-22s %-26s %.3e   %.1e" % (i, name, label, shape, ratio, tau))
        return "\n".join(lines)

    def worst_by_family(self):
        out = {}
        for _, name, label, _, ratio, tau in self.rows:
            out[tau] = max(out.get(tau, 0.0), ratio)
        return out


def count_input_copies(monkeypatch, conv_ops):
    """Wraps conv_ops._tc_input; the returned list gets the shape of every input the tensor-core layers copy."""
    real, copies = conv_ops._tc_input, []

    def counted(x, *args):
        xt, pads = real(x, *args)
        if xt is not x:
            copies.append(tuple(x.shape))
        return xt, pads
    monkeypatch.setattr(conv_ops, "_tc_input", counted)
    return copies


def run_checked_step(monkeypatch, augment):
    from unflow_b200 import _native
    from unflow_b200 import synthetic as synth
    from unflow_b200.e2eflow.core import conv_ops
    from unflow_b200.e2eflow.core.train import Trainer

    dev = torch.device("cuda", 0)
    prev = conv_ops.get_mode()
    conv_ops.set_mode("3xtf32")
    try:
        trainer = Trainer(dict(synth.KITTI_PARAMS, flownet="C"), synth.KITTI_NORMALIZATION, dev, seed=1234,
                          augment=augment)
        im1, im2, _ = synth.image_pair(4, 384, 1280, seed=1234)
        im1, im2 = im1.to(dev), im2.to(dev)
        torch.manual_seed(7)
        proxy = LibProxy(_native.lib())
        copies = count_input_copies(monkeypatch, conv_ops)
        monkeypatch.setattr(_native, "_lib", proxy)
        try:
            loss = trainer.step(im1, im2)
            torch.cuda.synchronize()
        finally:
            monkeypatch.setattr(_native, "_lib", proxy._real)
    finally:
        conv_ops.set_mode(prev)
    return proxy, copies, float(loss)


@pytest.mark.parametrize("augment", [False, True], ids=["plain", "augment"])
def test_every_other_launch_of_a_training_step(monkeypatch, augment):
    t0 = time.time()
    proxy, copies, loss = run_checked_step(monkeypatch, augment)
    print("\n" + proxy.table())
    worst = max(proxy.rows, key=lambda r: r[4] / r[5] if r[5] else (0 if r[4] == 0 else float("inf")))
    print("%d checked launches, worst |err|/A by TAU: %s, worst row %s, loss %.6f, %.1f s" % (
        proxy.launches, {"%.0e" % k: "%.3e" % v for k, v in proxy.worst_by_family().items()}, worst[:4], loss,
        time.time() - t0))
    print("entry points called: %s" % sorted(proxy.calls))
    assert not proxy.unchecked, "entry points without a checker: %s" % sorted(set(proxy.unchecked))
    assert not copies, "inputs copied for the tensor-core layers: %s" % copies
    bad = [r for r in proxy.rows if not r[4] <= r[5]]
    assert not bad, "over TAU: %s" % bad
    pinned = EP.AUGMENT_STEP_CALLS if augment else EP.PLAIN_STEP_CALLS
    assert proxy.calls == pinned, "entry points called changed: +%s -%s" % (
        sorted(proxy.calls - pinned), sorted(pinned - proxy.calls))
    if augment:
        assert any(r[1] == "backward_warp_fwd" and r[2] == "mode2" for r in proxy.rows)
