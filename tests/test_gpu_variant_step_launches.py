"""Every launch of the other training steps the project runs, checked against float64 at the step's own shapes.

tests/test_gpu_step_launches.py and tests/test_gpu_tc_step_launches.py check one configuration, the eager FlowNetC
step at batch 4 and 384x1280.  The configurations below take paths that step never reaches: the first layer of a
FlowNetS (6 channels, a 64-wide row window) and of a stacked S network (14 channels: im1, im2, flow, warp, diff; a
128-wide window), the space-to-depth first layer of a train_all stack whose input requires a gradient (56 channels,
4x4 filter, stride 1, with its input gradient), the image_warp gradient into the previous network's flow
(unflow_backward_warp_bwd), the supervised loss, the single-direction correlation of the supervised FlowNetC,
frozen networks and Adam over the last network only, the level loss without occlusion and fb terms, 5-row top
levels (320-high images), a 48x64 cost volume, and the small networks (channel_mult 3/8).

Each configuration runs one eager Trainer.step in 3xTF32 mode with the default options, with both shadow checks
installed: the Recorder of test_gpu_tc_step_launches.py on tc_conv (bound TAU) and the LibProxy of
test_gpu_step_launches.py on the library handle, here with VARIANT_CHECKERS (TAU_SUM, TAU_LOSS, TAU_ADAM as there).
The added checkers: the correlation forward and the warp gradient (dflow, and dimage when it is asked for) against
tests/float64_refs.py with TAU_SUM; the supervised loss against float64_refs.supervised_loss_grads with the bound of
tests/test_gpu_supervised.py (the loss within 1e-5 of its value, dflow within the float32 error budget the
reference returns: |err| / budget <= 1).  An entry point without a checker, a row over its bound, a missing path
or a change of the entry points a configuration calls (native_entry_points.VARIANT_STEP_CALLS) fails the test.

Measured on an H100 SXM 80 GB (HBM3) at a 700 W power limit: checked launches (library + tensor-core) and the worst
|err| / A per family (TAU: tensor core 1e-5, sum 4e-6, level loss 6e-5, Adam 2e-6; the supervised dflow in units of
its budget).  Copies (relayout, weight split) are bit-exact in every configuration.

  config              launches    tensor core   sum       level loss   Adam      other
  C-chairs            114 + 61    2.4e-6        1.2e-6    5.1e-6       2.8e-7    fold 6.0e-8
  C-kitti1152         114 + 61    3.2e-6        1.2e-6    1.3e-5       2.7e-7    fold 6.0e-8
  S-synthia           104 + 58    3.1e-6        3.8e-7    1.1e-5       2.6e-7
  cs-cityscapes       133 + 77    3.9e-6        8.8e-7    4.3e-6       2.7e-7
  CSS-bench           158 + 95    4.7e-6        1.2e-6    7.9e-6       2.3e-7
  CSS-ft-train_all    248 + 187   5.0e-6        1.2e-6    -            3.1e-7    supervised loss 2.2e-7, dflow 0.30

The float atomics of a step make later operands differ slightly from run to run; over three runs the worst were
1.4e-5 (level loss, C-kitti1152), 5.2e-6 (tensor core) and 0.45 (supervised dflow).  The space-to-depth layer
end to end: y 5.3e-7, dL/dx 8.3e-7, dL/dw 2.6e-8 of A.  The file takes about 25 s of GPU time (1 to 6 s per
configuration).
"""
import time

import pytest
import torch
import torch.nn.functional as F

import float64_refs as R
import native_entry_points as EP
from test_gpu_step_launches import (CHECKERS, TAU_ADAM, TAU_FOLD, TAU_LOSS, TAU_SUM, LibProxy, _corr_args,
                                    count_input_copies)
from test_gpu_tc_step_launches import TAU, Recorder

pytestmark = pytest.mark.gpu

TAU_SUPERVISED_LOSS = 1e-5      # |loss - ref| <= 1e-5 * ref, as tests/test_gpu_supervised.py
TAU_SUPERVISED_GRAD = 1.0       # |dflow - ref| <= the float32 error budget of supervised_loss_grads


# ---- checkers of the entry points the FlowNetC step does not call ---------------------------------------------------
def check_corr_fwd(a, call):
    (B, C, H, W), attrs = _corr_args(a[3:12])
    ngr, D, oh, ow = R.corr_geometry(H, W, *attrs)
    call()
    in0, in1 = R.view(a[0], (B, C, H, W)).double(), R.view(a[1], (B, C, H, W)).double()
    got = R.view(a[2], (B, D * D, oh, ow))
    return [("out", "%dx%dx%dx%d d%d" % (B, C, H, W, attrs[1]),
             R.worst_ratio(got, R.correlation(in0, in1, *attrs), R.correlation(in0.abs(), in1.abs(), *attrs)), TAU_SUM)]


def check_backward_warp_bwd(a, call, skip_tap=None):
    grad_p, img_p, flow_p, dflow_p, dimg_p, B, H, W, C, mode = a[:10]
    old = R.view(dimg_p, (B, H, W, C)).double() if dimg_p else None      # the image gradient accumulates
    call()
    grad = R.view(grad_p, (B, H, W, C)).double()
    img, flow = R.view(img_p, (B, H, W, C)).double(), R.view(flow_p, (B, H, W, 2)).double()
    di, df, Ai, Af = R.warp_grads(grad, img, flow, mode, skip_tap)
    shape = "%dx%dx%dx%d mode%d" % (B, H, W, C, mode)
    out = [("dflow", shape, R.worst_ratio(R.view(dflow_p, (B, H, W, 2)), df, Af), TAU_SUM)]
    if dimg_p:
        out.append(("dimage", shape, R.worst_ratio(R.view(dimg_p, (B, H, W, C)), old + di, old.abs() + Ai), TAU_SUM))
    return out


def _supervised_views(flow_p, gt_p, mask_p, B, h, w, H, W):
    return (R.view(flow_p, (B, h, w, 2)), R.view(gt_p, (B, H, W, 2)),
            R.view(mask_p, (B, H, W, 1)) if mask_p else None)


def check_supervised_fwd(a, call, ignore_mask=False):
    flow_p, gt_p, mask_p, loss_p, ws_p, B, h, w, H, W, scale = a[:11]
    call()
    flow, gt, mask = _supervised_views(flow_p, gt_p, mask_p, B, h, w, H, W)
    want, _, _ = R.supervised_loss_grads(flow, gt, None if ignore_mask else mask, scale)
    return [("loss", "%dx%dx%d -> %dx%d" % (B, h, w, H, W),
             R.worst_ratio(R.view(loss_p, (1,)), want.view(1), want.abs().view(1)), TAU_SUPERVISED_LOSS)]


def check_supervised_bwd(a, call, ignore_mask=False):
    gl_p, flow_p, gt_p, mask_p, dflow_p, B, h, w, H, W, scale = a[:11]
    call()
    flow, gt, mask = _supervised_views(flow_p, gt_p, mask_p, B, h, w, H, W)
    gl = float(R.view(gl_p, (1,)))
    _, dflow, budget = R.supervised_loss_grads(flow, gt, None if ignore_mask else mask, scale)
    return [("dflow / budget", "%dx%dx%d -> %dx%d" % (B, h, w, H, W),
             R.worst_ratio(R.view(dflow_p, (B, h, w, 2)), gl * dflow, abs(gl) * budget + 1e-30), TAU_SUPERVISED_GRAD)]


VARIANT_CHECKERS = {
    **CHECKERS,
    "unflow_correlation_fwd": check_corr_fwd,
    "unflow_backward_warp_bwd": check_backward_warp_bwd,
    "unflow_supervised_loss_fwd": check_supervised_fwd,
    "unflow_supervised_loss_bwd": check_supervised_bwd,
}


# ---- the configurations -------------------------------------------------------------------------------------------
# config_template/config.ini [train] + [train_chairs]: [train]'s loss (no occlusion mask, no fb term)
CHAIRS_PARAMS = dict(flownet='C', pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0,
                     learning_rate=1.0e-4)
# [train] + [train_kitti]
KITTI_PARAMS = dict(flownet='C', pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0,
                    fb_weight=0.2, mask_occlusion='fb', occ_weight=12.4, learning_rate=1.0e-5)
# [train] + [train_synthia]: [train]'s loss, as chairs
SYNTHIA_PARAMS = dict(flownet='S', pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0,
                      learning_rate=1.0e-4)
# [train] + [train_cityscapes]: the KITTI loss (fb, occlusion weight 12.4), here with the small cs stack
CITYSCAPES_PARAMS = dict(flownet='cs', pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0,
                         fb_weight=0.2, mask_occlusion='fb', occ_weight=12.4, learning_rate=1.0e-5)
# [train] + [train_kitti] with flownet = CSS: what bench.py --spec CSS trains
CSS_BENCH_PARAMS = dict(flownet='CSS', pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0,
                        fb_weight=0.2, mask_occlusion='fb', occ_weight=12.4, learning_rate=1.0e-5)
# [train] + [train_kitti_ft] with flownet = CSS and train_all = True: the supervised fine-tune of a whole stack
KITTI_FT_PARAMS = dict(flownet='CSS', train_all=True, pyramid_loss=True, border_mask=True, ternary_weight=1.0,
                       smooth_2nd_weight=3.0, manual_decay_iters=[45000, 20000, 20000, 10000, 2500, 2500],
                       manual_decay_lrs=[0.5e-5, 0.25e-5, 0.1e-5, 0.05e-5, 0.25e-6, 0.1e-6])

# id -> (loss parameters, supervised, B, H, W)
CONFIGS = {
    "C-chairs": (CHAIRS_PARAMS, False, 4, 384, 512),
    "C-kitti1152": (KITTI_PARAMS, False, 4, 320, 1152),
    "S-synthia": (SYNTHIA_PARAMS, False, 4, 512, 768),
    "cs-cityscapes": (CITYSCAPES_PARAMS, False, 2, 512, 1024),
    "CSS-bench": (CSS_BENCH_PARAMS, False, 2, 384, 1280),
    "CSS-ft-train_all": (KITTI_FT_PARAMS, True, 4, 320, 768),
}


def run_checked_step(monkeypatch, params, supervised, B, H, W):
    from unflow_b200 import _native
    from unflow_b200 import synthetic as synth
    from unflow_b200.e2eflow.core import conv_ops, tc_conv
    from unflow_b200.e2eflow.core.train import Trainer

    dev = torch.device("cuda", 0)
    prev = conv_ops.get_mode()
    conv_ops.set_mode("3xtf32")
    rec = Recorder(tc_conv, conv_ops)
    try:
        trainer = Trainer(dict(params), synth.KITTI_NORMALIZATION, dev, seed=1234, supervised=supervised)
        batch = synth.supervised_batch(B, H, W, seed=1234) if supervised else synth.image_pair(B, H, W, seed=1234)[:2]
        batch = [t.to(dev) for t in batch]
        torch.manual_seed(7)
        proxy = LibProxy(_native.lib(), VARIANT_CHECKERS)
        rec.install(monkeypatch)
        copies = count_input_copies(monkeypatch, conv_ops)
        monkeypatch.setattr(_native, "_lib", proxy)
        try:
            loss = trainer.step(*batch)
            torch.cuda.synchronize()
        finally:
            monkeypatch.setattr(_native, "_lib", proxy._real)
    finally:
        conv_ops.set_mode(prev)
    return proxy, rec, copies, trainer, float(loss)


def worst_by_family(proxy, rec):
    names = {TAU_SUM: "sum", TAU_LOSS: "level loss", TAU_ADAM: "adam", TAU_FOLD: "fold", 0.0: "exact"}
    out = {"tensor core": max(r["ratio"] for r in rec.rows)}
    for _, name, label, _, ratio, tau in proxy.rows:
        fam = ("supervised " + label) if name.startswith("supervised") else names[tau]
        out[fam] = max(out.get(fam, 0.0), ratio)
    return out


def _contraction(r):
    """The contraction width of a row-window launch (8 * the channel pitch of the window)."""
    return int(r["ch"].split("->")[0]) if r["kind"] == "window fwd" else int(r["ch"].split("x")[1])


def path_misses(cid, proxy, rec, trainer):
    """The paths configuration `cid` must take and did not (descriptions); empty when it took them all."""
    spec, train_all = trainer.params["flownet"], bool(trainer.params.get("train_all"))
    win = lambda kind, k: [r for r in rec.rows if r["kind"] == kind and _contraction(r) == k]
    lib = lambda name, label=None: [r for r in proxy.rows if r[1] == name and (label is None or r[2] == label)]
    need = []
    if spec[0] in "Ss":
        need.append(("6-channel FlowNetS window fwd (64)", bool(win("window fwd", 64))))
    if len(spec) > 1 and not train_all:
        need.append(("14-channel stacked window fwd (128), one per S network",
                     len(win("window fwd", 128)) == len(spec) - 1))
    if cid == "CSS-bench":
        wg = [r for r in rec.rows if r["kind"] == "window wgrad"]
        need.append(("one window wgrad (128), of the trained net only",
                     len(wg) == 1 and _contraction(wg[0]) == 128))
    if train_all and len(spec) > 1:
        s2d = lambda kind, ch: [r for r in rec.rows if r["kind"] == kind and r["k"] == 4 and r["ch"] == ch]
        need += [("no stacked window fwd (the input requires grad)", not win("window fwd", 128)),
                 ("space-to-depth conv1 (56->64, k4 s1)", len(s2d("conv s1", "56->64")) == len(spec) - 1),
                 ("its input gradient (transposed s1, 64->56)", len(s2d("transposed s1", "64->56")) == len(spec) - 1),
                 ("its weight gradient (64x56)", len(s2d("conv wgrad", "64x56")) == len(spec) - 1),
                 ("backward_warp_bwd with a flow gradient", bool(lib("backward_warp_bwd", "dflow")))]
    if trainer.supervised:
        need += [("supervised_loss_fwd", bool(lib("supervised_loss_fwd"))),
                 ("supervised_loss_bwd", bool(lib("supervised_loss_bwd")))]
    if cid == "C-chairs":
        need.append(("correlation at 48x64",
                     any("x48x64 " in r[3] for r in proxy.rows if r[1].startswith("correlation_fwd"))))
        level = lib("level_loss_fwd")
        need.append(("level loss with occl0, no fb / occ term",
                     bool(level) and all("occl0" in r[3] for r in level) and not {r[2] for r in level} & {"fb", "occ"}))
    if cid in ("C-kitti1152", "CSS-ft-train_all"):
        need.append(("a tc_conv launch on a 5-row level", any(r["nhw"][1] == 5 for r in rec.rows)))
    adam = lib("adam_step_l2", "param")
    need.append(("one Adam launch", len(adam) == 1))
    if len(spec) > 1 and not train_all:
        last = sum(p.numel() for sc in trainer.variables.scopes_of_net(len(spec) - 1)
                   for p in trainer.variables.weights(sc))
        n = int(adam[0][3].split()[0][2:]) if adam else -1
        need.append(("Adam over the last network's %d elements" % last,
                     trainer.num_params == last and n == (last + 3) // 4 * 4))
    return [d for d, ok in need if not ok]


@pytest.mark.parametrize("cid", list(CONFIGS))
def test_every_launch_of_a_variant_step(monkeypatch, cid):
    t0 = time.time()
    proxy, rec, copies, trainer, loss = run_checked_step(monkeypatch, *CONFIGS[cid])
    print("\n" + proxy.table())
    print(rec.table())
    print("%s: %d + %d checked launches, worst |err|/A by family: %s, loss %.6f, %.1f s" % (
        cid, proxy.launches, len(rec.rows), {k: "%.3e" % v for k, v in worst_by_family(proxy, rec).items()}, loss,
        time.time() - t0))
    print("entry points called: %s" % sorted(proxy.calls))
    assert not proxy.unchecked, "entry points without a checker: %s" % sorted(set(proxy.unchecked))
    assert not copies, "inputs copied for the tensor-core layers: %s" % copies
    bad = [r for r in proxy.rows if not r[4] <= r[5]]
    assert not bad, "over TAU: %s" % bad
    bad_tc = [i for i, r in enumerate(rec.rows) if not r["ratio"] <= TAU]
    assert not bad_tc, "tensor-core launches over TAU = %g: %s" % (TAU, bad_tc)
    missing = path_misses(cid, proxy, rec, trainer)
    assert not missing, "%s did not take: %s" % (cid, missing)
    pinned = EP.VARIANT_STEP_CALLS[cid]
    assert proxy.calls == pinned, "entry points called changed: +%s -%s" % (
        sorted(proxy.calls - pinned), sorted(pinned - proxy.calls))


def test_bench_css_runs_these_parameters():
    from unflow_b200 import synthetic as synth
    assert CSS_BENCH_PARAMS == dict(synth.KITTI_PARAMS, learning_rate=1.0e-5, flownet="CSS")


# ---- the space-to-depth first layer end to end -----------------------------------------------------------------
def _s2d_wrong_side(real, x, w, pads):
    """space_to_depth_operands (`real`) with the filter's zero row and column on the wrong side (before the first
    tap instead of after the last)."""
    xs, _ = real(x, w, pads)
    Co, C, k, _ = w.shape
    m = (k + 1) // 2
    ws = F.pad(w, (1, 0, 1, 0)).reshape(Co, C, m, 2, m, 2).permute(0, 3, 5, 1, 2, 4).reshape(Co, 4 * C, m, m)
    return xs, ws


def _conv_vjp(x, w, g, pads):
    """(y, dx, dw) of the 7x7 stride-2 layer in float64: y = conv2d(pad(x), w), dx, dw = its vjp with g."""
    x, w = x.detach().requires_grad_(True), w.detach().requires_grad_(True)
    with torch.enable_grad():
        y = F.conv2d(F.pad(x, (pads[2], pads[3], pads[0], pads[1])), w, stride=2)
        dx, dw = torch.autograd.grad(y, (x, w), g)
    return y.detach(), dx, dw


def s2d_layer_ratios(monkeypatch, N, H, W, operands=None):
    """conv_ops.conv2d on FlowNetS conv1 of a stacked network (14 channels, 7x7, stride 2, SAME, bias, leaky ReLU)
    with an input that requires grad, against float64: worst |err| / A of y, dL/dx and dL/dw.  `operands`
    replaces space_to_depth_operands (a wrong regrouping, for the negative control)."""
    from unflow_b200.e2eflow.core import conv_ops
    C, Co, k, pads = 14, 64, 7, (2, 3, 2, 3)
    g = torch.Generator(device="cuda").manual_seed(N + H)
    x = (torch.rand(N, H, W, C, device="cuda", generator=g) * 2 - 0.8).permute(0, 3, 1, 2).requires_grad_(True)
    w = (torch.randn(Co, k, k, C, device="cuda", generator=g) * 0.05).permute(0, 3, 1, 2).requires_grad_(True)
    b = (torch.randn(Co, device="cuda", generator=g) * 0.1).requires_grad_(True)
    real = conv_ops.space_to_depth_operands
    used = []
    monkeypatch.setattr(conv_ops, "space_to_depth_operands",
                        lambda *a: (used.append(1), operands(real, *a) if operands else real(*a))[1])
    prev = conv_ops.get_mode()
    conv_ops.set_mode("3xtf32")
    try:
        conv_ops.new_forward_generation()          # as every network forward pass does: no stale gradient slots
        y = conv_ops.conv2d(x, w, b, 2, pads, act=True)
        gy = torch.randn(y.shape, device="cuda", generator=g)
        y.backward(gy)
        torch.cuda.synchronize()
    finally:
        conv_ops.set_mode(prev)
        monkeypatch.setattr(conv_ops, "space_to_depth_operands", real)
    assert used, "the layer did not take the space-to-depth path"
    xd, wd, bd = x.detach().double(), w.detach().double(), b.detach().double().view(1, -1, 1, 1)
    # the backward differentiates the leaky ReLU at the kernel's own output, so the reference does too
    gpre = gy.double() * torch.where(y.detach() > 0, 1.0, 0.1).double()
    pre, dx, dw = _conv_vjp(xd, wd, gpre, pads)
    Ay, Ax, Aw = _conv_vjp(xd.abs(), wd.abs(), gpre.abs(), pads)
    return (R.worst_ratio(y.detach(), F.leaky_relu(pre + bd, 0.1), Ay + bd.abs()),
            R.worst_ratio(x.grad, dx, Ax), R.worst_ratio(w.grad, dw, Aw))


def test_space_to_depth_layer_end_to_end(monkeypatch):
    """The Recorder checks the kernel on the operands after the transform; this checks the transform too, at the
    shape the stacked S networks of a batch-4 step see (both directions: 8 x 14 x 320 x 768)."""
    ry, rx, rw = s2d_layer_ratios(monkeypatch, 8, 320, 768)
    print("\ny %.3e  dL/dx %.3e  dL/dw %.3e" % (ry, rx, rw))
    assert max(ry, rx, rw) <= TAU


# ---- negative controls --------------------------------------------------------------------------------------------
def test_space_to_depth_bound_catches_a_misplaced_zero_row(monkeypatch):
    """The end-to-end check of the space-to-depth layer with the filter's zero-extended row and column before its
    first tap.  Measured: correct y 4.7e-7, dL/dx 6.6e-7, dL/dw 2.7e-7; misplaced y 0.30, dL/dx 0.66, dL/dw 0.22
    (over 2e4 x TAU)."""
    good = s2d_layer_ratios(monkeypatch, 2, 64, 96)
    bad = s2d_layer_ratios(monkeypatch, 2, 64, 96, operands=_s2d_wrong_side)
    print("\ncorrect y %.3e dx %.3e dw %.3e, zero row misplaced y %.3e dx %.3e dw %.3e" % (good + bad))
    assert max(good) <= TAU
    assert min(bad) > 1000 * TAU


def test_warp_gradient_bound_catches_a_dropped_tap():
    """check_backward_warp_bwd against a reference whose gather leaves out the (y1, x1) tap.  Measured: correct
    dflow 1.3e-7, dimage 2.1e-7; tap dropped dflow 0.95, dimage 0.50 (over 1e5 x TAU_SUM)."""
    from unflow_b200 import _native
    B, H, W, C = 2, 96, 320, 3
    g = torch.Generator(device="cuda").manual_seed(9)
    img = torch.rand(B, H, W, C, device="cuda", generator=g)
    flow = (torch.rand(B, H, W, 2, device="cuda", generator=g) * 2 - 1) * 6
    grad = torch.randn(B, H, W, C, device="cuda", generator=g)
    dflow, dimg = torch.empty_like(flow), torch.zeros_like(img)
    args = (grad.data_ptr(), img.data_ptr(), flow.data_ptr(), dflow.data_ptr(), dimg.data_ptr(), B, H, W, C,
            _native.BORDER_CLAMP, torch.cuda.current_stream().cuda_stream)

    def call():
        assert _native.lib().unflow_backward_warp_bwd(*args) == 0
        torch.cuda.synchronize()
    good = [r[2] for r in check_backward_warp_bwd(args, call)]
    bad = [r[2] for r in check_backward_warp_bwd(args, call, skip_tap=3)]
    print("\ncorrect dflow %.3e dimage %.3e, tap dropped dflow %.3e dimage %.3e" % tuple(good + bad))
    assert max(good) <= TAU_SUM
    assert min(bad) > 1000 * TAU_SUM


def test_supervised_bound_catches_an_ignored_mask():
    """The supervised checkers against a reference that ignores mask_gt, at the fine-tune's shape (flow2 of a
    batch-4 step at 320x768, 40 % of the pixels valid).  Measured in units of the bound: correct loss 0.011,
    dflow 0.022; mask ignored loss 6.0e4, dflow 3.8e3."""
    from unflow_b200 import _native
    B, h, w, H, W = 4, 80, 192, 320, 768
    g = torch.Generator(device="cuda").manual_seed(11)
    flow = torch.randn(B, h, w, 2, device="cuda", generator=g) * 0.5
    gt = torch.randn(B, H, W, 2, device="cuda", generator=g) * 8.0
    mask = (torch.rand(B, H, W, 1, device="cuda", generator=g) < 0.4).float()
    lib = _native.lib()
    loss, gl, dflow = torch.empty(1, device="cuda"), torch.ones(1, device="cuda"), torch.empty_like(flow)
    ws = torch.empty(int(lib.unflow_supervised_loss_workspace_bytes(B, H, W)), device="cuda", dtype=torch.uint8)
    st = torch.cuda.current_stream().cuda_stream
    fwd = (flow.data_ptr(), gt.data_ptr(), mask.data_ptr(), loss.data_ptr(), ws.data_ptr(), B, h, w, H, W, 20.0, st)
    bwd = (gl.data_ptr(), flow.data_ptr(), gt.data_ptr(), mask.data_ptr(), dflow.data_ptr(), B, h, w, H, W, 20.0, st)

    def caller(fn, args):
        def call():
            assert fn(*args) == 0
            torch.cuda.synchronize()
        return call
    ratios = []
    for ignore in (False, True):
        for chk, fn, args in ((check_supervised_fwd, lib.unflow_supervised_loss_fwd, fwd),
                              (check_supervised_bwd, lib.unflow_supervised_loss_bwd, bwd)):
            (_, _, ratio, tau), = chk(args, caller(fn, args), ignore_mask=ignore)
            ratios.append(ratio / tau)
    print("\ncorrect loss %.3e dflow %.3e, mask ignored loss %.3e dflow %.3e (in units of their bound)" % tuple(ratios))
    assert max(ratios[:2]) <= 1
    assert min(ratios[2:]) > 1000
