"""The assembled networks against a float64 network: every flow and every variable gradient, end to end.

The per-launch checks (test_gpu_*step_launches.py) evaluate each library call on the operands that call received, so
they cannot see a call that gets the wrong operands or a gradient that never reaches its destination: the gradient
slots of conv_ops (a later consumer adds into the buffer the first one registered), the concat buffers whose members
are born in their slice and get views of one gradient back, the fold of the reverse cost volume, the Siamese 2B
batch, frozen and train_all stacks, the space-to-depth conv1 and the weight gradients accumulated straight into the
Trainer's flat buffer.  Here the product runs in 3xTF32 and the oracle's own restatement of the graph
(oracle/flownet.py, oracle/supervised.py) runs in float64 on the GPU on the same inputs and variables, with
float64_refs.correlation and float64_refs.warp (its bilinear fraction rounded to fp32, as the kernel and the
reference op take it) in place of the CPU float32 ops.

Objectives: the linear functional L = sum over networks, directions and levels of <G, flow> with fixed random G
scaled by 1 / sqrt(numel), so that every level contributes comparably (no masks, no loss kernels: the network's own
forward and vector-Jacobian product), and the supervised loss (augment=False, regularisation included) of the
supervised configurations.  Gradients go into the Trainer's flat buffer (read back from there, as Adam reads them),
except in one case that starts from ``.grad = None``; one case runs two forward / backward passes on different
inputs and must equal the sum of the two float64 gradients (no gradient slot outlives its forward pass).  Variables
get small random biases so the bias paths carry signal.

Every flow and every variable gradient (weights and biases separately) is scored by its relative L2 error
||got - ref|| / ||ref|| and its max error max|got - ref| / max|ref|; the bound is on the larger of the two.  Variables
of frozen networks must get no gradient, as in the reference.

The float64 network takes each leaky ReLU's side of the kink from the product's own activations
(float64_refs.follow_kink_sides).  Where fp32 and float64 disagree on the sign of a pre-activation within rounding
of zero, the slopes differ (1 vs 0.1), and on the coarse levels (5x18 pixels at 320x1152) one such element is a
sizeable share of a weight gradient: with the float64 network's own signs the gradients differed by up to 2.6e-2
(max) / 3.3e-3 (rel L2), in fp32 mode as well (9.6e-3 / 2.2e-3), which would have hidden the reverse-volume control
below.

Measured on an H100 SXM 80 GB (HBM3) at a 700 W power limit (worst rel L2 / max over the tensors):

  case                          flows               weight gradients    bias gradients
  C-kitti                       8.1e-6 / 1.0e-5     1.4e-5 / 1.4e-5     7.3e-6 / 6.0e-6
  C-kitti, fp32 mode (cuDNN)    2.5e-6 / 4.6e-6     4.3e-6 / 9.6e-6     3.5e-6 / 4.1e-6
  S-synthia (.grad = None)      1.5e-5 / 1.6e-5     1.9e-5 / 1.8e-5     7.8e-6 / 7.0e-6
  cs-cityscapes (two passes)    1.6e-5 / 1.7e-5     1.9e-5 / 2.0e-5     1.2e-5 / 1.2e-5
  CSS-bench                     2.7e-5 / 3.0e-5     2.8e-5 / 2.7e-5     9.8e-6 / 1.0e-5
  CSS-ft-train_all supervised   -                   7.0e-4 / 5.7e-4     4.3e-4 / 4.2e-4
  CSS-ft-train_all functional   2.5e-5 / 2.8e-5     3.6e-3 / 3.0e-3     5.9e-3 / 6.4e-3
  s-full_res functional         1.3e-5 / 1.5e-5     1.6e-5 / 1.9e-5     7.5e-6 / 9.6e-6
  s-full_res supervised         -                   2.0e-4 / 2.7e-4     2.8e-4 / 2.7e-4
  eval C (4 sizes)              3.3e-6 / 5.4e-6
  eval CSS (4 sizes)            1.6e-5 / 1.9e-5

3xTF32 stays within about 3x of the exact-fp32 mode on the same case.  Two families sit above the rest, both explained
by where the gradient is evaluated rather than by the arithmetic: the supervised loss is evaluated at each network's
own flow, so the 1e-5 forward difference enters its gradient through the Charbonnier curvature (the linear
functional, whose cotangent does not depend on the flow, stays at 1.6e-5 on the same s-full_res network); and a
train_all stack differentiates image_warp and |warp - im1| of the previous network's flow, whose floor() and sign
flip where the two flows straddle an integer or a zero.  Bounds, 3x the worst measured: TAU_FLOW 9e-5, TAU_GRAD
8.4e-4, TAU_GRAD_WARP 1.9e-2 (the train_all stacks only).

Negative controls on C-kitti (test_bound_catches_a_wiring_error), worst gradient error / its rel L2:
  a later consumer overwrites the gradient slot instead of adding    1.09 (1300x TAU_GRAD) / 1.04
  the reverse cost volume's gradient is not folded                   4.7e-2 (56x TAU_GRAD) / 3.9e-2
  flow6 hands conv6_1 no input gradient                              0.86 (1000x TAU_GRAD) / 0.86
All three are above the 5e-3 / 1e-2 relative L2 bounds of the float32-oracle tests too, but those run other cases
at a loose bound; the reverse-volume one is within 4x of them.  The file takes about 40 s of GPU time.
"""
import time

import pytest
import torch

import float64_refs as R
from oracle import flownet as oflownet
from oracle import supervised as osup
from oracle import tf_compat as tfc

pytestmark = pytest.mark.gpu

TAU_FLOW = 9e-5         # 3x the worst measured (see the docstring)
TAU_GRAD = 8.4e-4
TAU_GRAD_WARP = 1.9e-2  # train_all stacks: gradients that cross image_warp's floor and |warp - im1|

# the loss parameters of the configurations (tests/test_gpu_variant_step_launches.py); the functional objective
# reads only flownet / train_all / full_res from them
_FT = dict(pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0)

# id -> (spec, train_all, full_res, bidirectional, B, H, W, objective, gradient storage, passes)
CASES = {
    "C-kitti": ("C", False, False, True, 2, 320, 1152, "functional", "flat", 1),
    "S-synthia": ("S", False, False, True, 2, 512, 768, "functional", "none", 1),
    "cs-cityscapes": ("cs", False, False, True, 2, 512, 1024, "functional", "flat", 2),
    "CSS-bench": ("CSS", False, False, True, 2, 384, 1280, "functional", "flat", 1),
    "CSS-ft-train_all-supervised": ("CSS", True, False, False, 2, 320, 768, "supervised", "flat", 1),
    "CSS-ft-train_all-functional": ("CSS", True, False, False, 2, 320, 768, "functional", "flat", 1),
    "s-full_res-functional": ("s", False, True, True, 2, 128, 256, "functional", "flat", 1),
    "s-full_res-supervised": ("s", False, True, False, 2, 128, 256, "supervised", "flat", 1),
}

EVAL_SIZES = [(384, 1280), (384, 512), (512, 1024), (512, 640)]


def _norm():
    from unflow_b200 import synthetic as synth
    return synth.KITTI_NORMALIZATION


def _variables(spec, full_res, seed):
    """The oracle's initial variables with small random biases (TF layout, float32 CPU)."""
    tfv = oflownet.init_variables(spec, full_res, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in tfv:
        if k.endswith('/biases'):
            tfv[k] = torch.randn(tfv[k].shape, generator=g) * 0.02
    return tfv


def _float64_ops(monkeypatch):
    monkeypatch.setattr(oflownet, "correlation", lambda a, b: R.correlation(a, b, 1, 20, 20, 1, 2))
    monkeypatch.setattr(oflownet, "image_warp", lambda img, flow: R.warp(img, flow, 1))


def _net_images(B, H, W, seed):
    """Mean-subtracted network inputs, float32 on the GPU (the product's; the oracle gets them in float64)."""
    from unflow_b200 import synthetic as synth
    im1, im2, _ = synth.image_pair(B, H, W, seed=seed)
    mean = torch.tensor([m / 255.0 for m in _norm()[0]], dtype=torch.float32)
    return (im1 / 255.0 - mean).cuda(), (im2 / 255.0 - mean).cuda()


def _flow_list(out, bidir):
    """[(name, flow)] over networks, directions and levels."""
    fw, bw = out if bidir else (out, [])
    names = []
    for d, stack in (("fw", fw), ("bw", bw)):
        for i, net in enumerate(stack):
            for lvl, f in enumerate(net):
                names.append(("net%d %s %dx%d" % (i, d, f.shape[1], f.shape[2]), f))
    return names


def _weights_G(flows, seed):
    """The functional's G, one per flow: float32 values, so that both networks see the same G."""
    dev = flows[0][1].device
    g = torch.Generator(device=dev).manual_seed(seed)
    return [torch.randn(f.shape, device=dev, dtype=torch.float32, generator=g) / f.numel() ** 0.5
            for _, f in flows]


def _functional(flows, G):
    return sum((Gi.to(f.dtype) * f).sum() for (_, f), Gi in zip(flows, G) if f.requires_grad)


def _trainable(spec, train_all, names):
    if train_all or len(spec) == 1:
        return set(names)
    root = 'stack_%d_flownet/' % (len(spec) - 1)
    return {n for n in names if n.startswith(root)}


def run_product(case, tfv, inputs, mode="3xtf32"):
    """The product on ``inputs`` (one tuple per pass): (flows of every pass, {name: gradient}, frozen names with
    a gradient).  Gradients are read from the Trainer's flat buffer (plus the L2 term the Adam kernel adds)."""
    from unflow_b200.e2eflow.core import conv_ops
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables, flownet
    from unflow_b200.e2eflow.core.supervised import supervised_loss
    from unflow_b200.e2eflow.core.train import Trainer
    spec, train_all, full_res, bidir, B, H, W, objective, storage, passes = case
    params = dict(_FT, flownet=spec, train_all=train_all, full_res=full_res)
    v = FlowNetVariables(spec, full_res, seed=0).load_tf_dict(tfv)
    prev = conv_ops.get_mode()
    conv_ops.set_mode(mode)
    try:
        tr = Trainer(params, _norm(), torch.device("cuda", 0), variables=v, supervised=objective == "supervised")
        if storage == "none":
            for p in tr.trainable:
                p.grad = None
            v.l2_in_optimizer = False
        all_flows = []
        for k, batch in enumerate(inputs):
            if objective == "functional":
                out = flownet(batch[0], batch[1], spec, full_res, train_all=train_all, backward_flow=bidir,
                              variables=v)
                flows = _flow_list(out, bidir)
                loss = _functional(flows, _weights_G(flows, 100 + k))
            else:
                loss = supervised_loss(batch, params, _norm(), augment=False, variables=v)
                flows = None
            loss.backward()
            torch.cuda.synchronize()
            all_flows.append([(n, f.detach()) for n, f in flows] if flows else [])
    finally:
        conv_ops.set_mode(prev)
    grads = {}
    if storage == "none":
        for name, p in zip(tr.trainable_names, tr.trainable):
            grads[name] = p.grad
    else:
        flat = tr.flat_grad + (tr.l2_gradient() if objective == "supervised" else 0)
        for name, p, off in zip(tr.trainable_names, tr.trainable, tr._offsets):
            grads[name] = tr._view_like(flat[off:off + p.numel()], p)
    frozen = [n for n in v.variable_names() if n not in grads and _param(v, n).grad is not None]
    return all_flows, grads, frozen


def _param(v, name):
    scope, kind = name.rsplit('/', 1)
    w, b = v.weights(scope)
    return w if kind == 'weights' else b


def run_oracle(monkeypatch, case, tfv, inputs):
    """The oracle in float64 on the GPU: (flows of every pass, {name: summed gradient in the product's layout})."""
    spec, train_all, full_res, bidir, B, H, W, objective, storage, passes = case
    _float64_ops(monkeypatch)
    names = list(tfv)
    train = _trainable(spec, train_all, names)
    leaves = {k: t.double().cuda().requires_grad_(k in train) for k, t in tfv.items()}
    params = dict(_FT, flownet=spec, train_all=train_all, full_res=full_res)
    all_flows = []
    for k, batch in enumerate(inputs):
        b64 = [t.double() for t in batch]
        if objective == "functional":
            out = oflownet.flownet(leaves, b64[0], b64[1], spec, full_resolution=full_res, train_all=train_all,
                                   backward_flow=bidir)
            flows = _flow_list(out, bidir)
            loss = _functional(flows, _weights_G(flows, 100 + k))
        else:
            loss = osup.supervised_loss(leaves, b64, params, normalization=_norm())
            flows = None
        loss.backward()
        all_flows.append([(n, f.detach()) for n, f in flows] if flows else [])
    grads = {}
    for k in train:
        g = leaves[k].grad
        grads[k] = g.permute(3, 2, 0, 1) if k.endswith('/weights') else g
    return all_flows, grads


def compare(got_flows, ref_flows, got_grads, ref_grads):
    """{'flow' | 'weights' | 'biases': [(score, rel L2, max, name)]}; a missing gradient scores infinity."""
    rows = {"flow": [], "weights": [], "biases": []}
    for k, (gf, rf) in enumerate(zip(got_flows, ref_flows)):
        assert [n for n, _ in gf] == [n for n, _ in rf]
        for (n, g), (_, r) in zip(gf, rf):
            l2, mx = R.errors(g, r)
            rows["flow"].append((max(l2, mx), l2, mx, "pass%d %s" % (k, n)))
    assert set(got_grads) == set(ref_grads), (sorted(set(got_grads) ^ set(ref_grads)))
    for name, r in ref_grads.items():
        g = got_grads[name]
        fam = "weights" if name.endswith('/weights') else "biases"
        if g is None:
            rows[fam].append((float("inf"), float("inf"), float("inf"), name))
            continue
        l2, mx = R.errors(g, r)
        rows[fam].append((max(l2, mx), l2, mx, name))
    return rows


def table(cid, rows, seconds):
    lines = ["%s (%.1f s)" % (cid, seconds),
             "  %-8s %5s  %-10s %-10s worst" % ("family", "n", "rel L2", "max")]
    for fam, rs in rows.items():
        if not rs:
            continue
        w = max(rs)
        lines.append("  %-8s %5d  %-10.3e %-10.3e %s" % (fam, len(rs), max(r[1] for r in rs),
                                                         max(r[2] for r in rs), w[3]))
    return "\n".join(lines)


def worst(rows):
    """(worst flow score, worst gradient score, worst gradient rel L2)."""
    f = max((r[0] for r in rows["flow"]), default=0.0)
    g = [r for fam in ("weights", "biases") for r in rows[fam]]
    return f, max(r[0] for r in g), max(r[1] for r in g)


def case_inputs(case, seed=0):
    from unflow_b200 import synthetic as synth
    spec, train_all, full_res, bidir, B, H, W, objective, storage, passes = case
    out = []
    for k in range(passes):
        if objective == "functional":
            out.append(_net_images(B, H, W, seed=31 + 7 * k + seed))
        else:
            out.append(tuple(t.cuda() for t in synth.supervised_batch(B, H, W, seed=41 + 7 * k + seed)))
    return out


def check_case(monkeypatch, cid, mode="3xtf32"):
    """Case ``cid``: the product, then the float64 oracle on its side of every kink; the comparison rows."""
    t0 = time.time()
    case = CASES[cid]
    tfv = _variables(case[0], case[2], seed=5)
    inputs = case_inputs(case)
    with monkeypatch.context() as m:
        sides = R.record_kink_sides(m)
        flows, grads, frozen = run_product(case, tfv, inputs, mode=mode)
    with monkeypatch.context() as m:
        used, cat = R.follow_kink_sides(m, sides)
        ref_flows, ref_grads = run_oracle(m, case, tfv, inputs)
    assert all(used[k] == cat[k].shape[0] for k in cat), "activations the oracle did not consume"
    rows = compare(flows, ref_flows, grads, ref_grads)
    torch.cuda.synchronize()
    return rows, frozen, time.time() - t0


@pytest.mark.parametrize("cid", list(CASES))
def test_network_matches_float64(monkeypatch, cid):
    rows, frozen, dt = check_case(monkeypatch, cid)
    print("\n" + table(cid, rows, dt))
    assert not frozen, "variables of frozen networks got a gradient: %s" % frozen
    f, g, _ = worst(rows)
    tau = TAU_GRAD_WARP if CASES[cid][1] and len(CASES[cid][0]) > 1 else TAU_GRAD
    assert f <= TAU_FLOW, "flows: %s" % max(rows["flow"])
    assert g <= tau, "gradients: %s" % max(rows["weights"] + rows["biases"])


def test_fp32_mode_yardstick(monkeypatch):
    """C-kitti with exact fp32 convolutions (cuDNN): what float32 arithmetic itself costs on this network."""
    rows, frozen, dt = check_case(monkeypatch, "C-kitti", mode="fp32")
    print("\n" + table("C-kitti fp32 mode", rows, dt))
    assert not frozen
    f, g, _ = worst(rows)
    assert f <= TAU_FLOW and g <= TAU_GRAD


@pytest.mark.parametrize("spec", ["C", "CSS"])
def test_evaluation_flows_match_float64(monkeypatch, spec):
    """eval.network_flow_fn (batch 1, no gradient, the four evaluation sizes) against the float64 network's final
    flows, resize_bilinear(flow2, [H, W]) * 20 of the last network (reference unsupervised.py:97-106)."""
    from unflow_b200 import synthetic as synth
    from unflow_b200.e2eflow.core import conv_ops
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.eval import network_flow_fn
    _float64_ops(monkeypatch)
    tfv = _variables(spec, False, seed=9)
    v = FlowNetVariables(spec, False, seed=0).load_tf_dict(tfv).cuda()
    v64 = {k: t.double().cuda() for k, t in tfv.items()}
    params = dict(synth.KITTI_PARAMS, flownet=spec)
    mean = torch.tensor(_norm()[0], dtype=torch.float64, device="cuda") / 255.0
    prev = conv_ops.get_mode()
    conv_ops.set_mode("3xtf32")
    rows = []
    try:
        fn = network_flow_fn(params, _norm(), v)
        for H, W in EVAL_SIZES:
            im1, im2, _ = synth.image_pair(1, H, W, seed=H + W)
            im1, im2 = im1.cuda(), im2.cuda()
            fw, bw = fn(im1, im2)
            with torch.no_grad():
                a, b = im1.double() / 255.0 - mean, im2.double() / 255.0 - mean
                rfw, rbw = oflownet.flownet(v64, a, b, spec, backward_flow=True)
            for d, got, ref in (("fw", fw, rfw[-1][0]), ("bw", bw, rbw[-1][0])):
                l2, mx = R.errors(got, tfc.resize_bilinear_legacy(ref, [H, W]) * (oflownet.FLOW_SCALE * 4))
                rows.append((max(l2, mx), l2, mx, "%dx%d %s" % (H, W, d)))
    finally:
        conv_ops.set_mode(prev)
    print("\n" + table("eval %s" % spec, {"flow": rows}, 0.0))
    assert max(rows)[0] <= TAU_FLOW, max(rows)


# ---- negative controls: wiring errors the per-launch checks cannot see ------------------------------------------
def _slot_overwrite(monkeypatch):
    """A later consumer of an activation overwrites the gradient the first one registered instead of adding."""
    from unflow_b200.e2eflow.core import conv_ops
    real = conv_ops._input_grad_into_slot
    monkeypatch.setattr(conv_ops, "_input_grad_into_slot",
                        lambda gen, x, launch: real(gen, x, lambda dst, acc: launch(dst, False)))


class _NoReverseFold:
    """The library with a correlation fold that passes the forward volume's gradient through and drops the reverse
    volume's."""

    def __init__(self, real):
        self._real = real

    def __getattr__(self, name):
        return getattr(self._real, name)

    def unflow_correlation_fold_grad(self, gout, grev, geff, B, C, H, W, ks, md, pad, s1, s2, stream):
        n = B * (2 * (md // s2) + 1) ** 2 * H * W
        R.view(geff, (n,)).copy_(R.view(gout, (n,)))
        return 0


def _no_reverse_fold(monkeypatch):
    from unflow_b200 import _native
    monkeypatch.setattr(_native, "_lib", _NoReverseFold(_native.lib()))


def _flow6_head_dropped(monkeypatch):
    """flow6 hands conv6_1 no input gradient (its weight and bias gradients stay)."""
    from unflow_b200.e2eflow.core import conv_ops
    real = conv_ops._NarrowConv3x3.backward

    def backward(ctx, g):
        if ctx.saved_tensors[0].shape[1] != 1024:
            return real(ctx, g)
        keep = conv_ops._input_grad_into_slot
        conv_ops._input_grad_into_slot = lambda gen, x, launch: None
        try:
            return real(ctx, g)
        finally:
            conv_ops._input_grad_into_slot = keep
    monkeypatch.setattr(conv_ops._NarrowConv3x3, "backward", staticmethod(backward))


CONTROLS = {"slot overwritten": _slot_overwrite, "reverse volume not folded": _no_reverse_fold,
            "flow6 input gradient dropped": _flow6_head_dropped}


@pytest.mark.parametrize("control", list(CONTROLS))
def test_bound_catches_a_wiring_error(monkeypatch, control):
    """C-kitti with one wiring error patched in: its worst gradient must exceed TAU_GRAD by 10x."""
    with monkeypatch.context() as m:
        CONTROLS[control](m)
        rows, _, dt = check_case(m, "C-kitti")
    f, g, l2 = worst(rows)
    print("\n" + table("C-kitti, %s" % control, rows, dt))
    print("%s: worst gradient %.3e = %.0f x TAU_GRAD, its rel L2 %.3e" % (control, g, g / TAU_GRAD, l2))
    assert g > 10 * TAU_GRAD
