"""The unsupervised training objective against float64, end to end: loss terms, flows and every variable gradient.

tests/test_gpu_float64_network.py holds the networks' backprop to a float64 network with a linear functional of
the flows as the objective; the per-launch checks hold each level-loss call to float64 on the operands it received.
Neither sees the host glue between the flows and the loss scalar: the image and border-mask pyramids (downsample by
4, then by 2 per level; under augment the product mask_local * mask_global), the per-level flow scale
top_scale / 2**lvl, the level weights and census radii (_LEVEL_WEIGHTS / _FULL_RES_WEIGHTS), the fused path's weight
vector and its dot product (fused_loss.TERM_ORDER against the config's <term>_weight), the unfused Sobel 'grad' term
on the kernel's masks, "only the last network is scored", the regularisation term and final_flow's legacy bilinear
resize.  Here unsupervised_loss runs in 3xTF32 with the gradients read from the Trainer's flat buffer (plus the L2
term the Adam kernel adds), as Adam reads them, and the oracle's own graph (oracle/unsupervised.py, oracle/losses.py,
oracle/flownet.py) runs in float64 on the GPU on the same inputs and variables, with the float64_refs correlation,
warp and downsample in place of its CPU float32 ops.

The float64 side takes the product's decisions, so that the bound can be tight:
  * flow values: the float64 network's flows enter the loss with the product's values and the float64 derivative
    (f64 + (f32 - f64).detach()), so the loss and its cotangent are evaluated at the point the product evaluated
    them.  Evaluated at the float64 network's own flows instead, the ~1e-5 forward difference of the flows enters
    the gradient through the Charbonnier curvature of the smoothness and fb terms (up to 2(1e-3)^-1.1 ~ 2000 where
    a second difference of the flow is near 0), and a flow head's bias gradient, in which the smoothness terms
    cancel exactly, came out 2.9e-2 off (cs-cityscapes stack_1 flow2/biases; 2.3e-2 rel L2).  That, not mask
    bits, is what the float32-oracle tests' 5e-3 / 1e-2 bounds absorb.  The networks' own flows (every level of
    the scored network, float64 against fp32) are scored separately in the flow family;
  * leaky-ReLU sides: float64_refs.record_kink_sides / follow_kink_sides, as the network file;
  * mask bits: per level and direction, the masks the level-loss kernel wrote (outgoing or border mask times the
    fb / disocc test).  The float64 loss uses the kernel's decisions (mask != 0) times its own border pyramid.  That
    is only legitimate if the decisions are right, so every case asserts they equal float64_refs.masks_f32, the
    mask formulas in fp32 on the product's own level flows (with the float64 side's border mask and the product's
    forward-warp splat maps), bit for bit, and that the kernel's mask values differ from those by fp32 rounding of
    the border pyramid at most.  Each case prints how many of those bits the float64 flows would have flipped;
  * bilinear taps: the loss's image_warp takes floor() from the product's fp32 level flow (the float64 level flow
    is the same value scaled without fp32 rounding) and the fraction from the float64 flow.  The file needs no
    separate warp bound (the network file's TAU_GRAD_WARP): no case here differentiates a stacked network's
    image_warp (frozen networks detach it), and the loss's warps follow the product's taps.
  * augmentation: the product's augmented loss images, network images and combined mask are fed to the float64
    side (they carry no gradient; the sampler is checked per launch).

Every scalar (the total loss, each tracked per-level term loss<k>/<term> and each tracked weighted sum loss/<term>),
both returned full-size flows (final_flow), every level flow of the scored network and every variable gradient
(weights and biases separately) is scored by the larger of its relative L2 error and its max error over max |ref|.
Variables of frozen networks must get no gradient.

Every case also checks that the forward-warp splat maps the kernel read are float64_refs.forward_warp of the
product's level flow of their direction (within TAU_SUM of the per-launch checks), and, where mask_occlusion is set,
that the occlusion test cleared bits inside the border.  The initial networks' flows are too small to disocclude
anything, so s-disocc-sym scales the flow heads (_FLOW_HEADS) until every level has disoccluded pixels in both
directions, on partly different pixels; that case asserts it per level.

Measured on an H100 SXM 80 GB (HBM3) at a 700 W power limit (worst rel L2 / max per family; the mask bits, all
equal to masks_f32, the bits the occlusion test cleared inside the border, and how many bits the float64 network's
own flows would have flipped):

  case               loss       flows               weight gradients    bias gradients      bits     occluded  flip
  C-kitti            8.0e-7     8.0e-6 / 1.0e-5     2.0e-5 / 1.9e-5     1.6e-5 / 1.9e-5     122760   49987     0
  C-chairs           4.3e-6     8.0e-6 / 9.9e-6     1.3e-5 / 1.6e-5     2.1e-5 / 1.9e-5     65472    -         0
  S-synthia          7.4e-7     1.5e-5 / 1.7e-5     2.8e-5 / 2.1e-5     2.1e-5 / 2.2e-5     130944   -         0
  cs-cityscapes      2.1e-6     1.6e-5 / 1.8e-5     2.2e-5 / 2.1e-5     7.5e-5 / 9.6e-5     174592   124567    0
  CSS-bench          3.6e-7     2.7e-5 / 2.8e-5     3.0e-5 / 3.1e-5     2.1e-4 / 2.1e-4     163680   126577    0
  s-full_res         1.6e-6     1.3e-5 / 1.2e-5     2.4e-5 / 2.6e-5     5.7e-5 / 6.7e-5     174752   -         0
  s-photo-outgoing   1.9e-6     1.3e-5 / 1.2e-5     7.6e-5 / 1.2e-4     1.0e-4 / 1.1e-4     10912    -         0
  s-disocc-sym       7.9e-7     3.4e-6 / 4.8e-6     1.9e-5 / 2.1e-5     4.6e-5 / 4.6e-5     10912    238       0
  s-grad             7.0e-6     1.3e-5 / 1.2e-5     2.6e-5 / 2.6e-5     1.8e-5 / 1.6e-5     10912    -         0
  s-no_pyramid       1.8e-7     1.3e-5 / 1.2e-5     3.9e-5 / 3.4e-5     7.6e-5 / 5.6e-5     8192     -         0
  s-augment          9.6e-7     1.4e-5 / 1.5e-5     2.5e-5 / 3.0e-5     2.0e-5 / 2.1e-5     10912    -         0
  C-kitti fp32 mode  2.8e-7     2.6e-6 / 3.9e-6     1.4e-5 / 1.3e-5     1.5e-5 / 1.4e-5     122760   49987     0

C-kitti's fb test clears bits on the finest level only, cs-cityscapes' and CSS-bench's on every level; s-disocc-sym
per level, fw / bw: 21/15 8/8 49/50 28/27 16/16 (the coarsest level entirely).  The augmented mask pyramid differs
from the float64 one by fp32 rounding (6e-8); every other kernel mask equals masks_f32 exactly.  The worst bias
gradient moves from run to run with the float atomics' order: CSS-bench's stack_2 flow2/biases measured 1.5e-5 in
one run and 2.1e-4 in another.  The loss family is the level-loss kernels and the host glue at one point, the flow
and gradient families add the networks (the flows as in the network file).  Bounds, 3x the worst measured:
TAU_LOSS 2.1e-5, TAU_FLOW 8.4e-5, TAU_GRAD 6.2e-4.  The file takes about 30 s of GPU time.

Negative controls on C-chairs (test_bound_catches_a_loss_wiring_error): the worst score and its multiple of its
family's bound, and the worst gradient score:
  level 2's flow scaled by top_scale / 2**3              loss4/smooth_2nd 4.6e-1 (22000x TAU_LOSS)    gradient 5.8e-1
  the weights of levels 1 and 2 swapped                  flow6_up5/biases 1.2e-1 (199x TAU_GRAD)      gradient 1.2e-1
  level 2 without the border mask                        loss4/ternary 8.2e-2 (3900x TAU_LOSS)        gradient 2.9e-2
  smooth_2nd's weight left out of the fused vector       loss/combined 2.2e-1 (10600x TAU_LOSS)       gradient 1.2
The level-weight swap moves no loss term the tracked scalars report per level, only loss/<term> (3.3e-3) and the
gradients; the border control also shows in the mask check (578 bits).
"""
import time
from types import SimpleNamespace

import pytest
import torch

import float64_refs as R
from oracle import flownet as oflownet
from oracle import losses as olosses
from oracle import unsupervised as ounsup
from test_gpu_float64_network import _float64_ops, _norm, _param, _trainable, _variables, table
from test_gpu_step_launches import TAU_SUM
from test_gpu_variant_step_launches import (CHAIRS_PARAMS, CITYSCAPES_PARAMS, CSS_BENCH_PARAMS, KITTI_PARAMS,
                                            SYNTHIA_PARAMS)

pytestmark = pytest.mark.gpu

TAU_LOSS = 2.1e-5       # 3x the worst measured (see the docstring)
TAU_FLOW = 8.4e-5
TAU_GRAD = 6.2e-4
TAU = {"loss": TAU_LOSS, "flow": TAU_FLOW, "weights": TAU_GRAD, "biases": TAU_GRAD}

_SMALL = dict(flownet='s', pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0)

# id -> (loss parameters, B, H, W, augment)
CASES = {
    "C-kitti": (KITTI_PARAMS, 2, 320, 1152, False),
    "C-chairs": (CHAIRS_PARAMS, 2, 384, 512, False),
    "S-synthia": (SYNTHIA_PARAMS, 2, 512, 768, False),
    "cs-cityscapes": (CITYSCAPES_PARAMS, 2, 512, 1024, False),
    "CSS-bench": (CSS_BENCH_PARAMS, 2, 384, 1280, False),
    "s-full_res": (dict(_SMALL, full_res=True), 2, 128, 256, False),
    # the branches the configurations above do not reach
    "s-photo-outgoing": (dict(flownet='s', pyramid_loss=True, border_mask=False, mask_occlusion='',
                              photo_weight=1.0, smooth_1st_weight=3.0), 2, 128, 256, False),
    "s-disocc-sym": (dict(_SMALL, mask_occlusion='disocc', sym_weight=1.0, occ_weight=12.4), 2, 128, 256, False),
    "s-grad": (dict(_SMALL, grad_weight=1.0), 2, 128, 256, False),
    "s-no_pyramid": (dict(_SMALL, pyramid_loss=False), 2, 128, 256, False),
    "s-augment": (_SMALL, 2, 128, 256, True),
}

# id -> (flow-head weight gain, flow-head bias shift in level pixels).  The initial networks' flows stay within a few
# pixels of zero and shrink towards the coarse levels (0.07 px at 2x4), so no pixel inside the border would be
# disoccluded at any level: this makes every level's flow diverge enough that each level, in each direction, has
# disoccluded pixels inside the border, and fw and bw differ on some of them.
_FLOW_HEADS = {"s-disocc-sym": (3.0, 2.5)}

_OCCL = {'': 0, 'fb': 1, 'disocc': 2}


def _case_variables(cid):
    params = CASES[cid][0]
    tfv = _variables(params['flownet'], params.get('full_res'), seed=5)
    if cid in _FLOW_HEADS:
        gain, shift = _FLOW_HEADS[cid]
        for n in range(2, 7):
            root = 'flownet_s/flow%d/' % n
            tfv[root + 'weights'] = tfv[root + 'weights'] * gain
            tfv[root + 'biases'] = tfv[root + 'biases'] + shift * 2 ** (n - 2) / oflownet.FLOW_SCALE
    return tfv


def _active(params):
    return [t for t in ounsup.LOSSES if params.get(t + '_weight')]


# ---- the product ----------------------------------------------------------------------------------------------------
def _record_loss_side(m, augment):
    """Record every level-loss call (its fp32 flows, the masks the kernel wrote, the forward-warp splat maps it
    read) and, under augment, the augmented images and mask."""
    from unflow_b200.e2eflow.core import fused_loss
    from unflow_b200.e2eflow.core import unsupervised as unsup
    rec = SimpleNamespace(levels=[], augmented=None, flows=None)
    real_fused, real_fwarp, real_flownet = fused_loss.compute_losses_fused, fused_loss.forward_warp, unsup.flownet
    splats = []

    def fwarp(flow):
        out = real_fwarp(flow)
        splats.append(out.detach())
        return out

    def fused(im1, im2, flow_fw, flow_bw, border_mask=None, mask_occlusion='', data_max_distance=1, terms=None,
              return_masks=False):
        del splats[:]
        losses, mfw, mbw = real_fused(im1, im2, flow_fw, flow_bw, border_mask, mask_occlusion, data_max_distance,
                                      terms, return_masks=True)
        rec.levels.append(dict(ffw=flow_fw.detach(), fbw=flow_bw.detach(), masks=(mfw[..., 0], mbw[..., 0]),
                               splats=tuple(splats) if splats else (None, None)))
        return (losses, mfw, mbw) if return_masks else losses
    m.setattr(fused_loss, "forward_warp", fwarp)
    m.setattr(fused_loss, "compute_losses_fused", fused)

    def flownet(*args, **kw):
        out = real_flownet(*args, **kw)
        rec.flows = [[[f.detach() for f in net] for net in stack] for stack in out]
        return out
    m.setattr(unsup, "flownet", flownet)
    if augment:
        real_aug = unsup._augmented

        def augmented(*args):
            out = real_aug(*args)
            rec.augmented = [t.detach() for t in out]
            return out
        m.setattr(unsup, "_augmented", augmented)
    return rec


def run_product(m, case, tfv, batch, mode, rec):
    """unsupervised_loss on ``batch``: ({loss, tracked scalars, flows}, {name: gradient}, frozen names with a
    gradient).  Gradients are read from the Trainer's flat buffer plus the L2 term the Adam kernel adds."""
    from unflow_b200.e2eflow.core import augment as aug
    from unflow_b200.e2eflow.core import conv_ops
    from unflow_b200.e2eflow.core import unsupervised as unsup
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.e2eflow.core.train import Trainer
    params, B, H, W, augment = case
    v = FlowNetVariables(params['flownet'], params.get('full_res'), seed=0).load_tf_dict(tfv)
    m.setattr(aug, "_device_rng", aug._device_rng)     # (the Trainer turns it on for augment)
    prev = conv_ops.get_mode()
    conv_ops.set_mode(mode)
    try:
        tr = Trainer(params, _norm(), torch.device("cuda", 0), variables=v, augment=augment)
        torch.cuda.manual_seed(17)
        loss, ffw, fbw = unsup.unsupervised_loss(batch, params, _norm(), augment=augment, return_flow=True,
                                                 variables=v)
        tracked = {k: t for k, t in unsup.tracked.items() if torch.is_tensor(t)}
        loss.backward()
        torch.cuda.synchronize()
    finally:
        conv_ops.set_mode(prev)
    flat = tr.flat_grad + tr.l2_gradient()
    grads = {name: tr._view_like(flat[off:off + p.numel()], p)
             for name, p, off in zip(tr.trainable_names, tr.trainable, tr._offsets)}
    frozen = [n for n in v.variable_names() if n not in grads and _param(v, n).grad is not None]
    net = [("net %s %dx%d" % (d, f.shape[1], f.shape[2]), f) for d, stack in zip(("fw", "bw"), rec.flows)
           for f in stack[-1]]
    out = dict(loss=loss.detach(), tracked=tracked, flows=[("fw", ffw.detach()), ("bw", fbw.detach())] + net)
    return out, grads, frozen


# ---- the float64 side -----------------------------------------------------------------------------------------------
def _own_decisions(ffw, fbw, border, occl):
    """The mask decisions ([B,h,w] bool, fw and bw) the float64 flows would take themselves (for the flip count)."""
    out = []
    for f, g in ((ffw, fbw), (fbw, ffw)):
        B, h, w, _ = f.shape
        if border is None:
            x = torch.arange(w, device=f.device, dtype=f.dtype).view(1, 1, w) + f[..., 0]
            y = torch.arange(h, device=f.device, dtype=f.dtype).view(1, h, 1) + f[..., 1]
            keep = (x >= 0) & (x <= w - 1) & (y >= 0) & (y <= h - 1)
        else:
            keep = (border[..., 0] != 0).expand(B, h, w)
        if occl == 1:
            gw = R.warp(g, f, 1)
            fd = f + gw
            keep = keep & ~((fd * fd).sum(-1) > 0.01 * ((f * f).sum(-1) + (gw * gw).sum(-1)) + 0.5)
        elif occl == 2:
            keep = keep & ~(R.forward_warp(g)[0][..., 0] < 0.8)
        out.append(keep)
    return out


def _follow_loss_side(m, rec, log, own_flows):
    """oracle/unsupervised.py's compute_losses with the product's decisions: the level-loss kernel's mask bits
    (times the float64 border pyramid), its forward-warp splat maps (the disocclusion of 'sym') and the floor() of
    its level flows (image_warp's taps).  Checks into ``log``: the recorded bits against float64_refs.masks_f32, the
    splat maps against float64_refs.forward_warp of the product's level flow of their direction, and how many bits
    inside the border (or outgoing mask) the occlusion test cleared."""
    levels = iter(rec.levels)
    real = olosses.compute_losses

    def compute_losses(im1, im2, ffw, fbw, border_mask=None, mask_occlusion='', data_max_distance=1):
        L = next(levels)
        occl = _OCCL[mask_occlusion]
        with torch.no_grad():
            ref = R.masks_f32(L['ffw'], L['fbw'], None if border_mask is None else border_mask.float(), occl,
                              *L['splats'])
            own = _own_decisions(*own_flows(len(log)), border_mask, occl)
            base = R.masks_f32(L['ffw'], L['fbw'], None if border_mask is None else border_mask.float(), 0,
                               None, None)
            splat = 0.0
            if L['splats'][0] is not None:
                for got_splat, f in zip(L['splats'], (L['ffw'], L['fbw'])):
                    want, count = R.forward_warp(f.double())
                    splat = max(splat, R.worst_ratio(got_splat, want, want + count * 2.0 ** -24 / TAU_SUM))
        scale = 1.0 if border_mask is None else border_mask[..., 0].double()
        masks = iter([(scale * (k != 0).double())[..., None] for k in L['masks']])
        splats = iter([None if s is None else s.double() for s in L['splats']])
        follow = {id(ffw): L['ffw'], id(fbw): L['fbw']}
        with pytest.MonkeyPatch.context() as mm:
            mm.setattr(olosses, "image_warp", lambda im, f: R.warp(im, f, 1, floor_from=follow[id(f)]))
            mm.setattr(olosses, "create_outgoing_mask", lambda f: next(masks))
            mm.setattr(olosses, "_ops", SimpleNamespace(
                forward_warp=lambda f: next(splats) if L['splats'][0] is not None else f[..., :1] * 0 + 1))
            out = real(im1, im2, ffw, fbw, None, '', data_max_distance)
        log.append(dict(
            terms={k: v.detach() for k, v in out.items() if torch.is_tensor(v)},
            bits=sum(k.numel() for k in L['masks']),
            disagree=sum(int(((k != 0) != (r != 0)).sum()) for k, r in zip(L['masks'], ref)),
            value_diff=max(float((k - r).abs().max()) for k, r in zip(L['masks'], ref)),
            flipped=sum(int(((k != 0) != o).sum()) for k, o in zip(L['masks'], own)),
            occluded=[int(((b != 0) & (k == 0)).sum()) for k, b in zip(L['masks'], base)],
            splat=splat))
        return out
    m.setattr(ounsup, "compute_losses", compute_losses)


def run_float64(m, case, tfv, batch, rec):
    """oracle/unsupervised.py in float64 on the GPU, on the product's decisions and at the product's flow values:
    ({loss, per-level terms, weighted sums, flows}, {name: gradient in the product's layout}, the mask log of every
    level)."""
    params, B, H, W, augment = case
    spec, full_res = params['flownet'], params.get('full_res')
    _float64_ops(m)
    m.setattr(ounsup, "downsample", lambda t, n: R.downsample(t.contiguous(), n))
    batch64 = [t.double() for t in batch]
    if augment:
        geo1, geo2, net1, net2, mask = [t.double() for t in rec.augmented]
        mean = torch.tensor(_norm()[0], dtype=torch.float64, device="cuda") / 255.0
        batch64 = [geo1 * 255.0, geo2 * 255.0]
        m.setattr(ounsup, "create_border_mask", lambda t, ratio: mask)
    real_flownet = ounsup.flownet
    own = []

    def flownet(variables, a, b, **kw):
        """The float64 network; the flows it hands on carry the product's values with the float64 derivative."""
        if augment:
            a, b = net1 - mean, net2 - mean
        out = real_flownet(variables, a, b, **kw)
        own.extend(out)
        return [[[f + (g.double() - f).detach() for f, g in zip(n64, n32)] for n64, n32 in zip(s64, s32)]
                for s64, s32 in zip(out, rec.flows)]
    m.setattr(ounsup, "flownet", flownet)
    top = oflownet.FLOW_SCALE * (4 if full_res else 1)
    log = []
    _follow_loss_side(m, rec, log, lambda k: [s[-1][k].detach() * (top / 2 ** k) for s in own])
    train = _trainable(spec, params.get('train_all'), list(tfv))
    leaves = {k: t.double().cuda().requires_grad_(k in train) for k, t in tfv.items()}
    loss, ffw, fbw, by_term = ounsup.unsupervised_loss(leaves, batch64, params, normalization=_norm(),
                                                       return_flow=True, return_terms=True)
    loss.backward()
    grads = {}
    for k in train:
        g = leaves[k].grad
        grads[k] = g.permute(3, 2, 0, 1) if k.endswith('/weights') else g
    net = [("net %s %dx%d" % (d, f.shape[1], f.shape[2]), f.detach()) for d, stack in zip(("fw", "bw"), own)
           for f in stack[-1]]
    by_term = {k: v.detach() if torch.is_tensor(v) else v for k, v in by_term.items()}
    out = dict(loss=loss.detach(), by_term=by_term, flows=[("fw", ffw.detach()), ("bw", fbw.detach())] + net)
    return out, grads, log


# ---- comparison -----------------------------------------------------------------------------------------------------
def compare(params, got, ref, log, got_grads, ref_grads):
    """{'loss' | 'flow' | 'weights' | 'biases': [(score, rel L2, max, name)]}; a missing gradient scores infinity."""
    rows = {"loss": [], "flow": [], "weights": [], "biases": []}

    def add(fam, g, r, name):
        l2, mx = R.errors(g, r)
        rows[fam].append((max(l2, mx), l2, mx, name))
    add("loss", got["loss"], ref["loss"], "loss/combined")
    active = _active(params)
    for k, lvl in enumerate(log):
        for t in active:
            add("loss", got["tracked"]["loss%d/%s" % (k + 2, t)], lvl["terms"][t], "loss%d/%s" % (k + 2, t))
    assert not any(k.startswith("loss%d/" % (len(log) + 2)) for k in got["tracked"]), "levels the oracle did not score"
    for t in active:
        add("loss", got["tracked"]["loss/" + t], ref["by_term"][t], "loss/" + t)
    assert [n for n, _ in got["flows"]] == [n for n, _ in ref["flows"]]
    for (n, g), (_, r) in zip(got["flows"], ref["flows"]):
        add("flow", g, r, "flow " + n)
    assert set(got_grads) == set(ref_grads), sorted(set(got_grads) ^ set(ref_grads))
    for name, r in ref_grads.items():
        fam = "weights" if name.endswith('/weights') else "biases"
        add(fam, got_grads[name], r, name)
    return rows


def mask_line(log):
    bits = sum(lvl["bits"] for lvl in log)
    return ("masks: %d levels, %d bits, %d disagree with masks_f32 on the product's flows (values within %.1e); "
            "the float64 flows would flip %d\n  occluded inside the border, fw / bw per level: %s; splat maps "
            "%.1e of TAU_SUM" % (len(log), bits, sum(lvl["disagree"] for lvl in log),
                                 max(lvl["value_diff"] for lvl in log), sum(lvl["flipped"] for lvl in log),
                                 " ".join("%d/%d" % tuple(lvl["occluded"]) for lvl in log),
                                 max(lvl["splat"] for lvl in log) / TAU_SUM))


def assert_case(params, rows, log, frozen):
    """The checks every case passes: no gradient into frozen networks, the kernel's mask bits, its splat maps, an
    occlusion test that actually masks pixels when one is configured, every family within its bound."""
    assert not frozen, "variables of frozen networks got a gradient: %s" % frozen
    assert all(lvl["disagree"] == 0 for lvl in log), "the level-loss kernel's mask bits: %s" % mask_line(log)
    assert all(lvl["value_diff"] <= 1e-6 for lvl in log), mask_line(log)
    assert all(lvl["splat"] <= TAU_SUM for lvl in log), mask_line(log)
    occl = params.get('mask_occlusion', '')
    if occl:
        assert sum(sum(lvl["occluded"]) for lvl in log) > 0, "the occlusion test masks nothing: %s" % mask_line(log)
    if occl == 'disocc':
        assert all(min(lvl["occluded"]) > 0 for lvl in log), "a level without disocclusion: %s" % mask_line(log)
    for fam, rs in rows.items():
        assert max(rs)[0] <= TAU[fam], "%s: %s" % (fam, max(rs))


def case_batch(case, seed=0):
    from unflow_b200 import synthetic as synth
    params, B, H, W, augment = case
    im1, im2, _ = synth.image_pair(B, H, W, seed=53 + seed)
    return im1.cuda(), im2.cuda()


def check_case(monkeypatch, cid, mode="3xtf32", control=None):
    """Case ``cid`` (with a wiring error patched into the product, if ``control``): the product, then the float64
    oracle on its decisions; the comparison rows, the mask log, frozen variables with a gradient, seconds."""
    t0 = time.time()
    case = CASES[cid]
    params = case[0]
    tfv = _case_variables(cid)
    batch = case_batch(case)
    with monkeypatch.context() as m:
        if control is not None:
            control(m)
        sides = R.record_kink_sides(m)
        rec = _record_loss_side(m, case[4])
        got, got_grads, frozen = run_product(m, case, tfv, batch, mode, rec)
    with monkeypatch.context() as m:
        used, cat = R.follow_kink_sides(m, sides)
        ref, ref_grads, log = run_float64(m, case, tfv, batch, rec)
    assert all(used[k] == cat[k].shape[0] for k in cat), "activations the oracle did not consume"
    assert len(log) == len(rec.levels), "level-loss calls the oracle did not make"
    rows = compare(params, got, ref, log, got_grads, ref_grads)
    torch.cuda.synchronize()
    return rows, log, frozen, time.time() - t0


def over(rows):
    """(worst score / its family's bound, that row)."""
    return max(((r[0] / TAU[fam], r) for fam, rs in rows.items() for r in rs), key=lambda x: x[0])


@pytest.mark.parametrize("cid", list(CASES))
def test_objective_matches_float64(monkeypatch, cid):
    rows, log, frozen, dt = check_case(monkeypatch, cid)
    print("\n" + table(cid, rows, dt) + "\n  " + mask_line(log))
    assert_case(CASES[cid][0], rows, log, frozen)


def test_fp32_mode_yardstick(monkeypatch):
    """C-kitti with exact fp32 convolutions (cuDNN): what float32 arithmetic itself costs on this objective."""
    rows, log, frozen, dt = check_case(monkeypatch, "C-kitti", mode="fp32")
    print("\n" + table("C-kitti fp32 mode", rows, dt) + "\n  " + mask_line(log))
    assert_case(CASES["C-kitti"][0], rows, log, frozen)


# ---- negative controls: loss-side wiring errors ---------------------------------------------------------------------
_CONTROL_LEVEL = 2


def _at_level(m, change):
    """The product's compute_losses with ``change(flow_fw, flow_bw, kwargs)`` applied at level _CONTROL_LEVEL."""
    from unflow_b200.e2eflow.core import unsupervised as unsup
    real = unsup.compute_losses
    calls = [0]

    def compute_losses(im1, im2, ffw, fbw, **kw):
        if calls[0] == _CONTROL_LEVEL:
            ffw, fbw, kw = change(ffw, fbw, kw)
        calls[0] += 1
        return real(im1, im2, ffw, fbw, **kw)
    m.setattr(unsup, "compute_losses", compute_losses)


def _flow_scale_halved(m):
    """One level's flow in pixels scaled by top_scale / 2**(lvl+1) instead of top_scale / 2**lvl."""
    _at_level(m, lambda f, b, kw: (f * 0.5, b * 0.5, kw))


def _level_weights_swapped(m):
    """The weights of levels 1 and 2 (4.35, 3.9) swapped."""
    from unflow_b200.e2eflow.core import unsupervised as unsup
    w = list(unsup._LEVEL_WEIGHTS)
    w[1], w[2] = w[2], w[1]
    m.setattr(unsup, "_LEVEL_WEIGHTS", w)


def _border_dropped(m):
    """One level's loss without the border mask."""
    _at_level(m, lambda f, b, kw: (f, b, dict(kw, border_mask=None)))


def _term_weight_dropped(m):
    """smooth_2nd's weight left out of the fused weight vector (0 in its TERM_ORDER slot)."""
    from unflow_b200.e2eflow.core import fused_loss
    from unflow_b200.e2eflow.core import unsupervised as unsup
    real = unsup._device_constant
    slot = fused_loss.TERM_ORDER.index('smooth_2nd')

    def constant(values, device):
        values = list(values)
        if len(values) == len(fused_loss.TERM_ORDER):
            values[slot] = 0.0
        return real(values, device)
    m.setattr(unsup, "_device_constant", constant)


CONTROLS = {"level flow scale halved": _flow_scale_halved, "level weights swapped": _level_weights_swapped,
            "border mask dropped": _border_dropped, "term weight dropped": _term_weight_dropped}


@pytest.mark.parametrize("control", list(CONTROLS))
def test_bound_catches_a_loss_wiring_error(monkeypatch, control):
    """C-chairs with one loss-side wiring error patched into the product: its worst score must exceed its
    family's bound by 10x."""
    rows, log, _, dt = check_case(monkeypatch, "C-chairs", control=CONTROLS[control])
    ratio, row = over(rows)
    print("\n" + table("C-chairs, %s" % control, rows, dt) + "\n  " + mask_line(log))
    print("%s: worst %.3e = %.0f x its bound (%s)" % (control, row[0], ratio, row[3]))
    assert ratio > 10
