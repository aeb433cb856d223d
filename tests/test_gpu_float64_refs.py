"""The float64 references on the GPU equal themselves on the CPU.

tests/test_float64_refs_cpu.py pins the references on the CPU; the step checks evaluate them on the GPU, where
scatter_add_ (warp_grads, level_loss_grad_scale, forward_warp), gather and the cuDNN float64 convolutions
(ref_conv, ref_wgrad, census) take other code paths.  One case evaluates every pinned reference at the shapes the
GPU tests use (FlowNetC's 48x160 correlation with d = 20 on 16 of its channels, the level loss of a 12x40 level with
R = 3 in every occlusion mode, the tensor-core layer shapes) on cuda and on the CPU, and compares them: worst
relative deviation 3.6e-15 on an H100 SXM 80 GB (ref_wgrad_window, a cuDNN float64 weight gradient), bound 1e-13.
It also reads a tensor back through float64_refs.view, which only the GPU files use.
"""
import pytest
import torch

import float64_refs as R
from test_gpu_step_launches import adam_reference, l2_bits, tf32_rna
from test_gpu_tc_step_launches import ref_conv, ref_conv_window, ref_wgrad, ref_wgrad_window

pytestmark = pytest.mark.gpu

TOL = 1e-13


def worst(got, want):
    """max |got - want| / max |want| over matching outputs (tuples and lists walked)."""
    if isinstance(got, (tuple, list)):
        return max([worst(g, w) for g, w in zip(got, want)] + [0.0])
    if not torch.is_tensor(got):
        return 0.0
    got, want = got.detach().cpu().double(), want.detach().cpu().double()
    assert got.shape == want.shape
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-300)) if got.numel() else 0.0


def cases(dev):
    g = torch.Generator().manual_seed(17)
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64).to(dev)
    u = lambda *s: torch.rand(*s, generator=g, dtype=torch.float64).to(dev)
    out = {}
    at = (1, 20, 20, 1, 2)
    a, b = r(1, 16, 48, 160), r(1, 16, 48, 160)
    c = R.correlation(a, b, *at)
    out["correlation"] = c
    out["correlation_grads"] = R.correlation_grads(r(*c.shape), a, b, at)
    out["fold_reverse"] = R.fold_reverse(c, 2, 10)
    img, flow = u(2, 96, 320, 3), r(2, 96, 320, 2) * 4
    out["downsample"] = R.downsample(img, 4)
    for mode in (0, 1, 2):
        f = flow if mode != 2 else u(2, 96, 320, 2) * torch.tensor([330.0, 100.0], device=dev) - 5
        out["warp %d" % mode] = (R.warp(img, f, mode), R.warp_abs(img, f, mode))
        out["warp_grads %d" % mode] = R.warp_grads(r(*img.shape), img, f, mode)
    fw = r(2, 48, 160, 2) * 3
    out["forward_warp"] = R.forward_warp(fw)
    out["forward_warp_grads"] = R.forward_warp_grads(r(2, 48, 160, 1), fw)
    B, h, w = 2, 12, 40
    im1, im2, ffw, fbw = u(B, h, w, 3), u(B, h, w, 3), r(B, h, w, 2) * 2, r(B, h, w, 2) * 2
    border = (u(B, h, w, 1) > 0.1).double()
    splat_fw, splat_bw = R.forward_warp(ffw)[0], R.forward_warp(fbw)[0]
    gl = r(8).abs()
    gl[R.TERMS.index('grad')] = 0
    bits = sum(1 << k for k, n in enumerate(R.TERMS) if n != 'grad')
    for occl in (0, 1, 2):
        L = R.LevelInputs(im1, im2, ffw, fbw, border if occl else None, splat_fw, splat_bw, occl, 3, bits)
        mfw, mbw = R.masks_f32(ffw, fbw, L.border, occl, splat_fw, splat_bw)
        assert mfw.device == ffw.device
        mfw, mbw = mfw.double(), mbw.double()
        out["masks %d" % occl] = (mfw, mbw)
        out["level_losses %d" % occl] = R.level_losses(L, L.ffw, L.fbw, mfw, mbw)
        out["level_loss_grads %d" % occl] = R.level_loss_grads(L, mfw, mbw, gl)
        out["level_loss_grad_scale %d" % occl] = R.level_loss_grad_scale(L, mfw, mbw, gl)
    out["census"] = R.census(R.gray255(im1), 3)
    out["supervised_loss_grads"] = R.supervised_loss_grads(r(2, 24, 80, 2), r(2, 96, 320, 2) * 20,
                                                           (u(2, 96, 320, 1) > 0.3).double())
    x = r(2, 48, 96, 160)
    wt = r(9, 64, 48)
    out["ref_conv 0"] = ref_conv(x, wt, 0, 2, 3, 3, 0, 0, 48, 80)
    out["ref_wgrad 0"] = ref_wgrad(r(2, 64, 48, 80), x, 2, 3, 3, 0, 0)
    xd, wd = r(2, 32, 24, 40), r(16, 16, 32)
    out["ref_conv 1"] = ref_conv(xd, wd, 1, 2, 4, 4, 1, 1, 48, 80)
    out["ref_wgrad 1"] = ref_wgrad(xd, r(2, 16, 48, 80), 2, 4, 4, 1, 1)
    xp, ww = r(2, 96, 320, 4), r(7, 24, 32)
    out["ref_conv_window"] = ref_conv_window(xp, ww, 2, 7, 3, 48, 160)
    out["ref_wgrad_window"] = ref_wgrad_window(r(2, 24, 48, 160), xp, 2, 7, 3)
    n = 4096
    mask = torch.randint(0, 16, (n // 4,), generator=g, dtype=torch.uint8).to(dev)
    out["adam_reference"] = adam_reference(r(n) * 0.05, r(n) * 1e-3, r(n) * 1e-4, u(n) * 1e-6, 1e-4, 0.9, 0.999, 1e-8,
                                           0.5, 7.0, l2_bits(mask, n), 4e-4)
    out["tf32_rna"] = tf32_rna(r(n).float()).double()
    return out


def test_references_on_the_gpu_equal_the_cpu():
    gpu, cpu = cases("cuda"), cases("cpu")
    ratios = {k: worst(gpu[k], cpu[k]) for k in cpu}
    print("\n" + "\n".join("%-28s %.2e" % kv for kv in sorted(ratios.items(), key=lambda kv: -kv[1])))
    bad = {k: v for k, v in ratios.items() if not v <= TOL}
    assert not bad, bad
    t = torch.arange(12, dtype=torch.float32, device="cuda")
    assert torch.equal(R.view(t.data_ptr(), (3, 2), (4, 1)), t.view(3, 4)[:, :2])
