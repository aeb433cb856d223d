"""The supervised fine-tune (dataset = kitti_ft) on the GPU: the fused loss kernel of
csrc/supervised_loss.cu against a float64 evaluation of the unfused expression, supervised_loss
against the CPU oracle, the Trainer in supervised mode (eager, CUDA graph, prefetch) and run.py's
kitti_ft branch."""
import ctypes
import glob
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import flownet as oflownet
from oracle import supervised as osup
from unflow_b200 import synthetic as usynth
import synth
from float64_refs import supervised_loss_grads


def _inputs(B, h, w, H, W, mask_kind, seed):
    g = torch.Generator().manual_seed(seed)
    flow = torch.randn(B, h, w, 2, generator=g) * 0.5               # network units: x20 -> ~10 px
    gt = torch.randn(B, H, W, 2, generator=g) * 8.0
    mask = None
    if mask_kind == "sparse":
        mask = (torch.rand(B, H, W, 1, generator=g) < 0.3).float()
    elif mask_kind == "zero":
        mask = torch.zeros(B, H, W, 1)
    elif mask_kind == "invalid":                                     # KITTI: invalid pixels decode to -512
        mask = (torch.rand(B, H, W, 1, generator=g) < 0.6).float()
        gt = torch.where(mask > 0, gt, torch.full_like(gt, -512.0))
    return flow, gt, mask


def _kernel(flow, gt, mask, grad=1.0, scale=20.0):
    from unflow_b200 import _native
    lib = _native.lib()
    B, h, w, _ = flow.shape
    H, W = gt.shape[1:3]
    flow, gt = flow.cuda().contiguous(), gt.cuda().contiguous()
    mask = mask.cuda().contiguous() if mask is not None else None
    loss = torch.empty(1, device="cuda")
    ws = torch.empty(int(lib.unflow_supervised_loss_workspace_bytes(B, H, W)), device="cuda", dtype=torch.uint8)
    mp = mask.data_ptr() if mask is not None else None
    st = torch.cuda.current_stream().cuda_stream
    _native.check(lib.unflow_supervised_loss_fwd(flow.data_ptr(), gt.data_ptr(), mp, loss.data_ptr(), ws.data_ptr(),
                                                 B, h, w, H, W, scale, st), "fwd")
    gl = torch.tensor([grad], device="cuda")
    dflow = torch.full_like(flow, float("nan"))                      # every element must be written
    _native.check(lib.unflow_supervised_loss_bwd(gl.data_ptr(), flow.data_ptr(), gt.data_ptr(), mp, dflow.data_ptr(),
                                                 B, h, w, H, W, scale, st), "bwd")
    torch.cuda.synchronize()
    return loss.cpu()[0], dflow.cpu()


@pytest.mark.parametrize("mask_kind", ["none", "sparse", "zero", "invalid"])
@pytest.mark.parametrize("shape", [(4, 80, 192, 320, 768), (2, 13, 19, 50, 75), (2, 32, 32, 32, 32)],
                         ids=["x4", "odd", "ratio1"])
def test_kernel_vs_float64(shape, mask_kind):
    B, h, w, H, W = shape
    flow, gt, mask = _inputs(B, h, w, H, W, mask_kind, seed=sum(shape) + len(mask_kind))
    want_loss, want_d, budget = supervised_loss_grads(flow, gt, mask)
    got_loss, got_d = _kernel(flow, gt, mask)
    assert torch.isfinite(got_d).all()
    if mask_kind == "zero":
        assert float(got_loss) == 0.0 and float(got_d.abs().max()) == 0.0
    else:
        assert abs(float(got_loss) - float(want_loss)) <= 1e-5 * float(want_loss), (float(got_loss), float(want_loss))
        err = (got_d.double() - want_d).abs()
        ratio = float((err / (budget + 1e-30)).max())
        assert bool((err <= budget + 1e-30).all()), "dflow outside the float32 budget: worst ratio %.3g" % ratio
    # deterministic: a second run is bit-identical; a half upstream gradient gives exactly half
    again_loss, again_d = _kernel(flow, gt, mask)
    assert torch.equal(again_loss, got_loss) and torch.equal(again_d, got_d)
    _, half_d = _kernel(flow, gt, mask, grad=0.5)
    assert torch.equal(half_d * 2, got_d)


def test_kernel_argument_checks():
    from unflow_b200 import _native
    lib = _native.lib()
    buf = torch.zeros(4 * 64 * 64 * 2, device="cuda")
    ws = torch.zeros(int(lib.unflow_supervised_loss_workspace_bytes(1, 64, 64)), device="cuda", dtype=torch.uint8)
    p, s = buf.data_ptr(), torch.cuda.current_stream().cuda_stream
    fwd, bwd = lib.unflow_supervised_loss_fwd, lib.unflow_supervised_loss_bwd
    assert fwd(p, p, None, p, ws.data_ptr(), 1, 16, 16, 64, 64, 20.0, s) == _native.UNFLOW_OK
    for args in ((p, p, None, p, ws.data_ptr(), 0, 16, 16, 64, 64), (p, p, None, p, ws.data_ptr(), 1, 0, 16, 64, 64),
                 (p, p, None, p, ws.data_ptr(), 1, 16, 16, 64, -1), (None, p, None, p, ws.data_ptr(), 1, 16, 16, 64, 64),
                 (p, None, p, p, ws.data_ptr(), 1, 16, 16, 64, 64), (p, p, p, None, ws.data_ptr(), 1, 16, 16, 64, 64),
                 (p, p, p, p, None, 1, 16, 16, 64, 64), (p, p, None, p, ws.data_ptr(), 1, 16, 16, 1 << 16, 1 << 15)):
        assert fwd(*args, 20.0, s) == _native.UNFLOW_EINVAL, args
    assert bwd(p, p, p, None, p, 1, 16, 16, 64, 64, 20.0, s) == _native.UNFLOW_OK
    for args in ((None, p, p, None, p, 1, 16, 16, 64, 64), (p, None, p, None, p, 1, 16, 16, 64, 64),
                 (p, p, None, None, p, 1, 16, 16, 64, 64), (p, p, p, None, None, 1, 16, 16, 64, 64),
                 (p, p, p, None, p, 1, 16, 0, 64, 64)):
        assert bwd(*args, 20.0, s) == _native.UNFLOW_EINVAL, args
    assert lib.unflow_supervised_loss_workspace_bytes(0, 64, 64) == 0
    torch.cuda.synchronize()


def _close(got, want, rtol, atol_rel=1e-5):
    want, got = want.detach().cpu(), got.detach().cpu()
    np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=rtol,
                               atol=atol_rel * max(float(want.abs().max()), 1e-12))


@pytest.mark.parametrize("spec,hw,train_all", [("C", (128, 256), False), ("CS", (64, 128), True)])
def test_supervised_loss_vs_oracle(spec, hw, train_all):
    """The fused path on the GPU against the CPU restatement of the reference: loss value and the
    gradient of every trained variable (relative L2, as test_unsupervised_loss_vs_oracle)."""
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.e2eflow.core.supervised import supervised_loss
    params = dict(flownet=spec, train_all=train_all)
    tfv = oflownet.init_variables(spec, False, seed=13)
    for k in tfv:
        tfv[k] = tfv[k].clone().requires_grad_(True)
    v = FlowNetVariables(spec, False, seed=0).load_tf_dict({k: t.detach() for k, t in tfv.items()}).cuda()
    batch = usynth.supervised_batch(2, hw[0], hw[1], seed=17)
    want = osup.supervised_loss(tfv, batch, params, synth.KITTI_NORMALIZATION)
    got = supervised_loss(tuple(t.cuda() for t in batch), params, synth.KITTI_NORMALIZATION, augment=False, variables=v)
    _close(got, want, rtol=2e-4)
    want.backward()
    got.backward()
    checked = 0
    for scope in v.kinds:
        w, b = v.weights(scope)
        for g, t, suffix in ((w.grad, tfv[scope + '/weights'].grad, '/weights'), (b.grad, tfv[scope + '/biases'].grad, '/biases')):
            if t is None or float(t.norm()) == 0.0:
                continue
            t = t.permute(3, 2, 0, 1) if suffix == '/weights' else t
            err = float((g.cpu() - t).norm() / t.norm())
            assert err < 5e-3, "%s%s: relative L2 gradient error %.3e" % (scope, suffix, err)
            checked += 1
    assert checked >= 20


def test_fused_matches_unfused_on_the_gpu():
    """flow_loss: the CUDA kernel and the unfused torch expression agree (value and gradient)."""
    from unflow_b200.e2eflow.core.supervised import flow_loss
    flow, gt, mask = _inputs(2, 24, 40, 96, 160, "invalid", seed=3)
    a = flow.cuda().requires_grad_(True)
    b = flow.cuda().requires_grad_(True)
    la = flow_loss(a, gt.cuda(), mask.cuda(), fused=True)
    lb = flow_loss(b, gt.cuda(), mask.cuda(), fused=False)
    _close(la, lb, rtol=1e-5)
    la.backward()
    lb.backward()
    _close(a.grad, b.grad, rtol=1e-4, atol_rel=1e-5)


def test_supervised_trainer_graph_and_prefetch_match_eager():
    from unflow_b200.e2eflow.core.train import Trainer
    params = dict(flownet='CS', train_all=True, learning_rate=1e-4)
    b1 = tuple(t.cuda() for t in usynth.supervised_batch(1, 128, 256, seed=4))
    b2 = tuple(t.cuda() for t in usynth.supervised_batch(1, 128, 256, seed=5))
    a = Trainer(params, synth.KITTI_NORMALIZATION, "cuda", seed=9, supervised=True)
    b = Trainer(params, synth.KITTI_NORMALIZATION, "cuda", seed=9, supervised=True)
    p0 = b.flat_param.clone()
    b.capture(*b1)
    assert torch.equal(b.flat_param, p0) and b.iteration == 0 and len(b._static) == 4
    la = [float(a.step(*b1)), float(a.step(*b2)), float(a.step(*b1))]
    lb = [float(b.step(*b1)), float(b.step(*b2)), float(b.step(*b1))]
    np.testing.assert_allclose(lb, la, rtol=2e-4)
    diff = (a.flat_param - b.flat_param).abs()
    assert float((diff > 2e-5).float().mean()) < 0.02, float((diff > 2e-5).float().mean())
    assert b.graph_replays == 3
    # prefetch / step_prefetched with the four pinned host tensors
    c = Trainer(params, synth.KITTI_NORMALIZATION, "cuda", seed=9, supervised=True)
    c.capture(*b1)
    c.prefetch(*(t.cpu().pin_memory() for t in b1))
    lc = [float(c.step_prefetched())]
    c.prefetch(*(t.cpu().pin_memory() for t in b2))
    lc.append(float(c.step_prefetched()))
    np.testing.assert_allclose(lc, la[:2], rtol=2e-4)
    with pytest.raises(ValueError):
        c.prefetch(b1[0].cpu(), b1[1].cpu())


CFG = """
[dirs]
log = {d}/log
checkpoints = {d}/log/checkpoints
data = {data}
[run]
batch_size = 2
gpu_list = 0
dataset = kitti_ft
development = False
[train]
learning_rate = 1.0e-4
decay_interval = 100000
save_interval = 2
display_interval = 1
flownet = CSS
train_all = True
[train_kitti_ft]
height = 64
width = 128
manual_decay_iters = 3,3
manual_decay_lrs = 0.5e-5,0.25e-5
"""


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_run_kitti_ft_synthetic(tmp_path, capsys, graph):
    from unflow_b200 import run as R
    ini = tmp_path / "config.ini"
    ini.write_text(CFG.format(d=str(tmp_path), data=str(tmp_path / "nodata")))
    R.main(["--ex", "ft", "--config", str(ini), "--synthetic", "--max-iters", "4"] + (["--graph"] if graph else []))
    out = capsys.readouterr().out
    assert "-- training from i = 1 to 4" in out and "-- train: i = 4, loss" in out
    ck = sorted(glob.glob(str(tmp_path / "log" / "checkpoints" / "ft" / "model.ckpt-*.pt")))
    assert [os.path.basename(c) for c in ck] == ["model.ckpt-2.pt", "model.ckpt-4.pt"]
    assert "stack_2_flownet/flownet_s/conv1/weights" in torch.load(ck[-1])["variables"]


def test_run_kitti_ft_on_a_kitti_tree_evaluates_on_2015(tmp_path, capsys):
    """Ground-truth batches from both KITTI training sets (41 pairs each: one left after the 40
    held out) and evaluation on the 40 held-out 2015 pairs after every save_interval chunk."""
    cv2 = pytest.importorskip("cv2")
    from unflow_b200 import run as R
    from unflow_b200.e2eflow.core import flow_io
    data = tmp_path / "data"
    rng = np.random.default_rng(0)
    base = cv2.GaussianBlur(rng.integers(0, 255, (80, 150, 3), dtype=np.uint8), (0, 0), 3)
    for top, imdir in (("data_scene_flow", "image_2"), ("data_stereo_flow", "colored_0")):
        tr = data / top / "training"
        for sub in (imdir, "flow_occ", "flow_noc"):
            (tr / sub).mkdir(parents=True)
        for i in range(41):
            im = np.roll(base, i, axis=1)
            cv2.imwrite(str(tr / imdir / ("%06d_10.png" % i)), im)
            cv2.imwrite(str(tr / imdir / ("%06d_11.png" % i)), np.roll(im, 2, axis=1))
            flow = np.full((80, 150, 2), 2.0, np.float32)
            valid = (rng.random((80, 150)) < 0.5).astype(np.float32)
            for sub in ("flow_occ", "flow_noc"):
                flow_io.write_kitti_flow(str(tr / sub / ("%06d_10.png" % i)), flow, valid)
    ini = tmp_path / "config.ini"
    ini.write_text(CFG.format(d=str(tmp_path), data=str(data)).replace("flownet = CSS", "flownet = C"))
    R.main(["--ex", "ftk", "--config", str(ini), "--max-iters", "2"])
    out = capsys.readouterr().out
    assert "-- train: i = 2, loss" in out and "-- eval: i = 2" in out
    assert "num_examples = 40" in out and "AEE/occluded" in out
    assert os.path.exists(str(tmp_path / "log" / "checkpoints" / "ftk" / "model.ckpt-2.pt"))
