"""The training and evaluation geometries of FlyingChairs (384x512), SYNTHIA (512x768), Cityscapes /
Sintel (512x1024) and Middlebury (512x640) on the GPU: no kernel changes for them, so this checks
the existing shape-generic kernels there against the CPU oracle, and runs ``unflow_b200.run`` /
``unflow_b200.eval`` end to end on generated dataset trees at the real frame sizes.

Tolerances as in test_gpu_baseline_sizes: loss 2e-4 relative, flows 1e-4 of the maximum magnitude,
per-variable gradient L2 1e-2 (hard occlusion masks make gradients jump by O(1/pixels))."""
import glob
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import flownet as oflownet
from oracle import unsupervised as ounsup
import synth

BASE_PARAMS = dict(flownet='C', pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0)
# config_template/config.ini: [train_chairs] / [train_synthia] keep [train]'s loss, [train_cityscapes]
# adds the forward-backward consistency terms
DATASET_PARAMS = {'chairs': BASE_PARAMS, 'synthia': BASE_PARAMS,
                  'cityscapes': dict(BASE_PARAMS, fb_weight=0.2, mask_occlusion='fb', occ_weight=12.4)}


def rel_err(got, want):
    want = want.detach().cpu().double()
    got = got.detach().cpu().double()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-12))


@pytest.fixture(scope="module")
def modes():
    from unflow_b200.e2eflow.core import conv_ops
    prev = conv_ops.get_mode()
    yield conv_ops
    conv_ops.set_mode(prev)


@pytest.mark.parametrize("dataset,hw", [("chairs", (384, 512)), ("synthia", (512, 768)), ("cityscapes", (512, 1024))])
def test_flownet_c_training_loss_at_dataset_sizes(dataset, hw, modes):
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.e2eflow.core.unsupervised import unsupervised_loss
    params = DATASET_PARAMS[dataset]
    tfv = oflownet.init_variables('C', False, seed=19)
    for k in tfv:
        tfv[k] = tfv[k].clone().requires_grad_(True)
    im1, im2, _ = synth.image_pair(1, hw[0], hw[1], seed=37)
    want_loss, want_fw, want_bw = ounsup.unsupervised_loss(tfv, (im1, im2), params, synth.KITTI_NORMALIZATION,
                                                           augment=False, return_flow=True)
    want_loss.backward()
    report = {}
    for mode in ("fp32", "3xtf32"):
        modes.set_mode(mode)
        v = FlowNetVariables('C', False, seed=0).load_tf_dict({k: t.detach() for k, t in tfv.items()}).cuda()
        got_loss, got_fw, got_bw = unsupervised_loss((im1.cuda(), im2.cuda()), params, synth.KITTI_NORMALIZATION,
                                                     augment=False, return_flow=True, variables=v)
        got_loss.backward()
        e_loss = abs(float(got_loss) - float(want_loss)) / abs(float(want_loss))
        worst_g, worst_name = 0.0, ""
        for scope in v.kinds:
            w, b = v.weights(scope)
            for got, want, nm in ((w.grad.cpu(), tfv[scope + '/weights'].grad.permute(3, 2, 0, 1), '/weights'),
                                  (b.grad.cpu(), tfv[scope + '/biases'].grad, '/biases')):
                e = float((got - want).norm() / want.norm().clamp_min(1e-20))
                if e > worst_g:
                    worst_g, worst_name = e, scope + nm
        report[mode] = (e_loss, rel_err(got_fw, want_fw), rel_err(got_bw, want_bw), worst_g)
        print("%s %s %s: loss rel %.2e, flow_fw %.2e, flow_bw %.2e, worst grad L2 %.2e (%s)"
              % (dataset, hw, mode, *report[mode], worst_name))
    for mode, (e_loss, e_fw, e_bw, worst_g) in report.items():
        assert e_loss < 2e-4, (mode, e_loss)
        assert e_fw < 1e-4 and e_bw < 1e-4, (mode, e_fw, e_bw)
        assert worst_g < 1e-2, (mode, worst_g)


@pytest.mark.parametrize("file_hw,dims", [((436, 1024), (512, 1024)), ((388, 584), (512, 640))])
def test_evaluation_path_at_sintel_and_middlebury_sizes(file_hw, dims, modes):
    """resize_input -> FlowNetC -> resize_output_flow, as eval.evaluate_examples runs it."""
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.e2eflow.core.input import resize_image_with_crop_or_pad, resize_input, resize_output_flow
    from unflow_b200.eval import network_flow_fn
    h, w = file_hw
    params = dict(synth.KITTI_PARAMS)
    tfv = oflownet.init_variables('C', False, seed=29)
    raw1, raw2, _ = synth.image_pair(1, h, w, seed=43)
    # what the input classes deliver: the file-size frame cropped / padded to the network size
    items = [resize_image_with_crop_or_pad(r[0], *dims).unsqueeze(0) for r in (raw1, raw2)]
    a, b = (resize_input(t, h, w, *dims) for t in items)
    with torch.no_grad():
        _, want_fw, want_bw = ounsup.unsupervised_loss(tfv, (a, b), params, synth.KITTI_NORMALIZATION,
                                                       augment=False, return_flow=True)
    want_fw, want_bw = resize_output_flow(want_fw, h, w), resize_output_flow(want_bw, h, w)
    for mode in ("fp32", "3xtf32"):
        modes.set_mode(mode)
        v = FlowNetVariables('C', False, seed=0).load_tf_dict(tfv).cuda()
        fn = network_flow_fn(params, synth.KITTI_NORMALIZATION, v)
        ga, gb = (resize_input(t.cuda(), h, w, *dims) for t in items)
        got_fw, got_bw = fn(ga, gb)
        got_fw, got_bw = resize_output_flow(got_fw, h, w), resize_output_flow(got_bw, h, w)
        assert tuple(got_fw.shape) == (1, h, w, 2)
        e_fw, e_bw = rel_err(got_fw, want_fw), rel_err(got_bw, want_bw)
        print("eval %s at %s %s: flow_fw %.2e, flow_bw %.2e" % (file_hw, dims, mode, e_fw, e_bw))
        assert e_fw < 1e-4 and e_bw < 1e-4, (mode, e_fw, e_bw)


# ---- end to end on generated trees ----------------------------------------------------------------
CFG = """
[dirs]
log = {d}/log
checkpoints = {d}/log/checkpoints
data = {d}/data
[run]
batch_size = 2
gpu_list = 0
num_input_threads = 2
dataset = {dataset}
development = True
[train]
decay_interval = 100000
save_interval = 1
display_interval = 1
flownet = C
pyramid_loss = True
border_mask = True
ternary_weight = 1.0
smooth_2nd_weight = 3.0
[train_chairs]
height = 384
width = 512
num_iters = 600000
learning_rate = 1.0e-4
decay_after = 200000
[train_synthia]
height = 512
width = 768
num_iters = 500000
learning_rate = 1.0e-4
decay_after = 100000
[train_cityscapes]
height = 512
width = 1024
num_iters = 500000
learning_rate = 1.0e-5
decay_after = 100000
fb_weight = 0.2
mask_occlusion = fb
occ_weight = 12.4
"""


def _png(path, im):
    import cv2
    os.makedirs(os.path.dirname(path), exist_ok=True)
    assert cv2.imwrite(path, np.ascontiguousarray(im.clamp(0, 255).byte().numpy()[:, :, ::-1]))


def _frames(h, w, n, seed):
    """``n`` consecutive frames of a synthetic sequence (each the previous one moved by a smooth flow)."""
    out = []
    for i in range(0, n, 2):
        a, b, _ = synth.image_pair(1, h, w, seed=seed + i)
        out += [a[0], b[0]]
    return out[:n]


@pytest.fixture(scope="module")
def trees(tmp_path_factory):
    from unflow_b200.e2eflow.core import flow_io
    root = tmp_path_factory.mktemp("datasets")
    data = str(root / "data")
    j = os.path.join
    # FlyingChairs: 384x512 training pairs in image/, validation pairs + .flo in test_image/, flow/
    for i in range(3):
        a, b, f = synth.image_pair(1, 384, 512, seed=100 + i)
        _png(j(data, 'flying_chairs', 'image', '%05d_img1.png' % i), a[0])
        _png(j(data, 'flying_chairs', 'image', '%05d_img2.png' % i), b[0])
    for i in range(2):
        a, b, f = synth.image_pair(1, 384, 512, seed=200 + i)
        _png(j(data, 'flying_chairs', 'test_image', '%05d_img1.png' % i), a[0])
        _png(j(data, 'flying_chairs', 'test_image', '%05d_img2.png' % i), b[0])
        os.makedirs(j(data, 'flying_chairs', 'flow'), exist_ok=True)
        flow_io.write_flo(j(data, 'flying_chairs', 'flow', '%05d_flow.flo' % i), f[0].numpy())
    # SYNTHIA: 760x1280 frames, one sequence, two views
    seq = 'SYNTHIA-SEQS-01-SUMMER'
    for v, view in enumerate(('Omni_F', 'Omni_B')):
        for i, im in enumerate(_frames(760, 1280, 3, 300 + 10 * v)):
            _png(j(data, 'synthia', seq, seq, 'RGB', 'Stereo_Left', view, '%06d.png' % i), im)
    # Cityscapes: 1024x2048 frames of one city, one snippet
    for i, im in enumerate(_frames(1024, 2048, 3, 400)):
        _png(j(data, 'cs', 'leftImg8bit_sequence_trainvaltest', 'train', 'aachen',
               'aachen_000000_%06d_leftImg8bit.png' % (17 + i)), im)
    # Sintel: 436x1024 training sequence with flow, 0/255 invalid and occlusion masks
    frames = _frames(436, 1024, 3, 500)
    for pas in ('clean', 'final'):
        for i, im in enumerate(frames):
            _png(j(data, 'sintel', 'training', pas, 'alley_1', 'frame_%04d.png' % (i + 1)), im)
    for i in range(3):
        mask = np.zeros((436, 1024), np.uint8)
        mask[:, :10 + i] = 255
        import cv2
        for sub in ('invalid',) + (('occlusions',) if i < 2 else ()):
            os.makedirs(j(data, 'sintel', 'training', sub, 'alley_1'), exist_ok=True)
            cv2.imwrite(j(data, 'sintel', 'training', sub, 'alley_1', 'frame_%04d.png' % (i + 1)), mask)
        if i < 2:
            os.makedirs(j(data, 'sintel', 'training', 'flow', 'alley_1'), exist_ok=True)
            flow = synth.image_pair(1, 436, 1024, seed=510 + i)[2][0].numpy()
            flow_io.write_flo(j(data, 'sintel', 'training', 'flow', 'alley_1', 'frame_%04d.flo' % (i + 1)), flow)
    # Middlebury: one 388x584 pair with ground truth
    a, b, f = synth.image_pair(1, 388, 584, seed=600)
    _png(j(data, 'middlebury', 'other-data', 'Grove2', 'frame10.png'), a[0])
    _png(j(data, 'middlebury', 'other-data', 'Grove2', 'frame11.png'), b[0])
    os.makedirs(j(data, 'middlebury', 'other-gt-flow', 'Grove2'))
    flow_io.write_flo(j(data, 'middlebury', 'other-gt-flow', 'Grove2', 'flow10.flo'), f[0].numpy())
    # KITTI 2012 training set the runs evaluate on: two 375x1242 pairs
    tr = j(data, 'data_stereo_flow', 'training')
    for i in range(2):
        a, b, f = synth.image_pair(1, 375, 1242, seed=700 + i)
        _png(j(tr, 'colored_0', '%06d_10.png' % i), a[0])
        _png(j(tr, 'colored_0', '%06d_11.png' % i), b[0])
        for sub in ('flow_occ', 'flow_noc'):
            os.makedirs(j(tr, sub), exist_ok=True)
            flow_io.write_kitti_flow(j(tr, sub, '%06d_10.png' % i), f[0].numpy())
    return root


@pytest.mark.parametrize("dataset", ["chairs", "synthia", "cityscapes"])
def test_run_and_eval_end_to_end(dataset, trees, capsys):
    from unflow_b200 import eval as E
    from unflow_b200 import run as R
    ini = trees / ("config_%s.ini" % dataset)
    ini.write_text(CFG.format(d=str(trees), dataset=dataset))
    ex = 'e2e_' + dataset
    R.main(["--ex", ex, "--config", str(ini), "--max-iters", "2"])
    out = capsys.readouterr().out
    losses = [float(l.split("loss = ")[1]) for l in out.splitlines() if l.startswith("-- train: i = ")]
    assert len(losses) == 2 and all(math.isfinite(x) for x in losses), out
    assert "-- eval: i = 1" in out and "-- eval: i = 2" in out and "num_examples = 2" in out, out
    ck = sorted(os.path.basename(p) for p in glob.glob(str(trees / "log" / "checkpoints" / ex / "model.ckpt-*.pt")))
    assert ck == ["model.ckpt-1.pt", "model.ckpt-2.pt"]
    for ds, variant, n in (("chairs", "test", 2), ("sintel", "train_clean", 2), ("mdb", "train", 1)):
        res = E.main(["--dataset", ds, "--variant", variant, "--ex", ex, "--num", "-1", "--config", str(ini),
                      "--out", str(trees / "out")])
        metrics = res[ex]
        want = {'EPE_noc', 'EPE_all', 'outliers_noc', 'outliers_all'} if ds == 'sintel' else {'EPE_all'}
        assert set(metrics) == want and all(math.isfinite(v) for v in metrics.values()), (ds, metrics)
        print("%s -> %s/%s: %s" % (dataset, ds, variant, metrics))
        assert ("-- evaluating: on -1 pairs from %s/%s" % (ds, variant)) in capsys.readouterr().out
