"""Evaluation pages on the H100: ``eval --output_pages`` end to end on generated KITTI 2015, Sintel and
FlyingChairs trees with two experiments of different weights, ``[run] interactive_plot`` in training,
and the copies and launches the pages add to the evaluation loops (none when they are off)."""
import glob
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

import synth
from unflow_b200.e2eflow.core import flow_io, flow_util, pages

KITTI_SLOTS = ['overlay', 'brightness error', 'flow', 'flow error']
GT_SLOTS = ['overlay', 'brightness error', 'flow', 'gt']
TRAIN_SLOTS = ['warped image', 'flow', 'occ', 'reverse disocc', 'flow error']
LOSS = ("flownet = C\npyramid_loss = True\nborder_mask = True\nternary_weight = 1.0\nsmooth_2nd_weight = 3.0\n"
        "fb_weight = 0.2\nmask_occlusion = fb\nocc_weight = 12.4\n")


def read_rgb(path):
    im = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    assert im is not None, path
    return np.ascontiguousarray(im[:, :, ::-1])


def tiles_of(page, rows, ncols, h, w):
    origins = pages.layout('', rows, ncols, h, w)[2]
    return [[page[y:y + h, x:x + w] for (y, x) in row] for row in origins]


def _png(path, im):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    assert cv2.imwrite(path, np.ascontiguousarray(im.clamp(0, 255).byte().numpy()[:, :, ::-1]))


@pytest.fixture(scope="module")
def trees(tmp_path_factory):
    """KITTI 2015 training (two 375x1242 pairs), Sintel training (two 436x1024 pairs with flow, invalid
    and occlusion maps) and FlyingChairs validation (two 384x512 pairs), and experiments wA and wB: FlowNetC
    checkpoints of different weights."""
    from unflow_b200.e2eflow.core import tf_checkpoint as ck
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    root = tmp_path_factory.mktemp("pages")
    data = str(root / "data")
    j = os.path.join
    tr = j(data, 'data_scene_flow', 'training')
    for i in range(2):
        a, b, f = synth.image_pair(1, 375, 1242, seed=800 + i)
        _png(j(tr, 'image_2', '%06d_10.png' % i), a[0])
        _png(j(tr, 'image_2', '%06d_11.png' % i), b[0])
        noc = np.ones((375, 1242))
        noc[:, :300] = 0
        for sub, mask in (('flow_occ', np.ones((375, 1242))), ('flow_noc', noc)):
            os.makedirs(j(tr, sub), exist_ok=True)
            flow_io.write_kitti_flow(j(tr, sub, '%06d_10.png' % i), f[0].numpy(), mask)
    frames = []
    for i in range(0, 3, 2):
        a, b, _ = synth.image_pair(1, 436, 1024, seed=900 + i)
        frames += [a[0], b[0]]
    for i, im in enumerate(frames[:3]):
        _png(j(data, 'sintel', 'training', 'clean', 'alley_1', 'frame_%04d.png' % (i + 1)), im)
    for i in range(3):
        mask = np.zeros((436, 1024), np.uint8)
        mask[:, :10 + i] = 255
        for sub in ('invalid',) + (('occlusions',) if i < 2 else ()):
            os.makedirs(j(data, 'sintel', 'training', sub, 'alley_1'), exist_ok=True)
            cv2.imwrite(j(data, 'sintel', 'training', sub, 'alley_1', 'frame_%04d.png' % (i + 1)), mask)
        if i < 2:
            os.makedirs(j(data, 'sintel', 'training', 'flow', 'alley_1'), exist_ok=True)
            flow = synth.image_pair(1, 436, 1024, seed=910 + i)[2][0].numpy()
            flow_io.write_flo(j(data, 'sintel', 'training', 'flow', 'alley_1', 'frame_%04d.flo' % (i + 1)), flow)
    os.makedirs(j(data, 'flying_chairs', 'image'))
    os.makedirs(j(data, 'flying_chairs', 'flow'))
    for i in range(2):
        a, b, f = synth.image_pair(1, 384, 512, seed=950 + i)
        _png(j(data, 'flying_chairs', 'test_image', '%05d_img1.png' % i), a[0])
        _png(j(data, 'flying_chairs', 'test_image', '%05d_img2.png' % i), b[0])
        flow_io.write_flo(j(data, 'flying_chairs', 'flow', '%05d_flow.flo' % i), f[0].numpy())
    (root / "config.ini").write_text("[dirs]\nlog = %s/log\ncheckpoints = %s/ckpts\ndata = %s\n[run]\nbatch_size = 4\n"
                                     "[train]\n%s" % (root, root, data, LOSS))
    for seed, name in ((11, 'wA'), (12, 'wB')):
        ck.save_variables(FlowNetVariables('C', False, seed=seed), str(root / "ckpts" / name / "model.ckpt-1"))
    return root


@pytest.mark.parametrize("dataset,variant,slots,hw", [("kitti", "train_2015", KITTI_SLOTS, (375, 1242)),
                                                      ("sintel", "train_clean", KITTI_SLOTS, (436, 1024)),
                                                      ("chairs", "test", GT_SLOTS, (384, 512))])
def test_eval_pages_show_flow_util_of_the_computed_flows(trees, dataset, variant, slots, hw):
    """The flows eval computed are read back from its exact ``.flo`` output; the page's flow and flow
    error (or gt) tiles must be ``flow_util`` of them, converted with ``to_uint8``."""
    from unflow_b200 import eval as E
    from unflow_b200.e2eflow.core.input import resize_image_with_crop_or_pad
    out = trees / ("out_" + dataset)
    E.main(["--dataset", dataset, "--variant", variant, "--ex", "wA,wB", "--num", "2", "--output_pages",
            "--output_benchmark", "--no-output_png", "--config", str(trees / "config.ini"), "--out", str(out)])
    h, w = hw
    assert sorted(os.listdir(out / "pages")) == ["000000.png", "000001.png"]
    data_input, input_fn = E.dataset_input(dataset, variant, str(trees / "data"))
    for i, item in enumerate(input_fn()):
        page = read_rgb(str(out / "pages" / ("%06d.png" % i)))
        title = "Flow eval: %s/%s %06d" % (dataset, variant, i)
        assert page.shape[:2] == pages.layout(title, slots, 2, h, w)[:2]
        grid = tiles_of(page, slots, 2, h, w)
        truth = [resize_image_with_crop_or_pad(t[0].cuda(), h, w).unsqueeze(0) for t in item[3:]]
        flows = []
        for c, name in enumerate(("wA", "wB")):
            flow = torch.from_numpy(flow_io.read_flo(str(out / name / ("%06d_10.flo" % i)))[0]).cuda()[None]
            flows.append(flow)
            want_flow = pages.to_uint8(flow_util.flow_to_color(flow) * 255)[0].cpu().numpy()
            assert np.array_equal(grid[2][c], want_flow), (dataset, i, name, 'flow')
            if len(truth) == 4:
                last = flow_util.flow_error_image(flow, truth[0], truth[1], truth[3])
            else:
                last = flow_util.flow_to_color(truth[0], truth[1])
            want_last = pages.to_uint8(last * 255)[0].cpu().numpy()
            assert np.array_equal(grid[3][c], want_last), (dataset, i, name, slots[3])
        # the experiments' weights differ, and so do their flows and flow tiles; the overlay is the same
        assert not torch.equal(flows[0], flows[1]) and not np.array_equal(grid[2][0], grid[2][1])
        assert np.array_equal(grid[0][0], grid[0][1])


# ---- [run] interactive_plot ------------------------------------------------------------------------
RUN_CFG = """
[dirs]
log = {d}/log
checkpoints = {d}/log/checkpoints
data = {d}/data
[run]
batch_size = 2
gpu_list = {gpus}
dataset = kitti
development = False
{plot}
[train]
decay_interval = 100000
save_interval = 2
display_interval = 1
flownet = C
pyramid_loss = True
border_mask = True
ternary_weight = 1.0
smooth_2nd_weight = 3.0
[train_kitti]
height = 128
width = 256
num_iters = 6
learning_rate = 1.0e-5
decay_after = 100000
fb_weight = 0.2
mask_occlusion = fb
occ_weight = 12.4
"""
EVAL_HW = (120, 280)


@pytest.fixture(scope="module")
def kitti_tree(tmp_path_factory):
    """KITTI raw sequence frames to train on and a KITTI 2012 training set of two 120x280 pairs."""
    root = tmp_path_factory.mktemp("plot")
    data = root / "data"
    rng = np.random.default_rng(0)
    base = cv2.GaussianBlur(rng.integers(0, 255, (150, 300, 3), dtype=np.uint8), (0, 0), 3)
    for view in ("image_02", "image_03"):
        d = data / "kitti_raw" / "2011_09_26" / "2011_09_26_drive_0001_extract" / view / "data"
        d.mkdir(parents=True)
        for n in range(6):
            assert cv2.imwrite(str(d / ("%010d.png" % n)), np.roll(base, 2 * n, axis=1))
    tr = data / "data_stereo_flow" / "training"
    for sub in ("colored_0", "flow_occ", "flow_noc"):
        (tr / sub).mkdir(parents=True)
    for i in range(2):
        im = np.roll(base, 5 * i, axis=0)[:120, :280]
        cv2.imwrite(str(tr / "colored_0" / ("%06d_10.png" % i)), im)
        cv2.imwrite(str(tr / "colored_0" / ("%06d_11.png" % i)), np.roll(im, 3, axis=1))
        flow = np.zeros((120, 280, 2), np.float32)
        flow[..., 0] = 3.0
        for sub in ("flow_occ", "flow_noc"):
            flow_io.write_kitti_flow(str(tr / sub / ("%06d_10.png" % i)), flow, np.ones((120, 280)))
    return root


def _ini(root, name, plot, gpus="0"):
    ini = root / ("%s.ini" % name)
    ini.write_text(RUN_CFG.format(d=str(root), gpus=gpus, plot=plot))
    return str(ini)


def check_pages(page_dir, ex, iteration):
    """One page per evaluated pair, laid out and titled as ``render`` does for this evaluation."""
    files = sorted(os.listdir(page_dir))
    assert files == ["000000.png", "000001.png"], files
    h, w = EVAL_HW
    for f in files:
        page = read_rgb(os.path.join(page_dir, f))
        title = "%s (i=%d)" % (ex, iteration)
        assert page.shape[:2] == pages.layout(title, TRAIN_SLOTS, 1, h, w)[:2]
        grid = tiles_of(page, TRAIN_SLOTS, 1, h, w)
        assert np.array_equal(page, pages.render(title, TRAIN_SLOTS, [ex], grid)), (f, title)
        for r in (2, 3):        # occ and reverse disocc: binary masks, drawn gray
            t = grid[r][0]
            assert set(np.unique(t).tolist()) <= {0, 255} and (t == t[:, :, :1]).all()


def test_interactive_plot_writes_each_evaluation_and_replaces_the_last(kitti_tree, capsys):
    from unflow_b200 import run as R
    ini = _ini(kitti_tree, "plot", "interactive_plot = True")
    page_dir = kitti_tree / "log" / "ex" / "p1" / "eval_pages"
    R.main(["--ex", "p1", "--config", ini, "--max-iters", "2"])
    assert "-- eval: i = 2" in capsys.readouterr().out
    check_pages(str(page_dir), "p1", 2)
    (page_dir / "stale").write_text("from the first evaluation")
    # resumed with --debug, which writes the pages too: the evaluation at i = 4 replaces them
    R.main(["--ex", "p1", "--config", ini, "--max-iters", "4", "--debug"])
    assert "-- eval: i = 4" in capsys.readouterr().out
    check_pages(str(page_dir), "p1", 4)
    assert not os.path.exists(str(page_dir) + ".partial")
    # without the key the directory never appears
    R.main(["--ex", "p2", "--config", _ini(kitti_tree, "noplot", ""), "--max-iters", "2"])
    assert "-- eval: i = 2" in capsys.readouterr().out
    assert os.path.isdir(kitti_tree / "log" / "ex" / "p2")
    assert not glob.glob(str(kitti_tree / "log" / "ex" / "p2" / "eval_pages*"))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_interactive_plot_data_parallel_rank_0_writes(kitti_tree):
    from unflow_b200 import run as R
    R.main(["--ex", "p_dp", "--config", _ini(kitti_tree, "plot_dp", "interactive_plot = True", gpus="0,1"),
            "--max-iters", "2"])
    check_pages(str(kitti_tree / "log" / "ex" / "p_dp" / "eval_pages"), "p_dp", 2)


# ---- what the pages add to the evaluation loops ------------------------------------------------------
def profile_counts(make, reps=3):
    """(device-to-host copies, kernels) of the GPU work ``make()`` runs, from torch.profiler: per count, the
    median of ``reps`` sessions, each running a fresh ``make()`` (a page collector fills up).  A session can
    miss activities issued right at its start, or take in records of the work before it; the median is the
    count of a session that did neither."""
    runs = [_profile_once(make()) for _ in range(reps)]
    return tuple(sorted(c)[reps // 2] for c in zip(*runs))


def _profile_once(fn):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    dev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    copies = sum(1 for e in dev if e.name.startswith("Memcpy DtoH"))
    kernels = sum(1 for e in dev if not e.name.startswith(("Memcpy", "Memset")))
    return copies, kernels


def test_pages_add_one_copy_per_paged_example_and_nothing_when_off(trees):
    from unflow_b200 import eval as E
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.e2eflow.core.input import resize_image_with_crop_or_pad
    from unflow_b200.e2eflow.core.train import evaluate
    v = FlowNetVariables('C', False, seed=3).cuda()
    data_input, input_fn = E.dataset_input("kitti", "train_2015", str(trees / "data"))
    items = list(input_fn())
    fn = E.network_flow_fn(dict(synth.KITTI_PARAMS), synth.KITTI_NORMALIZATION, v)

    def eval_loop(collector):
        return lambda: E.evaluate_examples("w", items, data_input.dims, fn, torch.device("cuda"), num=2,
                                           pages=collector, log=open(os.devnull, "w"))
    eval_loop(pages.Tiles(2))()        # warm-up of every shape
    off, idle, on = (profile_counts(lambda k=k: eval_loop(None if k is None else pages.Tiles(k))) for k in (None, 0, 1))
    print("eval loop, 2 pairs: (copies, kernels) off %s, collector full %s, one page %s" % (off, idle, on))
    assert idle == off
    assert on[0] == off[0] + 1 and on[1] > off[1]

    examples = []
    for item in items:
        h, w = int(item[2][0, 0]), int(item[2][0, 1])
        examples.append(tuple(resize_image_with_crop_or_pad(t[0], h, w).unsqueeze(0).cuda()
                              for t in (item[0], item[1]) + item[3:]))

    def train_eval(collector):
        return lambda: evaluate(v, dict(synth.KITTI_PARAMS), synth.KITTI_NORMALIZATION, examples, pages=collector)
    train_eval(pages.Tiles())()
    off, on = profile_counts(lambda: train_eval(None)), profile_counts(lambda: train_eval(pages.Tiles()))
    print("training evaluation, 2 pairs: (copies, kernels) off %s, pages %s" % (off, on))
    assert on[0] == off[0] + 2 and on[1] > off[1]
    collected = pages.Tiles()
    res, images = evaluate(v, dict(synth.KITTI_PARAMS), synth.KITTI_NORMALIZATION, examples, pages=collected)
    assert collected.names == TRAIN_SLOTS and len(collected.examples) == 2
    assert [t.shape[2] for t in collected.examples[1]] == [3, 3, 1, 1, 3]
    for name, t in zip(collected.names, collected.examples[1]):       # the last example's tensors, converted
        assert np.array_equal(t, pages.to_uint8(images[name] * 255)[0].cpu().numpy()), name
