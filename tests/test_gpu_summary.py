"""TensorBoard summaries of ``python -m unflow_b200.run`` on the GPU: the train and eval event files
read back with tensorboard's own reader, their values against the printed loss and an eager
``unsupervised_loss`` on the same batch, and the launches and copies a display step adds to the
captured step (torch.profiler with CUDA activity)."""
import json
import os
import re

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_summaries.json")))

CFG = """
[dirs]
log = {d}/log
checkpoints = {d}/log/checkpoints
data = {data}
[run]
batch_size = 2
gpu_list = 0
dataset = {dataset}
development = False
[train]
decay_interval = 100000
save_interval = 4
display_interval = 2
flownet = C
pyramid_loss = True
border_mask = True
ternary_weight = 1.0
smooth_2nd_weight = 3.0
[train_kitti]
height = 128
width = 256
num_iters = 100
learning_rate = 1.0e-5
decay_after = 100000
fb_weight = 0.2
mask_occlusion = fb
occ_weight = 12.4
[train_kitti_ft]
height = 64
width = 128
manual_decay_iters = 50,50
manual_decay_lrs = 0.5e-5,0.25e-5
"""


def _acc(path):
    from tensorboard.backend.event_processing import event_accumulator as ea
    acc = ea.EventAccumulator(str(path), size_guidance={ea.SCALARS: 0, ea.IMAGES: 0})
    acc.Reload()
    return acc


def _printed_losses(out):
    return {int(i): float(v) for i, v in re.findall(r"-- train: i = (\d+), loss = (\S+)", out)}


def _expected_train_scalars(config):
    return [t for kind, t in GOLDEN["configs"][config]["train_summaries"] if kind == "scalar"]


def _kitti_tree(root, n_eval=2):
    """KITTI raw sequences and a KITTI 2012 training set with ground truth (as test_gpu_run.py)."""
    cv2 = pytest.importorskip("cv2")
    from unflow_b200.e2eflow.core import flow_io
    rng = np.random.default_rng(0)
    base = cv2.GaussianBlur(rng.integers(0, 255, (150, 300, 3), dtype=np.uint8), (0, 0), 3)
    for view in ("image_02", "image_03"):
        d = root / "kitti_raw" / "2011_09_26" / "2011_09_26_drive_0001_extract" / view / "data"
        d.mkdir(parents=True)
        for n in range(6):
            assert cv2.imwrite(str(d / ("%010d.png" % n)), np.roll(base, 2 * n, axis=1))
    tr_dir = root / "data_stereo_flow" / "training"
    for sub in ("colored_0", "flow_occ", "flow_noc"):
        (tr_dir / sub).mkdir(parents=True)
    for i in range(n_eval):
        im = np.roll(base, 5 * i, axis=0)[:120, :280]
        cv2.imwrite(str(tr_dir / "colored_0" / ("%06d_10.png" % i)), im)
        cv2.imwrite(str(tr_dir / "colored_0" / ("%06d_11.png" % i)), np.roll(im, 3, axis=1))
        flow = np.zeros((120, 280, 2), np.float32)
        flow[..., 0] = 3.0
        for sub in ("flow_occ", "flow_noc"):
            flow_io.write_kitti_flow(str(tr_dir / sub / ("%06d_10.png" % i)), flow, np.ones((120, 280)))


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
def test_run_writes_train_summaries_synthetic(tmp_path, capsys, graph):
    from unflow_b200 import run as R
    from unflow_b200 import synthetic
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.e2eflow.core import unsupervised as U
    ini = tmp_path / "config.ini"
    ini.write_text(CFG.format(d=tmp_path, data=tmp_path / "nodata", dataset="kitti"))
    # two display intervals (steps 1, 2, 4) and one save interval (4); no augmentation, so step 1 can be
    # recomputed from the initial weights
    R.main(["--ex", "s", "--config", str(ini), "--synthetic", "--no-augment", "--max-iters", "4"]
           + (["--graph"] if graph else []))
    printed = _printed_losses(capsys.readouterr().out)
    assert sorted(printed) == [1, 2, 4]
    acc = _acc(tmp_path / "log" / "ex" / "s" / "train")
    want_tags = _expected_train_scalars("train_kitti")
    assert sorted(acc.Tags()["scalars"]) == sorted(want_tags)
    assert acc.Tags()["images"] == []                          # image summaries only with --debug
    for tag in want_tags:
        assert [e.step for e in acc.Scalars(tag)] == [1, 2, 4], tag
    for i, loss in printed.items():
        (ev,) = [e for e in acc.Scalars("loss/combined_1") if e.step == i]
        assert np.float32(ev.value) == np.float32(loss), (i, ev.value, loss)
    assert [e.value for e in acc.Scalars("params/train/learning_rate")] == [np.float32(1e-5)] * 3
    assert acc.Scalars("weight/occ_1")[0].value == np.float32(12.4)
    # step 1 against an eager unsupervised_loss on the same batch with the initial weights
    params = R.config_dict(str(ini))
    p = dict(params["train"], **params["train_kitti"])
    v = FlowNetVariables('C', None, seed=1234).cuda()
    batch = R.synthetic_batch(2, 128, 256, 1, 0, torch.device("cuda"))
    with torch.no_grad():
        U.unsupervised_loss(batch, p, R.KITTI_NORMALIZATION, augment=False, variables=v)
    from unflow_b200.e2eflow.core.train import read_scalars
    from unflow_b200.e2eflow.core.summary import train_tags
    want = read_scalars(U.tracked)
    tags = train_tags(U.tracked)["losses"]
    for name, value in want.items():
        (ev,) = [e for e in acc.Scalars(tags[name]) if e.step == 1]
        assert abs(ev.value - value) <= 2e-4 * max(abs(value), 1e-6), (name, ev.value, value)


def test_run_writes_eval_summaries_on_a_kitti_tree(tmp_path, capsys):
    from unflow_b200 import run as R
    data = tmp_path / "data"
    _kitti_tree(data)
    ini = tmp_path / "config.ini"
    ini.write_text(CFG.format(d=tmp_path, data=data, dataset="kitti"))
    R.main(["--ex", "k", "--config", str(ini), "--max-iters", "4"])
    out = capsys.readouterr().out
    assert "-- eval: i = 4" in out
    printed = {k: float(v) for k, v in re.findall(r"   (\S+) = (\S+)", out)}
    acc = _acc(tmp_path / "log" / "ex" / "k" / "eval")
    want = [t for _, t in GOLDEN["configs"]["train_kitti"]["eval_summaries"]]
    assert sorted(acc.Tags()["scalars"]) == sorted(want)
    for name in ("AEE/occluded", "outliers/occluded", "AEE/non-occluded", "outliers/non-occluded"):
        (ev,) = acc.Scalars(name + "_1")
        assert ev.step == 4 and np.float32(ev.value) == np.float32(printed[name]), name
    assert all(np.isfinite(acc.Scalars(t)[0].value) for t in want)
    assert sorted(_acc(tmp_path / "log" / "ex" / "k" / "train").Tags()["scalars"]) == \
        sorted(_expected_train_scalars("train_kitti"))
    # --ow removes the experiment's summaries with it (one step: save_interval shrinks to 1)
    R.main(["--ex", "k", "--config", str(ini), "--max-iters", "1", "--ow", "--debug"])
    capsys.readouterr()
    assert [e.step for e in _acc(tmp_path / "log" / "ex" / "k" / "train").Scalars("loss/combined_1")] == [1]
    assert [e.step for e in _acc(tmp_path / "log" / "ex" / "k" / "eval").Scalars("AEE/occluded_1")] == [1]


def test_run_kitti_ft_writes_summaries_and_images(tmp_path, capsys):
    """kitti_ft with --debug on a generated KITTI tree: the supervised scalars and images in train, the
    evaluation on the held-out 2015 pairs in eval."""
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
    ini.write_text(CFG.format(d=tmp_path, data=data, dataset="kitti_ft"))
    R.main(["--ex", "ft", "--config", str(ini), "--max-iters", "4", "--debug", "--graph"])
    out = capsys.readouterr().out
    printed = _printed_losses(out)
    assert sorted(printed) == [1, 2, 4] and "-- eval: i = 4" in out
    acc = _acc(tmp_path / "log" / "ex" / "ft" / "train")
    assert sorted(acc.Tags()["scalars"]) == ["loss/combined_1", "loss/regularization_1", "params/train/learning_rate"]
    for i, loss in printed.items():
        (ev,) = [e for e in acc.Scalars("loss/combined_1") if e.step == i]
        assert np.float32(ev.value) == np.float32(loss)
    # flownet C: one network, flow_pred_0; batch 2 -> images 0 and 1 of every tracked batch
    want_images = sorted("%s_1/image/%d" % (n, k) for n in ("train/im1_photo", "train/im2_photo", "train/flow_gt",
                                                            "train/mask_gt", "train/flow_pred_0") for k in (0, 1))
    assert sorted(acc.Tags()["images"]) == want_images
    for tag in want_images:
        evs = acc.Images(tag)
        assert [e.step for e in evs] == [1, 2, 4]
        assert (evs[0].height, evs[0].width) == (64, 128)
    ev_acc = _acc(tmp_path / "log" / "ex" / "ft" / "eval")
    for name in ("AEE/occluded", "outliers/occluded", "AEE/non-occluded", "outliers/non-occluded"):
        assert [e.step for e in ev_acc.Scalars(name + "_1")] == [4]
    assert "loss/combined_2" in ev_acc.Tags()["scalars"]


def _step_profile(fn, reps=5):
    """(kernels, device-to-host copies, other copies) of the GPU work ``fn`` issues: per count, the median
    of ``reps`` profiling sessions of one call each.  A session can take in records of the work before it,
    or miss some of its own; the median is the count of a session that did neither."""
    runs = [_profile_once(fn) for _ in range(reps)]
    return tuple(sorted(c)[reps // 2] for c in zip(*runs))


# A session can miss the activities the device runs right at its start: a graph replay profiled that way lost its
# two input copies and up to 193 of its 649 kernels, in two sessions of sixteen after the same process had run
# test_gpu_float64_captured_step.py, and in the full suite often enough that the median of three missed them too.
# Each session therefore opens with a spin kernel of about 25 ms (H100), which the device runs before any of
# ``fn``'s work, and which is not counted.
_SENTINEL_CYCLES = 50_000_000


def _profile_once(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.cuda._sleep(_SENTINEL_CYCLES)
        fn()
        torch.cuda.synchronize()
    kernels = dtoh = other = 0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name.lower()
        if "spin_kernel" in name:         # the sentinel
            continue
        if name.startswith("memcpy"):
            if "dtoh" in name:
                dtoh += 1
            else:
                other += 1
        elif not name.startswith("memset"):
            kernels += 1
    return kernels, dtoh, other


def test_display_steps_cost_under_graph(tmp_path):
    """Under --graph a non-display step issues exactly what a step of a run without summaries issues;
    a display step adds one device-to-host copy of the stacked scalars, plus, with image summaries,
    one copy per image batch."""
    from unflow_b200 import run as R
    from unflow_b200 import synthetic
    from unflow_b200.e2eflow.core import augment
    from unflow_b200.e2eflow.core.summary import SummaryWriter
    from unflow_b200.e2eflow.core.train import Trainer
    params = dict(synthetic.KITTI_PARAMS, learning_rate=1e-5)
    dev = torch.device("cuda")
    tr = Trainer(params, synthetic.KITTI_NORMALIZATION, dev, seed=1234, augment=True)
    tr.track_images = True
    augment.seed(1)
    batch = R.synthetic_batch(2, 128, 256, 1, 0, dev)
    tr.capture(*batch)
    for _ in range(2):
        tr.step(*batch)
    writer = SummaryWriter(str(tmp_path / "train"))

    def plain():
        float(tr.step(*batch))                # a display step of a run without summaries prints the loss

    def silent():
        tr.step(*batch)

    def display(images):
        def fn():
            loss = tr.step(*batch)
            float(loss)
            R.write_train_summaries(writer, tr, tr.iteration, 1e-5, images=images)
        return fn

    base_silent = _step_profile(silent)
    base_print = _step_profile(plain)
    assert base_silent[0] > 100                    # the replayed graph's kernels are seen
    assert base_print[1] == base_silent[1] + 1
    window = [_step_profile(f) for f in (silent, display(False), silent, silent, display(True), silent)]
    for k in (0, 2, 3, 5):
        assert window[k] == base_silent, (k, window[k], base_silent)
    kern, dtoh, other = window[1]
    assert dtoh == base_print[1] + 1 and other == base_print[2] and kern > base_print[0], window[1]
    kern, dtoh, other = window[4]
    n_images = len(tr.tracked()[2])
    assert n_images == 2
    assert dtoh == base_print[1] + 1 + n_images and other == base_print[2], window[4]
    writer.close()
    acc = _acc(tmp_path / "train")
    assert sorted(acc.Tags()["images"]) == sorted("train/augmented%d_1/image/%d" % (a, k)
                                                  for a in (1, 2) for k in (0, 1))
