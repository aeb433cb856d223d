"""TensorBoard summaries (core/summary.py, run.py): event files read back with tensorboard's own
reader, the ``tf.summary.image`` conversion against a restatement of TF's ImageSummary kernel, and the
product's summary tags against the reference's own code run under the TF stand-in
(tests/golden/make_reference_summaries.py -> tests/golden/reference_summaries.json)."""
import io
import json
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_summaries.json")))


def _accumulator(logdir):
    from tensorboard.backend.event_processing import event_accumulator as ea
    acc = ea.EventAccumulator(str(logdir), size_guidance={ea.SCALARS: 0, ea.IMAGES: 0})
    acc.Reload()
    return acc


def _decode_png(data):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(data)))


def tf_image_float64(x, max_outputs=3):
    """ImageSummary's float rule (summary_image_op.cc NormalizeFloatImage) in float64, per image."""
    x = np.asarray(x, dtype=np.float64)[:max_outputs]
    out = np.empty(x.shape, dtype=np.uint8)
    for n, im in enumerate(x):
        finite = np.isfinite(im).all(axis=-1)
        vals = im[finite]
        lo, hi = (vals.min(), vals.max()) if vals.size else (np.inf, -np.inf)
        if lo < 0:
            m = max(abs(lo), abs(hi))
            scale, offset = (0.0 if m < 1e-6 else 127.0 / m), 128.0
        else:
            scale, offset = (0.0 if hi < 1e-6 else 255.0 / hi), 0.0
        y = np.floor(im * scale + offset)
        y[~finite] = np.array([255, 0, 0])[:im.shape[-1]]
        out[n] = y.astype(np.uint8)
    return out


def _cases():
    g = torch.Generator().manual_seed(3)
    yield "nonneg", torch.rand(5, 6, 7, 3, generator=g) * 3
    yield "mixed", torch.randn(1, 6, 7, 3, generator=g)
    yield "mixed_1ch", torch.randn(4, 5, 9, 1, generator=g) * 10
    yield "nonneg_1ch", torch.rand(1, 8, 8, 1, generator=g)
    yield "mask", (torch.rand(2, 8, 8, 1, generator=g) > 0.5).float()
    yield "zeros", torch.zeros(2, 4, 4, 3)
    yield "positive_constant", torch.full((1, 4, 4, 1), 0.25)
    yield "negative_constant", torch.full((5, 4, 4, 3), -2.0)
    yield "tiny", torch.full((1, 3, 3, 3), 1e-7)
    nonfinite = torch.rand(2, 4, 5, 3, generator=g) - 0.2
    nonfinite[0, 1, 2, 0] = float('nan')
    nonfinite[1, 0, 0, 2] = float('inf')
    yield "nonfinite", nonfinite


@pytest.mark.parametrize("name,x", list(_cases()), ids=[c[0] for c in _cases()])
def test_image_conversion_against_tf_rule(name, x):
    from unflow_b200.e2eflow.core.summary import image_uint8
    got = image_uint8(x).numpy()
    assert got.dtype == np.uint8 and got.shape == (min(x.shape[0], 3),) + tuple(x.shape[1:])
    want = tf_image_float64(x.numpy())
    # TF scales in float32 and truncates: a value within float32 rounding of an integer may land one
    # level off the float64 restatement
    diff = want.astype(np.int32) - got.astype(np.int32)
    assert np.abs(diff).max() <= 1, (name, diff.min(), diff.max())
    assert (diff != 0).mean() < 0.05, name
    if name in ("mask", "zeros", "positive_constant", "negative_constant", "tiny"):
        assert np.array_equal(got, want), name


def test_writer_round_trip_through_tensorboard_reader(tmp_path):
    from unflow_b200.e2eflow.core.summary import SummaryWriter, image_uint8
    w = SummaryWriter(str(tmp_path / "run"))
    values = [0.1, 1.0 / 3.0, 12345.678, -2.5e-7]
    for step, v in enumerate(values, 1):
        w.scalar("loss/combined_1", v, step)
        w.scalar("params/train/learning_rate", torch.tensor(v * 2), step)
    g = torch.Generator().manual_seed(1)
    rgb = torch.rand(5, 6, 10, 3, generator=g) * 2 - 0.5
    gray = torch.rand(1, 7, 4, 1, generator=g)
    w.image("train/augmented1_1", rgb, 7)
    w.image("train/mask_gt_1", gray, 7)
    w.close()
    acc = _accumulator(tmp_path / "run")
    got = acc.Scalars("loss/combined_1")
    assert [e.step for e in got] == [1, 2, 3, 4]
    assert [np.float32(e.value) for e in got] == [np.float32(v) for v in values]           # bit-equal float32
    assert [np.float32(e.value) for e in acc.Scalars("params/train/learning_rate")] == \
        [np.float32(v * 2) for v in values]
    tags = acc.Tags()["images"]
    assert sorted(tags) == ["train/augmented1_1/image/%d" % i for i in range(3)] + ["train/mask_gt_1/image/0"]
    want = image_uint8(rgb).numpy()
    for i in range(3):
        (ev,) = acc.Images("train/augmented1_1/image/%d" % i)
        assert (ev.step, ev.width, ev.height) == (7, 10, 6)
        assert np.array_equal(_decode_png(ev.encoded_image_string), want[i])
    (ev,) = acc.Images("train/mask_gt_1/image/0")
    assert (ev.width, ev.height) == (4, 7)
    assert np.array_equal(_decode_png(ev.encoded_image_string), image_uint8(gray).numpy()[0, :, :, 0])


def test_writer_without_tensorboard_fails_loudly(tmp_path, monkeypatch):
    from unflow_b200.e2eflow.core.summary import SummaryWriter
    monkeypatch.setitem(sys.modules, "torch.utils.tensorboard", None)
    with pytest.raises(ImportError, match="tensorboard"):
        SummaryWriter(str(tmp_path / "run"))


def test_unique_name_follows_tf():
    from unflow_b200.e2eflow.core.summary import unique_name
    used = {}
    assert [unique_name(used, n) for n in ("a", "a", "a_1", "a", "A", "b")] == ["a", "a_1", "a_1_1", "a_2", "A_3", "b"]


def _product_on_cpu(monkeypatch):
    """The product's host path with its CUDA entry points swapped for the oracle's CPU ops (as
    test_oracle_vs_reference_run.py's test_product_* do), plus the augmentation's sampler."""
    from oracle import augment as oaug
    from oracle import image_warp as oimage_warp
    from oracle import ops as oops
    from oracle import util as outil
    from unflow_b200.e2eflow.core import augment as A
    from unflow_b200.e2eflow.core import flownet as F
    from unflow_b200.e2eflow.core import losses as L
    from unflow_b200.e2eflow.core import unsupervised as U
    monkeypatch.setattr(F, 'correlation', oops.correlation)
    monkeypatch.setattr(F, 'image_warp', oimage_warp.image_warp)
    monkeypatch.setattr(L, 'image_warp', oimage_warp.image_warp)
    monkeypatch.setattr(L, 'forward_warp', oops.forward_warp)
    monkeypatch.setattr(U, 'downsample', outil.downsample)
    monkeypatch.setattr(A, 'transformer', oaug.transformer)
    monkeypatch.setattr(U, 'track_images', True)
    return U


@pytest.mark.parametrize("config", sorted(GOLDEN["configs"]))
def test_summary_tags_match_the_reference(monkeypatch, config):
    from unflow_b200 import synthetic
    from unflow_b200.e2eflow.core import summary
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    from unflow_b200.e2eflow.core.supervised import supervised_loss
    ref = GOLDEN["configs"][config]
    params = ref["params"]
    U = _product_on_cpu(monkeypatch)
    v = FlowNetVariables(params["flownet"], False, seed=0)
    h, w = 128, 256
    with torch.no_grad():
        if "kitti_ft" in config:
            supervised_loss(synthetic.supervised_batch(1, h, w, seed=7), params, synthetic.KITTI_NORMALIZATION,
                            variables=v)
        else:
            im1, im2, _ = synthetic.image_pair(1, h, w, seed=7)
            U.unsupervised_loss((im1, im2), params, synthetic.KITTI_NORMALIZATION, augment=True, variables=v)
    assert list(U.tracked) == ref["losses"]
    assert list(U.tracked_params) == ref["params_collection"]
    assert list(U.tracked_images) == ref["train_images"]
    tags = summary.train_tags(U.tracked, U.tracked_params, U.tracked_images)
    got = ([["scalar", tags["learning_rate"]["learning_rate"]]] + [["scalar", t] for t in tags["losses"].values()]
           + [["scalar", t] for t in tags["params"].values()] + [["image", t] for t in tags["images"].values()])
    assert got == ref["train_summaries"]
    # the evaluation graph: unsupervised_loss without augmentation (train.py:277-281), then the placeholders
    with torch.no_grad():
        im1, im2, _ = synthetic.image_pair(1, h, w, seed=8)
        U.unsupervised_loss((im1, im2), params, synthetic.KITTI_NORMALIZATION, augment=False, variables=v)
    assert list(U.tracked) == ref["eval_losses"]
    assert [["scalar", t] for t in summary.eval_tags(U.tracked).values()] == ref["eval_summaries"]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _writer_worker(rank, world, port, logdir):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from unflow_b200 import run as R
    train, ev = R.summary_writers(logdir, "ex", dist.get_rank())
    assert (train is None and ev is None) == (rank != 0)
    if train is not None:
        train.scalar("loss/combined_1", 1.5, 1)
        train.close()
        ev.close()
    dist.barrier()
    dist.destroy_process_group()


def test_only_rank_zero_writes_summaries(tmp_path):
    logdir = str(tmp_path / "log")
    mp.spawn(_writer_worker, args=(2, _free_port(), logdir), nprocs=2, join=True)
    for sub in ("train", "eval"):
        files = os.listdir(os.path.join(logdir, "ex", "ex", sub))
        assert len(files) == 1 and files[0].startswith("events.out.tfevents."), files
    assert [e.value for e in _accumulator(os.path.join(logdir, "ex", "ex", "train")).Scalars("loss/combined_1")] == [1.5]


def test_overwrite_removes_earlier_summaries(tmp_path):
    from unflow_b200 import run as R
    log = str(tmp_path / "log")
    for overwrite, n_files in ((False, 1), (False, 2), (True, 1)):
        train, ev = R.summary_writers(log, "ex", 0, overwrite=overwrite)
        train.scalar("x", 1.0, 1)
        train.close()
        ev.close()
        assert len(os.listdir(os.path.join(log, "ex", "ex", "train"))) == n_files
