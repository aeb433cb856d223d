"""Experiment directories of ``python -m unflow_b200.run`` on the GPU (reference src/run.py:204-205,
src/e2eflow/experiment.py, core/data.py:27-36), on short synthetic FlowNetC runs shaped like test_gpu_run.py:
the final checkpoint is concluded into [dirs] log /ex/<name>, training resumes from there when the
checkpoints directory is gone, eval and finetune find it there, and [dirs] fast is staged."""
import glob
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

# at collection, not inside a test: eval.evaluate_examples binds sys.stdout as its default log when the
# module is imported, and a test's captured stdout is closed when that test ends
from unflow_b200 import eval as E

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CFG = """
[dirs]
log = {d}/log
checkpoints = {d}/log/checkpoints
data = {data}
{fast}
[run]
batch_size = {batch}
gpu_list = {gpu_list}
dataset = kitti
development = False
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
{finetune}
"""

WARNING = "Warning: intermediate checkpoints could not be restored."
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2,
                              reason="needs at least 2 visible GPUs, this machine shows %d"
                                     % torch.cuda.device_count())


def _config(d, data=None, fast=None, finetune=None, gpu_list="0", batch=2, name="config.ini"):
    ini = d / name
    ini.write_text(CFG.format(d=d, data=data or "%s/nodata" % d, fast="fast = %s" % fast if fast else "",
                              finetune="finetune = %s" % finetune if finetune else "",
                              gpu_list=gpu_list, batch=batch))
    return str(ini)


def _main(*args):
    from unflow_b200 import run as R
    R.main(list(args))


def _checkpoint_state(path):
    """Variables and Adam moments ``{name: (m, v)}`` of a checkpoint (``.pt`` file or TF prefix), as numpy."""
    if path.endswith(".pt"):
        state = torch.load(path)
        return ({k: v.numpy() for k, v in state["variables"].items()},
                {k: (m.numpy(), v.numpy()) for k, (m, v) in state["adam_slots"].items()})
    from unflow_b200.e2eflow.core import tf_checkpoint
    reader = tf_checkpoint.BundleReader(path)
    names = [k for k in reader.variables() if "/Adam" not in k]
    return ({k: reader.tensor(k) for k in names},
            {k: (reader.tensor(k + "/Adam"), reader.tensor(k + "/Adam_1")) for k in names if k + "/Adam" in reader})


def _record_first_step(monkeypatch):
    """The iteration counter, variables and Adam moments of the trainer when the run takes its first step."""
    from unflow_b200.e2eflow.core.train import Trainer
    real, seen = Trainer.step, []

    def step(self, *batch, **kw):
        if not seen:
            seen.append((self.iteration, {k: v.numpy() for k, v in self.variables.to_tf_dict().items()},
                         self.adam_slots()))
        return real(self, *batch, **kw)
    monkeypatch.setattr(Trainer, "step", step)
    return seen


def _bytes(path):
    with open(path, "rb") as f:
        return f.read()


def _kitti_tree(data):
    """A KITTI raw sequence (two views, six frames) and a two-pair KITTI 2012 training set."""
    import cv2
    from unflow_b200.e2eflow.core import flow_io
    rng = np.random.default_rng(0)
    base = cv2.GaussianBlur(rng.integers(0, 255, (150, 300, 3), dtype=np.uint8), (0, 0), 3)
    for view in ("image_02", "image_03"):
        d = data / "kitti_raw" / "2011_09_26" / "2011_09_26_drive_0001_extract" / view / "data"
        d.mkdir(parents=True)
        for n in range(6):
            assert cv2.imwrite(str(d / ("%010d.png" % n)), np.roll(base, 2 * n, axis=1))
    tr_dir = data / "data_stereo_flow" / "training"
    for sub in ("colored_0", "flow_occ", "flow_noc"):
        (tr_dir / sub).mkdir(parents=True)
    for i in range(2):
        im = np.roll(base, 5 * i, axis=0)[:120, :280]
        assert cv2.imwrite(str(tr_dir / "colored_0" / ("%06d_10.png" % i)), im)
        assert cv2.imwrite(str(tr_dir / "colored_0" / ("%06d_11.png" % i)), np.roll(im, 3, axis=1))
        flow = np.zeros((120, 280, 2), np.float32)
        flow[..., 0] = 3.0
        for sub in ("flow_occ", "flow_noc"):
            flow_io.write_kitti_flow(str(tr_dir / sub / ("%06d_10.png" % i)), flow, np.ones((120, 280)))
    return data


def _files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


@pytest.mark.parametrize("fmt", ["pt", "tf"])
def test_concluded_checkpoint_resumes_when_checkpoints_are_gone(tmp_path, capsys, monkeypatch, fmt):
    """The run to 4 concludes a byte-identical copy of its last checkpoint into log/ex; with the
    checkpoints directory deleted, the next run starts from it: its first step is iteration 5, taken from
    exactly the concluded variables and Adam moments (bit for bit, whatever the step's float atomics do)."""
    ini = _config(tmp_path)
    ckpt, ex = tmp_path / "log" / "checkpoints" / "r", tmp_path / "log" / "ex" / "r"
    args = ("--ex", "r", "--config", ini, "--synthetic", "--ckpt-format", fmt)
    _main(*args, "--max-iters", "4")
    out = capsys.readouterr().out
    assert "-- training from i = 1 to 4" in out and WARNING not in out
    names = ["model.ckpt-4.pt"] if fmt == "pt" else ["model.ckpt-4.data-00000-of-00001", "model.ckpt-4.index"]
    for name in names:
        assert _bytes(str(ex / name)) == _bytes(str(ckpt / name)), name
    if fmt == "tf":
        from unflow_b200.e2eflow.core import tf_checkpoint
        assert tf_checkpoint.get_checkpoint_state(str(ex)) == (str(ex / "model.ckpt-4"), [str(ex / "model.ckpt-4")])

    shutil.rmtree(str(ckpt))
    seen = _record_first_step(monkeypatch)
    _main(*args)
    out = capsys.readouterr().out
    assert WARNING in out and "-- training from i = 5 to 6" in out, out
    iteration, variables, slots = seen[0]
    want_variables, want_slots = _checkpoint_state(str(ex / "model.ckpt-4") + (".pt" if fmt == "pt" else ""))
    assert iteration == 4                     # Trainer.step counts it up to 5 before the update
    assert variables.keys() == want_variables.keys() and slots.keys() == want_slots.keys()
    for k in variables:
        assert np.array_equal(variables[k], want_variables[k]), k
    for k in slots:
        assert np.array_equal(slots[k][0], want_slots[k][0]) and np.array_equal(slots[k][1], want_slots[k][1]), k
    # the moments are those of 4 steps, not a fresh optimiser's zeros
    assert any(np.abs(m).max() > 0 for m, _ in slots.values())
    concluded = sorted(n for n in os.listdir(str(ex)) if n.startswith("model.ckpt-"))
    assert concluded == (["model.ckpt-4.pt", "model.ckpt-6.pt"] if fmt == "pt" else
                         ["model.ckpt-4.data-00000-of-00001", "model.ckpt-4.index",
                          "model.ckpt-6.data-00000-of-00001", "model.ckpt-6.index"])

    # a run with nothing left to train concludes too
    index = "model.ckpt-6.pt" if fmt == "pt" else "model.ckpt-6.index"
    os.remove(str(ex / index))
    _main(*args)
    assert "max_iter reached" in capsys.readouterr().out
    assert _bytes(str(ex / index)) == _bytes(str(ckpt / index))


def test_debug_run_concludes_nothing(tmp_path, capsys):
    ini = _config(tmp_path)
    _main("--ex", "dbg", "--config", ini, "--synthetic", "--debug", "--max-iters", "2")
    assert "-- training from i = 1 to 2" in capsys.readouterr().out
    assert not glob.glob(str(tmp_path / "log" / "ex" / "dbg" / "model.ckpt-*"))
    assert not os.path.exists(str(tmp_path / "log" / "ex" / "dbg" / "checkpoint"))


def test_eval_and_finetune_use_the_concluded_checkpoint(tmp_path, capsys):
    pytest.importorskip("cv2")
    data = _kitti_tree(tmp_path / "data")
    ini = _config(tmp_path, data=data)
    _main("--ex", "src", "--config", ini, "--synthetic", "--max-iters", "2")
    capsys.readouterr()
    concluded = str(tmp_path / "log" / "ex" / "src" / "model.ckpt-2.pt")
    shutil.rmtree(str(tmp_path / "log" / "checkpoints" / "src"))
    res = E.main(["--dataset", "kitti", "--variant", "train_2012", "--ex", "src", "--num", "2",
                  "--config", ini, "--out", str(tmp_path / "out")])
    assert res["src"] and all(math.isfinite(v) for v in res["src"].values()), res
    ini_ft = _config(tmp_path, data=data, finetune="src", name="config_ft.ini")
    _main("--ex", "ft", "--config", ini_ft, "--synthetic", "--max-iters", "2")
    out = capsys.readouterr().out
    assert "-- restore network 0 %s" % concluded in out and "-- training from i = 1 to 2" in out, out


def test_fast_is_staged_and_trained_from(tmp_path, capsys):
    pytest.importorskip("cv2")
    data = _kitti_tree(tmp_path / "data")
    fast = tmp_path / "fast"
    fast.mkdir()
    ini = _config(tmp_path, data=data, fast=fast)
    _main("--ex", "f", "--config", ini, "--max-iters", "2")
    out = capsys.readouterr().out
    assert ">> Copied kitti_raw" in out and ">> Copied data_stereo_flow" in out, out
    assert "Training on 10 frame pairs." in out and "-- eval: i = 2" in out and "num_examples = 2" in out, out
    assert sorted(os.listdir(str(fast))) == ["data_stereo_flow", "kitti_raw"]
    assert _files(str(fast)) == _files(str(data))
    # staged directories are kept and not copied again
    _main("--ex", "f", "--config", ini, "--max-iters", "4")
    out = capsys.readouterr().out
    assert ">> Copied" not in out and "-- training from i = 3 to 4" in out, out


def _run(*args):
    r = subprocess.run([sys.executable, "-m", "unflow_b200.run", *args], cwd=ROOT, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


@two_gpus
def test_two_gpus_conclude_resume_and_stage_once(tmp_path):
    pytest.importorskip("cv2")
    data = _kitti_tree(tmp_path / "data")
    fast = tmp_path / "fast"
    fast.mkdir()
    ini = _config(tmp_path, gpu_list="0,1", batch=4)
    ex = tmp_path / "log" / "ex" / "two"
    out = _run("--ex", "two", "--config", ini, "--synthetic", "--max-iters", "4")
    assert out.count("-- training from i = 1 to 4") == 1
    assert sorted(n for n in os.listdir(str(ex)) if n.startswith("model.ckpt")) == ["model.ckpt-4.pt"]
    shutil.rmtree(str(tmp_path / "log" / "checkpoints" / "two"))
    out = _run("--ex", "two", "--config", ini, "--synthetic")
    # both ranks restart at 5: a rank that started elsewhere would run a different number of all-reduces
    assert out.count(WARNING) == 1 and out.count("-- training from i = 5 to 6") == 1, out
    assert sorted(n for n in os.listdir(str(ex)) if n.startswith("model.ckpt")) == \
        ["model.ckpt-4.pt", "model.ckpt-6.pt"]
    ini = _config(tmp_path, data=data, fast=fast, gpu_list="0,1", batch=4, name="config_fast.ini")
    out = _run("--ex", "twofast", "--config", ini, "--max-iters", "2")
    assert out.count(">> Copied kitti_raw") == 1 and out.count(">> Copied data_stereo_flow") == 1, out
    assert sorted(os.listdir(str(fast))) == ["data_stereo_flow", "kitti_raw"]
    assert _files(str(fast)) == _files(str(data))
