"""[run] gpu_list on the GPU: ``python -m unflow_b200.run`` trains on the listed devices from one command
(reference src/run.py:40-49), on a short synthetic FlowNetC run shaped like test_gpu_run.py."""
import glob
import json
import os
import re
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LR = 1.0e-5

CFG = """
[dirs]
log = {d}/log
checkpoints = {d}/log/checkpoints
data = {d}/nodata
[run]
batch_size = {batch}
{gpu_list}
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
learning_rate = {lr}
decay_after = 100000
fb_weight = 0.2
mask_occlusion = fb
occ_weight = 12.4
"""

two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2,
                              reason="needs at least 2 visible GPUs, this machine shows %d"
                                     % torch.cuda.device_count())


def _config(tmp_path, gpu_list, batch):
    ini = tmp_path / "config.ini"
    ini.write_text(CFG.format(d=tmp_path, batch=batch, gpu_list=gpu_list, lr=LR))
    return str(ini)


def _run(*args, launcher=("-m", "unflow_b200.run")):
    r = subprocess.run([sys.executable, *launcher, *args], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def _processes_mentioning(text):
    """Pids of live processes (other than this one) whose command line contains ``text``."""
    found = []
    for d in glob.glob("/proc/[0-9]*"):
        try:
            with open(d + "/cmdline", "rb") as fh:
                cmdline = fh.read().decode(errors="replace")
        except OSError:
            continue
        if text in cmdline and int(d[6:]) != os.getpid():
            found.append(int(d[6:]))
    return found


def _checkpoints(tmp_path, ex):
    return sorted(os.path.basename(c) for c in
                  glob.glob(str(tmp_path / "log" / "checkpoints" / ex / "model.ckpt-*.pt")))


def _state(tmp_path, ex, it):
    return torch.load(str(tmp_path / "log" / "checkpoints" / ex / ("model.ckpt-%d.pt" % it)))


@two_gpus
def test_one_command_trains_on_two_gpus_and_resumes(tmp_path):
    ini = _config(tmp_path, "gpu_list = 0,1", batch=4)
    out = _run("--ex", "two", "--config", ini, "--synthetic", "--max-iters", "4")
    assert not _processes_mentioning(ini)
    assert _checkpoints(tmp_path, "two") == ["model.ckpt-2.pt", "model.ckpt-4.pt"]
    # rank 0 alone prints
    assert out.count("-- training from i = 1 to 4") == 1
    for i in range(1, 5):
        assert out.count("-- train: i = %d, loss" % i) == 1
    # resume from the newest checkpoint, again on both GPUs
    out = _run("--ex", "two", "--config", ini, "--synthetic")
    assert out.count("-- training from i = 5 to 6") == 1
    assert _checkpoints(tmp_path, "two")[-1] == "model.ckpt-6.pt"
    assert not _processes_mentioning(ini)


@two_gpus
def test_one_command_matches_torch_distributed_run(tmp_path):
    """The launch starts the same two ranks torch.distributed.run does, so the checkpoints agree to within
    the run-to-run spread of the step.  The tolerance is not a claim of bit-identity: the weight-gradient
    atomics and the K slices of the conv kernels add in an order that varies between runs.  Adam moves a
    weight by about the learning rate per step whatever the gradient, so a reordered sum that flips the
    sign of a near-zero gradient can move a weight by up to 2 x lr per step: after two steps the weights
    are held to 4 x lr absolute.  That bound hardly tells batches apart, so the first moments (the
    gradients themselves) are compared too, relative to their norm, at 1e-4.  Measured on one H100 80GB
    HBM3 at a 700 W power limit, three single-GPU runs of this config (batch 2) differ by at most 1.16 x lr
    in a weight and 3.0e-6 in the moments' relative norm, while a run on a different batch differs by
    0.27 in the moments.  The spread between two-GPU runs has not been measured."""
    ini = _config(tmp_path, "gpu_list = 0,1", batch=4)
    _run("--ex", "one", "--config", ini, "--synthetic", "--max-iters", "2")
    _run("--standalone", "--nproc-per-node", "2", "-m", "unflow_b200.run",
         "--ex", "tdr", "--config", ini, "--synthetic", "--max-iters", "2",
         launcher=("-m", "torch.distributed.run"))
    a, b = _state(tmp_path, "one", 2), _state(tmp_path, "tdr", 2)
    assert a["variables"].keys() == b["variables"].keys()
    worst = max(float((a["variables"][k] - b["variables"][k]).abs().max()) for k in a["variables"])
    assert worst <= 4 * LR, worst
    m_a = torch.cat([m.flatten() for m, _ in a["adam_slots"].values()])
    m_b = torch.cat([m.flatten() for m, _ in b["adam_slots"].values()])
    rel = float((m_a - m_b).norm() / m_b.norm())
    assert rel < 1e-4, rel


@two_gpus
def test_single_id_trains_in_process_on_that_device(tmp_path):
    ini = _config(tmp_path, "gpu_list = 1", batch=2)
    code = ("import json, torch; from unflow_b200 import run; "
            "run.main(['--ex', 'one', '--config', %r, '--synthetic', '--max-iters', '2']); "
            "print(json.dumps([torch.cuda.max_memory_allocated(d) for d in (0, 1)]))" % ini)
    out = _run(launcher=("-c", code))
    peak0, peak1 = json.loads(out.strip().splitlines()[-1])
    assert peak1 > 0 and peak0 == 0, (peak0, peak1)
    assert _checkpoints(tmp_path, "one") == ["model.ckpt-2.pt"]


def test_gpu_list_zero_runs_as_without_the_key(tmp_path):
    """``gpu_list = 0`` takes the new resolution path and must print and write what a run without the
    key (cuda:LOCAL_RANK) does; only the loss values, which the float atomics may vary, are left out."""
    outs, names = [], []
    for ex, gpu_list in (("listed", "gpu_list = 0"), ("unlisted", "")):
        d = tmp_path / ex
        d.mkdir()
        ini = _config(d, gpu_list, batch=2)
        out = _run("--ex", "t", "--config", ini, "--synthetic", "--max-iters", "4")
        outs.append(re.sub(r"loss = \S+", "loss = *", out))
        names.append(_checkpoints(d, "t"))
    assert outs[0] == outs[1] and "-- train: i = 4, loss = *" in outs[0]
    assert names[0] == names[1] == ["model.ckpt-2.pt", "model.ckpt-4.pt"]
