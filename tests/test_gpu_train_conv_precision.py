"""``[run] conv_precision`` on the GPU: ``unflow_b200.run`` trains, and evaluates after every chunk, on the
wgmma kernels when the config asks for 3xtf32, ``unflow_b200.eval`` evaluates an experiment in the mode of
its copied config, and every rank of a ``gpu_list`` run uses the same mode.  Runs on the generated FlyingChairs
tree of test_gpu_datasets.py (384x512, with the KITTI 2012 pairs the runs evaluate on).

Tolerances between the two modes as in test_gpu_datasets: loss 2e-4 relative, 1e-4 of the magnitude for
flow-derived numbers, per-variable L2 1e-2."""
import math
import os
import shutil
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

from test_gpu_datasets import CFG, trees  # noqa: F401,E402  (``trees``: the module-scoped dataset fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def mode_restored():
    from unflow_b200.e2eflow.core import conv_ops
    prev = conv_ops.get_mode()
    yield
    conv_ops.set_mode(prev)


def _config(trees, name, precision):
    """test_gpu_datasets' chairs config with ``conv_precision`` (None: no key) in [run]."""
    text = CFG.format(d=str(trees), dataset="chairs")
    line = "" if precision is None else "conv_precision = %s\n" % precision
    text = text.replace("[run]\n", "[run]\n" + line)
    ini = trees / ("config_%s.ini" % name)
    ini.write_text(text)
    return str(ini)


class _ConvSpy:
    """Counts the wgmma conv launches (through the library's entry points) and the cuDNN convolutions
    (torch.nn.functional.conv2d / conv_transpose2d, which the fp32 path calls)."""

    def __init__(self, monkeypatch):
        from unflow_b200 import _native
        from unflow_b200.e2eflow.core import conv_ops
        self.counts = {"unflow_tc_conv": 0, "unflow_tc_wgrad": 0, "cudnn": 0}
        lib = _native.lib()
        for name in ("unflow_tc_conv", "unflow_tc_wgrad"):
            monkeypatch.setattr(lib, name, self._counting(name, getattr(lib, name)))
        for name in ("conv2d", "conv_transpose2d"):
            monkeypatch.setattr(conv_ops.F, name, self._counting("cudnn", getattr(conv_ops.F, name)))

    def _counting(self, key, fn):
        def call(*a, **k):
            self.counts[key] += 1
            return fn(*a, **k)
        return call

    def reset(self):
        for k in self.counts:
            self.counts[k] = 0


def _train(ini, ex, capsys, *extra):
    from unflow_b200 import run as R
    R.main(["--ex", ex, "--config", ini, "--max-iters", "3", "--ow", *extra])
    out = capsys.readouterr().out
    losses = [float(l.split("loss = ")[1]) for l in out.splitlines() if l.startswith("-- train: i = ")]
    assert len(losses) == 3 and all(math.isfinite(x) for x in losses), out
    return out, losses


def test_3xtf32_config_trains_and_evaluates_on_the_wgmma_kernels(trees, capsys, monkeypatch, mode_restored):
    from unflow_b200.e2eflow.core import conv_ops
    conv_ops.set_mode("fp32")       # the key, not the process's mode, decides
    spy = _ConvSpy(monkeypatch)
    out, _ = _train(_config(trees, "tc", "3xtf32"), "prec_tc", capsys)
    assert "-- rank 0: conv precision 3xtf32" in out, out
    assert "-- eval: i = 3" in out, out          # the in-training evaluation ran inside the spied window
    assert spy.counts["unflow_tc_conv"] > 0 and spy.counts["unflow_tc_wgrad"] > 0, spy.counts
    assert spy.counts["cudnn"] == 0, spy.counts
    # and the fp32 key selects cuDNN
    spy.reset()
    out, _ = _train(_config(trees, "fp", "fp32"), "prec_fp", capsys)
    assert "-- rank 0: conv precision fp32" in out, out
    assert spy.counts["cudnn"] > 0 and spy.counts["unflow_tc_conv"] == 0 and spy.counts["unflow_tc_wgrad"] == 0, \
        spy.counts


def test_without_the_key_the_process_mode_is_kept(trees, capsys, mode_restored):
    from unflow_b200.e2eflow.core import conv_ops
    for mode in ("3xtf32", "fp32"):
        conv_ops.set_mode(mode)
        out, _ = _train(_config(trees, "nokey", None), "prec_nokey", capsys)
        assert "-- rank 0: conv precision %s" % mode in out, out
        assert conv_ops.get_mode() == mode


def _state(trees, ex, it):
    return torch.load(str(trees / "log" / "checkpoints" / ex / ("model.ckpt-%d.pt" % it)))


def test_3xtf32_run_matches_fp32_and_evaluates_in_its_own_mode(trees, capsys, monkeypatch, mode_restored):
    from unflow_b200 import eval as E
    runs = {}
    for mode in ("fp32", "3xtf32"):
        _, losses = _train(_config(trees, "par_" + mode, mode), "par_" + mode, capsys, "--no-augment")
        runs[mode] = (losses, _state(trees, "par_" + mode, 1), _state(trees, "par_" + mode, 3))
    (l_fp, first_fp, s_fp), (l_tc, first_tc, s_tc) = runs["fp32"], runs["3xtf32"]
    for a, b in zip(l_tc, l_fp):
        assert abs(a - b) / abs(b) < 2e-4, (l_tc, l_fp)
    # the first step's gradients, from identical parameters: Adam's first moment after one step is 0.1 g
    m_fp, m_tc = first_fp["adam_slots"], first_tc["adam_slots"]
    e_grad = max(float((m_tc[k][0] - m_fp[k][0]).norm() / m_fp[k][0].norm().clamp_min(1e-20)) for k in m_fp)
    # the parameters after three steps, over the whole network (per variable they are no measure: the first
    # Adam steps move every element by about the learning rate, and the biases start at zero, so where a
    # gradient is near zero its sign decides)
    v_fp, v_tc = s_fp["variables"], s_tc["variables"]
    p_fp = torch.cat([v_fp[k].flatten() for k in sorted(v_fp)])
    p_tc = torch.cat([v_tc[k].flatten() for k in sorted(v_fp)])
    e_params = float((p_tc - p_fp).norm() / p_fp.norm())
    print("losses fp32 %s 3xtf32 %s, worst first-step gradient L2 %.2e, parameters L2 after 3 steps %.2e"
          % (l_fp, l_tc, e_grad, e_params))
    assert e_grad < 1e-2 and e_params < 1e-2, (e_grad, e_params)
    # the 3xtf32 experiment evaluated as its copied config says, and the same checkpoint under an fp32 config
    log_ex = trees / "log" / "ex"
    twin = log_ex / "par_3xtf32_as_fp32"
    if twin.exists():
        shutil.rmtree(str(twin))
    shutil.copytree(str(log_ex / "par_3xtf32"), str(twin))
    (twin / "config.ini").write_text((twin / "config.ini").read_text().replace("conv_precision = 3xtf32",
                                                                               "conv_precision = fp32"))
    assert "3xtf32" not in (twin / "config.ini").read_text()
    spy = _ConvSpy(monkeypatch)
    # the config given on the command line has no key: each experiment's own copy decides
    ini = _config(trees, "eval_nokey", None)
    res = {}
    for ex in ("par_3xtf32", "par_3xtf32_as_fp32"):
        spy.reset()
        res[ex] = E.main(["--dataset", "chairs", "--variant", "test", "--ex", ex, "--num", "-1", "--config", ini,
                          "--out", str(trees / "out")])[ex]
        out = capsys.readouterr().out
        if ex == "par_3xtf32":
            assert "-- evaluating 'par_3xtf32' in conv precision 3xtf32" in out, out
            assert spy.counts["unflow_tc_conv"] > 0 and spy.counts["cudnn"] == 0, spy.counts
        else:
            assert "in conv precision fp32" in out, out
            assert spy.counts["cudnn"] > 0 and spy.counts["unflow_tc_conv"] == 0, spy.counts
    a, b = res["par_3xtf32"]["EPE_all"], res["par_3xtf32_as_fp32"]["EPE_all"]
    print("EPE 3xtf32 %.6f fp32 %.6f" % (a, b))
    assert abs(a - b) <= 1e-4 * max(abs(b), 1.0), (a, b)
    # several experiments in one command: each in its own mode, in either order
    both = E.main(["--dataset", "chairs", "--variant", "test", "--ex", "par_3xtf32_as_fp32,par_3xtf32", "--num", "-1",
                   "--config", ini, "--out", str(trees / "out")])
    out = capsys.readouterr().out
    assert "-- evaluating 'par_3xtf32_as_fp32' in conv precision fp32" in out, out
    assert "-- evaluating 'par_3xtf32' in conv precision 3xtf32" in out, out
    for ex in res:
        assert both[ex] == pytest.approx(res[ex], rel=1e-5), (ex, both[ex], res[ex])


@pytest.mark.parametrize("dataset", ["synthia", "cityscapes"])
def test_graph_capture_while_frames_decode_ahead(dataset, trees, capsys, mode_restored):
    """``--graph`` captures the first step while the pool decodes the next batches: the pool threads make no
    CUDA calls (the pinned batches are allocated on the training thread), so the capture stays valid."""
    ini = trees / ("config_graph_%s.ini" % dataset)
    ini.write_text(CFG.format(d=str(trees), dataset=dataset).replace(
        "[run]\n", "[run]\nconv_precision = 3xtf32\n").replace("num_input_threads = 2", "num_input_threads = 8"))
    _train(str(ini), "graph_" + dataset, capsys, "--graph")


@pytest.mark.skipif(torch.cuda.device_count() < 2,
                    reason="needs at least 2 visible GPUs, this machine shows %d" % torch.cuda.device_count())
def test_every_rank_of_a_gpu_list_run_uses_the_configured_mode(trees):
    ini = _config(trees, "two", "3xtf32")
    text = open(ini).read().replace("gpu_list = 0", "gpu_list = 0,1")
    with open(ini, "w") as f:
        f.write(text)
    r = subprocess.run([sys.executable, "-m", "unflow_b200.run", "--ex", "prec_two", "--config", ini,
                        "--max-iters", "2", "--ow"], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    for rank in (0, 1):
        assert r.stdout.count("-- rank %d: conv precision 3xtf32" % rank) == 1, r.stdout[-3000:]
    assert "conv precision fp32" not in r.stdout
