"""``[run] conv_precision`` without a GPU: how run.py reads it (absent key, both values, a rejected value
before any work), that ``eval.py`` sets each experiment's mode from its copied config, and that the key
overrides ``UNFLOW_CONV_PRECISION`` while its absence leaves that variable in charge."""
import argparse
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from unflow_b200 import eval as E
from unflow_b200 import run as R
from unflow_b200.e2eflow.core import conv_ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def mode_restored():
    prev = conv_ops.get_mode()
    yield
    conv_ops.set_mode(prev)


def _ini(tmp_path, run_extra, name="config.ini"):
    ini = tmp_path / name
    ini.write_text("[dirs]\nlog = %s/log\ncheckpoints = %s/ckpts\ndata = %s/data\n[run]\nbatch_size = 4\n%s"
                   "[train]\nflownet = s\nternary_weight = 1.0\nsave_interval = 1\n"
                   % (tmp_path, tmp_path, tmp_path, run_extra))
    return str(ini)


def test_conv_precision_values():
    assert R.conv_precision({}, 'fp32') == 'fp32'
    assert R.conv_precision({}, '3xtf32') == '3xtf32'
    for value in ('fp32', '3xtf32'):
        for default in ('fp32', '3xtf32'):
            assert R.conv_precision({'conv_precision': value}, default) == value
    for bad in ('tf32', 'FP32', 'bf16', '', 32, True):
        with pytest.raises(SystemExit) as e:
            R.conv_precision({'conv_precision': bad}, 'fp32')
        assert 'fp32' in str(e.value) and '3xtf32' in str(e.value) and 'conv_precision' in str(e.value)


def _main_until_device(monkeypatch, ini):
    """run.main up to the point where it needs a device: a CPU machine, or a GPU machine told it has none."""
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    with pytest.raises(SystemExit) as e:
        R.main(['--ex', 'exP', '--config', ini])
    return str(e.value)


def test_run_sets_the_mode_from_the_config_before_anything_else(tmp_path, monkeypatch):
    for value in ('3xtf32', 'fp32'):
        conv_ops.set_mode('fp32' if value == '3xtf32' else '3xtf32')
        msg = _main_until_device(monkeypatch, _ini(tmp_path, 'conv_precision = %s\n' % value))
        assert 'needs a CUDA device' in msg and conv_ops.get_mode() == value
    # absent: the process's mode stays
    for mode in ('3xtf32', 'fp32'):
        conv_ops.set_mode(mode)
        _main_until_device(monkeypatch, _ini(tmp_path, ''))
        assert conv_ops.get_mode() == mode


def test_run_rejects_an_invalid_value_before_any_work(tmp_path, monkeypatch):
    touched = []
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: touched.append('cuda') or True)
    monkeypatch.setattr(R, 'restore_concluded', lambda *a: touched.append('dirs'))
    conv_ops.set_mode('fp32')
    with pytest.raises(SystemExit) as e:
        R.main(['--ex', 'exP', '--config', _ini(tmp_path, 'conv_precision = 3xTF32\n')])
    assert str(e.value) == '[run] conv_precision = 3xTF32: must be fp32 or 3xtf32'
    assert touched == [] and not (tmp_path / 'log').exists() and not (tmp_path / 'ckpts').exists()
    assert conv_ops.get_mode() == 'fp32'


def test_the_key_overrides_the_environment_variable(tmp_path):
    """UNFLOW_CONV_PRECISION applies when flownet is imported; the key, read after that, wins."""
    code = ("import sys, torch\n"
            "torch.cuda.is_available = lambda: False\n"
            "from unflow_b200 import run as R\n"
            "from unflow_b200.e2eflow.core import conv_ops\n"
            "try:\n    R.main(['--ex', 'e', '--config', sys.argv[1]])\n"
            "except SystemExit:\n    pass\n"
            "print('MODE', conv_ops.get_mode())\n")
    env = dict(os.environ, UNFLOW_CONV_PRECISION='3xtf32', PYTHONPATH=ROOT)
    got = {}
    for name, extra in (('none', ''), ('fp32', 'conv_precision = fp32\n')):
        ini = _ini(tmp_path, extra, name='config_%s.ini' % name)
        r = subprocess.run([sys.executable, '-c', code, ini], cwd=ROOT, env=env, capture_output=True, text=True,
                           timeout=300)
        assert r.returncode == 0, r.stderr[-2000:]
        got[name] = [l for l in r.stdout.splitlines() if l.startswith('MODE ')][-1]
    assert got == {'none': 'MODE 3xtf32', 'fp32': 'MODE fp32'}


def test_eval_sets_each_experiments_mode_from_its_copied_config(tmp_path, capsys):
    cv2 = pytest.importorskip("cv2")
    from unflow_b200.e2eflow.core import flow_io
    from unflow_b200.e2eflow.core import tf_checkpoint as ck
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    tr = tmp_path / "data" / "data_stereo_flow" / "training"
    for sub in ("colored_0", "flow_occ", "flow_noc"):
        (tr / sub).mkdir(parents=True)
    im = np.random.default_rng(0).integers(0, 255, (20, 36, 3), dtype=np.uint8)
    for n in (10, 11):
        cv2.imwrite(str(tr / "colored_0" / ("000000_%d.png" % n)), im)
    for sub in ("flow_occ", "flow_noc"):
        flow_io.write_kitti_flow(str(tr / sub / "000000_10.png"), np.zeros((20, 36, 2), np.float32))
    ini = _ini(tmp_path, '')             # the command's own config: no key
    # three experiments, each with its config copied into log/ex/<name> by run.py
    for name, extra in (('exT', 'conv_precision = 3xtf32\n'), ('exF', 'conv_precision = fp32\n'), ('exN', '')):
        d = tmp_path / "log" / "ex" / name
        d.mkdir(parents=True)
        (d / "config.ini").write_text(open(_ini(tmp_path, extra, name='c_%s.ini' % name)).read())
        ck.save_variables(FlowNetVariables("s", False, seed=1), str(d / "model.ckpt-1"))
    seen = []

    def make(params, normalization, variables):
        seen.append(conv_ops.get_mode())

        def fn(im1, im2):
            return torch.zeros(1, 384, 1280, 2), torch.zeros(1, 384, 1280, 2)
        return fn

    for start in ('fp32', '3xtf32'):
        conv_ops.set_mode(start)
        seen.clear()
        args = argparse.Namespace(dataset='kitti', variant='train_2012', ex='exT,exN,exF,exN', num=1, gpu='0',
                                  output_benchmark=False, output_visual=False, output_backward=False,
                                  output_png=True, config=ini, out=str(tmp_path / "out"))
        E.run_eval(args, torch.device('cpu'), make_flow_fn=make)
        # exN has no key: the mode the command started in, also after exT / exF changed it
        assert seen == ['3xtf32', start, 'fp32', start], (start, seen)
        out = capsys.readouterr().out
        assert "-- evaluating 'exT' in conv precision 3xtf32" in out
        assert "-- evaluating 'exF' in conv precision fp32" in out
    # a bad value in a copied config stops the evaluation of that experiment with the message
    (tmp_path / "log" / "ex" / "exF" / "config.ini").write_text(
        open(_ini(tmp_path, 'conv_precision = tf32\n', name='c_bad.ini')).read())
    with pytest.raises(SystemExit, match='must be fp32 or 3xtf32'):
        E.experiment_setup('exF', ini, 'kitti')


def test_the_readme_config_trains_on_the_tensor_core_kernels(tmp_path):
    """The quick-start ``[run]`` block of README.md, as printed there, parses to what it says."""
    text = open(os.path.join(ROOT, 'README.md')).read()
    blocks = [b.split('```', 1)[0] for b in text.split('```ini\n')[1:]]
    block = next(b for b in blocks if 'conv_precision' in b)
    ini = tmp_path / 'readme.ini'
    ini.write_text(block)
    run_config = R.config_dict(str(ini))['run']
    assert R.conv_precision(run_config, 'fp32') == '3xtf32'
    assert isinstance(run_config['num_input_threads'], int) and isinstance(run_config['batch_size'], int)
