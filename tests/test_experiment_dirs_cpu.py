"""Experiment directories of ``run`` on the CPU (reference src/e2eflow/experiment.py, core/data.py:27-36):
concluding the newest checkpoint into [dirs] log /ex/<name>, restoring from there when [dirs] checkpoints
has none, ``--ow``'s removal of concluded checkpoints, and staging datasets into [dirs] fast."""
import os
import shutil

import numpy as np
import pytest
import torch

from unflow_b200 import run as R
from unflow_b200.e2eflow.core import data as D
from unflow_b200.e2eflow.core import tf_checkpoint


class _Variables:
    """The part of ``FlowNetVariables`` that ``tf_checkpoint.save_variables`` reads."""

    def __init__(self, seed):
        rng = np.random.default_rng(seed)
        self.tensors = {'flownet_c/conv1/weights': rng.standard_normal((3, 3, 2, 4)).astype(np.float32),
                        'flownet_c/conv1/biases': rng.standard_normal(4).astype(np.float32)}

    def to_tf_dict(self):
        return self.tensors


def _pt(ckpt_dir, it):
    os.makedirs(ckpt_dir, exist_ok=True)
    path = os.path.join(ckpt_dir, 'model.ckpt-%d.pt' % it)
    torch.save({'variables': {'flownet_c/conv1/biases': torch.full((4,), float(it))}, 'adam_slots': {}}, path)
    return path


def _tf(ckpt_dir, it, seed=None):
    return tf_checkpoint.save_variables(_Variables(it if seed is None else seed),
                                        os.path.join(ckpt_dir, 'model.ckpt-%d' % it))


def _bytes(path):
    with open(path, 'rb') as f:
        return f.read()


def _fail_halfway(monkeypatch, fail_on):
    """Make ``shutil.copyfile`` write half of a file whose name ends with ``fail_on`` and raise."""
    real = shutil.copyfile

    def copyfile(src, dst, **kw):
        if not src.endswith(fail_on):
            return real(src, dst, **kw)
        data = _bytes(src)
        with open(dst, 'wb') as f:
            f.write(data[:len(data) // 2])
        raise OSError(28, 'No space left on device')
    monkeypatch.setattr(shutil, 'copyfile', copyfile)


def test_conclude_copies_the_newest_pt_checkpoint(tmp_path):
    ckpt, ex = str(tmp_path / 'checkpoints' / 'a'), str(tmp_path / 'log' / 'ex' / 'a')
    for it in (2, 4):
        _pt(ckpt, it)
    got = R.conclude(ckpt, ex)
    assert got == os.path.join(ex, 'model.ckpt-4.pt')
    assert sorted(os.listdir(ex)) == ['model.ckpt-4.pt']
    assert _bytes(got) == _bytes(os.path.join(ckpt, 'model.ckpt-4.pt'))
    assert R.latest_checkpoint(ex) == (4, got)
    # a later conclusion leaves the earlier one in place
    _pt(ckpt, 6)
    R.conclude(ckpt, ex)
    assert sorted(os.listdir(ex)) == ['model.ckpt-4.pt', 'model.ckpt-6.pt']
    assert R.latest_checkpoint(ex)[0] == 6


def test_conclude_without_checkpoints_warns(tmp_path, capsys):
    assert R.conclude(str(tmp_path / 'none'), str(tmp_path / 'ex')) is None
    assert 'Warning: no checkpoints written' in capsys.readouterr().out
    assert not os.path.exists(str(tmp_path / 'ex'))


def test_conclude_tf_checkpoint_round_trips_through_the_state_file(tmp_path):
    ckpt, ex = str(tmp_path / 'checkpoints' / 'a'), str(tmp_path / 'log' / 'ex' / 'a')
    for it in (2, 4):
        _tf(ckpt, it)
    prefix = R.conclude(ckpt, ex)
    assert prefix == os.path.join(ex, 'model.ckpt-4')
    assert sorted(os.listdir(ex)) == ['checkpoint', 'model.ckpt-4.data-00000-of-00001', 'model.ckpt-4.index']
    # the state file names the basename only, as the reference's _copy_latest_checkpoint writes it
    assert _bytes(os.path.join(ex, 'checkpoint')) == \
        b'model_checkpoint_path: "model.ckpt-4"\nall_model_checkpoint_paths: "model.ckpt-4"\n'
    assert tf_checkpoint.get_checkpoint_state(ex) == (prefix, [prefix])
    assert R.latest_checkpoint(ex) == (4, prefix)
    reader = tf_checkpoint.BundleReader(prefix)
    for name, want in _Variables(4).tensors.items():
        assert np.array_equal(reader.tensor(name), want)


def test_a_failed_pt_copy_leaves_the_previous_checkpoint_newest(tmp_path, monkeypatch):
    ckpt, ex = str(tmp_path / 'checkpoints' / 'a'), str(tmp_path / 'log' / 'ex' / 'a')
    _pt(ckpt, 2)
    R.conclude(ckpt, ex)
    _pt(ckpt, 4)
    _fail_halfway(monkeypatch, 'model.ckpt-4.pt')
    with pytest.raises(OSError):
        R.conclude(ckpt, ex)
    assert R.latest_checkpoint(ex) == (2, os.path.join(ex, 'model.ckpt-2.pt'))
    assert sorted(os.listdir(ex)) == ['model.ckpt-2.pt']


@pytest.mark.parametrize('fail_on', ['.data-00000-of-00001', '.index'])
def test_a_failed_tf_copy_leaves_the_previous_checkpoint_newest(tmp_path, monkeypatch, fail_on):
    ckpt, ex = str(tmp_path / 'checkpoints' / 'a'), str(tmp_path / 'log' / 'ex' / 'a')
    _tf(ckpt, 2)
    R.conclude(ckpt, ex)
    before = sorted(os.listdir(ex))
    _tf(ckpt, 4)
    _fail_halfway(monkeypatch, 'model.ckpt-4' + fail_on)
    with pytest.raises(OSError):
        R.conclude(ckpt, ex)
    assert R.latest_checkpoint(ex) == (2, os.path.join(ex, 'model.ckpt-2'))
    left = sorted(os.listdir(ex))
    assert not any(n.startswith('model.ckpt-4' + fail_on) or n.endswith('.partial') for n in left), left
    assert set(before) <= set(left)


@pytest.mark.parametrize('kind', ['pt', 'tf'])
def test_concluding_the_same_checkpoint_again_copies_nothing(tmp_path, monkeypatch, kind):
    ckpt, ex = str(tmp_path / 'checkpoints' / 'a'), str(tmp_path / 'log' / 'ex' / 'a')
    (_pt if kind == 'pt' else _tf)(ckpt, 4)
    first = R.conclude(ckpt, ex)
    _fail_halfway(monkeypatch, '')      # any data copy would now fail
    assert R.conclude(ckpt, ex) == first
    assert R.latest_checkpoint(ex) == (4, first)


def test_a_different_tf_checkpoint_of_the_same_name_never_pairs_old_and_new_files(tmp_path, monkeypatch):
    ckpt, ex = str(tmp_path / 'checkpoints' / 'a'), str(tmp_path / 'log' / 'ex' / 'a')
    _tf(ckpt, 4, seed=1)
    R.conclude(ckpt, ex)
    shutil.rmtree(ckpt)
    _tf(ckpt, 4, seed=2)
    _fail_halfway(monkeypatch, 'model.ckpt-4.data-00000-of-00001')
    with pytest.raises(OSError):
        R.conclude(ckpt, ex)
    # the old index went first: the old data is not readable as the new checkpoint, nor the reverse
    assert not os.path.exists(os.path.join(ex, 'model.ckpt-4.index'))
    assert R.latest_checkpoint(ex) is None
    monkeypatch.undo()
    prefix = R.conclude(ckpt, ex)
    for suffix in ('.index', '.data-00000-of-00001'):
        assert _bytes(prefix + suffix) == _bytes(os.path.join(ckpt, 'model.ckpt-4' + suffix))
    reader = tf_checkpoint.BundleReader(prefix)
    for name, want in _Variables(2).tensors.items():
        assert np.array_equal(reader.tensor(name), want)


@pytest.mark.parametrize('ckpt_state', ['missing', 'empty'])
@pytest.mark.parametrize('kind', ['pt', 'tf'])
def test_restore_copies_the_concluded_checkpoint_back(tmp_path, capsys, ckpt_state, kind):
    ckpt, ex = str(tmp_path / 'checkpoints' / 'a'), str(tmp_path / 'log' / 'ex' / 'a')
    write = _pt if kind == 'pt' else _tf
    for it in (2, 4):
        write(ckpt, it)
    R.conclude(ckpt, ex)
    shutil.rmtree(ckpt)
    if ckpt_state == 'empty':
        os.makedirs(ckpt)
    got = R.restore_concluded(ckpt, ex)
    assert 'Warning: intermediate checkpoints could not be restored.' in capsys.readouterr().out
    assert R.latest_checkpoint(ckpt) == (4, got)
    name = 'model.ckpt-4.pt' if kind == 'pt' else 'model.ckpt-4.index'
    assert _bytes(os.path.join(ckpt, name)) == _bytes(os.path.join(ex, name))


def test_restore_leaves_an_experiment_with_its_own_checkpoint_alone(tmp_path, capsys):
    ckpt, ex = str(tmp_path / 'checkpoints' / 'a'), str(tmp_path / 'log' / 'ex' / 'a')
    _pt(ex, 6)
    _pt(ckpt, 2)
    assert R.restore_concluded(ckpt, ex) is None
    assert os.listdir(ckpt) == ['model.ckpt-2.pt']
    # neither directory has a checkpoint: nothing happens, training starts at iteration 1
    assert R.restore_concluded(str(tmp_path / 'c2'), str(tmp_path / 'ex2')) is None
    assert not os.path.exists(str(tmp_path / 'c2'))
    assert 'Warning' not in capsys.readouterr().out


def test_overwrite_removes_only_the_concluded_checkpoints(tmp_path):
    ex = tmp_path / 'log' / 'ex' / 'a'
    _pt(str(ex), 2)
    _tf(str(ex), 4)
    (ex / 'model.ckpt-6.pt.partial').write_bytes(b'x')
    (ex / 'config.ini').write_text('[run]\n')
    for d in ('train', 'eval'):
        (ex / d).mkdir()
        (ex / d / 'events.out').write_bytes(b'x')
    R.remove_concluded(str(ex))
    assert sorted(os.listdir(ex)) == ['config.ini', 'eval', 'train']
    assert os.listdir(ex / 'train') == ['events.out']
    R.remove_concluded(str(tmp_path / 'absent'))


def _tree(root, rel_files):
    for rel in rel_files:
        p = os.path.join(root, rel)
        os.makedirs(os.path.dirname(p), exist_ok=True)
        with open(p, 'w') as f:
            f.write(rel)


def _files(root):
    return sorted(os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)


def test_stage_copies_only_missing_directories(tmp_path, capsys):
    data, fast = str(tmp_path / 'data'), str(tmp_path / 'fast')
    _tree(data, ['kitti_raw/2011_09_26/d/image_02/data/0.png', 'data_stereo_flow/training/colored_0/0_10.png',
                 'synthia/S/S/RGB/Stereo_Left/Omni_F/0.png', 'cs/x.png'])
    _tree(fast, ['data_stereo_flow/prefilled.txt'])
    got = R.stage_datasets(data, fast, 'synthia')
    # data_scene_flow is not under data; cs belongs to another dataset; data_stereo_flow was there already
    assert got == ['kitti_raw', 'synthia']
    assert _files(fast) == ['data_stereo_flow/prefilled.txt', 'kitti_raw/2011_09_26/d/image_02/data/0.png',
                            'synthia/S/S/RGB/Stereo_Left/Omni_F/0.png']
    assert '>> Copied synthia' in capsys.readouterr().out
    assert R.stage_datasets(data, fast, 'synthia') == []
    assert _files(data) == sorted(['cs/x.png', 'data_stereo_flow/training/colored_0/0_10.png',
                                   'kitti_raw/2011_09_26/d/image_02/data/0.png',
                                   'synthia/S/S/RGB/Stereo_Left/Omni_F/0.png'])


def test_stage_redoes_an_interrupted_copy(tmp_path, monkeypatch):
    data, fast = str(tmp_path / 'data'), str(tmp_path / 'fast')
    _tree(data, ['kitti_raw/a/%d.png' % i for i in range(4)])
    real = shutil.copytree

    def interrupted(src, dst, **kw):
        _tree(dst, ['a/0.png'])
        raise OSError(5, 'Input/output error')
    monkeypatch.setattr(shutil, 'copytree', interrupted)
    with pytest.raises(OSError):
        D.stage(data, fast, ['kitti_raw'])
    assert os.listdir(fast) == ['kitti_raw.partial']      # not taken for a staged dataset
    monkeypatch.setattr(shutil, 'copytree', real)
    assert D.stage(data, fast, ['kitti_raw']) == ['kitti_raw']
    assert os.listdir(fast) == ['kitti_raw']
    assert _files(os.path.join(fast, 'kitti_raw')) == ['a/%d.png' % i for i in range(4)]


def test_stage_copies_on_local_rank_0_only(tmp_path):
    data, fast = str(tmp_path / 'data'), str(tmp_path / 'fast')
    _tree(data, ['kitti_raw/a/0.png'])
    assert R.stage_datasets(data, fast, 'kitti', local_rank=1) == []
    assert not os.path.exists(fast)
    assert R.stage_datasets(data, fast, 'kitti', local_rank=0) == ['kitti_raw']


def test_stage_converts_a_chairs_release_in_data_first(tmp_path):
    cv2 = pytest.importorskip('cv2')
    data, fast = tmp_path / 'data', tmp_path / 'fast'
    release = data / 'flying_chairs' / 'FlyingChairs_release' / 'data'
    release.mkdir(parents=True)
    rng = np.random.default_rng(0)
    for i in (1, 2):
        for k in (1, 2):
            assert cv2.imwrite(str(release / ('%05d_img%d.ppm' % (i, k))),
                               rng.integers(0, 255, (8, 12, 3), dtype=np.uint8))
        np.zeros(3, np.float32).tofile(str(release / ('%05d_flow.flo' % i)))
    (data / 'flying_chairs' / 'FlyingChairs_train_val.txt').write_text('1\n2\n')
    assert R.stage_datasets(str(data), str(fast), 'chairs') == ['flying_chairs']
    for root in (data, fast):
        d = root / 'flying_chairs'
        assert sorted(os.listdir(d / 'image')) == ['00001_img1.png', '00001_img2.png']
        assert sorted(os.listdir(d / 'test_image')) == ['00002_img1.png', '00002_img2.png']
        assert os.listdir(d / 'flow') == ['00002_flow.flo']
