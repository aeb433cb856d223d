"""The supervised fine-tune's host side without a GPU: the input_train_gt file order against the
reference's listing, its crop / decode rules on real PNGs, the hold-out split against
input_train_2015, run.py's kitti_ft configuration, and the new kernel's ptxas report."""
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_supervised.npz')


class _Data:
    def __init__(self, root):
        self.current_dir = str(root)


def test_train_gt_listing_matches_reference(tmp_path):
    from unflow_b200.e2eflow.kitti.input import KITTIInput
    want = json.loads(str(np.load(GOLDEN)['train_gt_listing_json']))
    for top, n in want['pairs'].items():
        img = 'image_2' if top == 'data_scene_flow' else 'colored_0'
        for sub, names in ((img, ['%06d_%d.png' % (i, j) for i in range(n) for j in (10, 11)]),
                           ('flow_occ', ['%06d_10.png' % i for i in range(n)])):
            os.makedirs(tmp_path / top / 'training' / sub)
            for name in names:
                (tmp_path / top / 'training' / sub / name).touch()
    inp = KITTIInput(_Data(tmp_path), batch_size=1, dims=(4, 6), normalize=False)
    got = inp.train_gt_files(want['hold_out'])
    rel = lambda p: os.path.relpath(p, str(tmp_path))
    assert [rel(a) for a, _, _ in got] == want['im1']
    assert [rel(b) for _, b, _ in got] == want['im2']
    assert [rel(g) for _, _, g in got] == want['gt']


def _tree(root, n, h=20, w=30):
    """Both KITTI training sets with n pairs each: real 8-bit frames and 16-bit ground truth."""
    cv2 = pytest.importorskip("cv2")
    from unflow_b200.e2eflow.core import flow_io
    rng = np.random.default_rng(1)
    for top, img in (('data_scene_flow', 'image_2'), ('data_stereo_flow', 'colored_0')):
        tr = root / top / 'training'
        for sub in (img, 'flow_occ', 'flow_noc'):
            (tr / sub).mkdir(parents=True)
        for i in range(n):
            for j in (10, 11):
                assert cv2.imwrite(str(tr / img / ('%06d_%d.png' % (i, j))),
                                   rng.integers(0, 255, (h, w, 3), dtype=np.uint8))
            flow = rng.integers(-3000, 3000, (h, w, 2)).astype(np.float32) / 64.0
            valid = (rng.random((h, w)) < 0.5).astype(np.float32)
            for sub in ('flow_occ', 'flow_noc'):
                flow_io.write_kitti_flow(str(tr / sub / ('%06d_10.png' % i)), flow, valid)


def test_input_train_gt_crop_and_decode(tmp_path):
    from unflow_b200.e2eflow.core import augment
    from unflow_b200.e2eflow.core.flow_io import read_png16
    from unflow_b200.e2eflow.core.input import read_png_image
    from unflow_b200.e2eflow.kitti.input import KITTIInput
    _tree(tmp_path, 3)
    inp = KITTIInput(_Data(tmp_path), batch_size=2, dims=(12, 16), normalize=False)
    triples = inp.train_gt_files(1)
    assert len(triples) == 4
    it = inp.input_train_gt(1, pin=False)
    im1, im2, flow, mask = next(it)
    it.close()
    assert [tuple(t.shape) for t in (im1, im2, flow, mask)] == [(2, 12, 16, 3), (2, 12, 16, 3), (2, 12, 16, 2),
                                                               (2, 12, 16, 1)]
    for k in range(2):
        fn1, fn2, fn_gt = triples[k]
        f1, f2 = read_png_image(fn1), read_png_image(fn2)
        raw = torch.from_numpy(read_png16(fn_gt).astype(np.float32))
        # the window the batch used: find it in frame 1, then it must be the same in frame 2 and the ground truth
        hits = [(y, x) for y in range(20 - 12 + 1) for x in range(30 - 16 + 1)
                if torch.equal(f1[y:y + 12, x:x + 16], im1[k])]
        assert len(hits) == 1
        y, x = hits[0]
        assert torch.equal(f2[y:y + 12, x:x + 16], im2[k])
        win = raw[y:y + 12, x:x + 16]
        assert torch.equal(flow[k], (win[..., 0:2] - 2 ** 15) / 64.0)
        assert torch.equal(mask[k], win[..., 2:3])
        assert set(mask[k].unique().tolist()) <= {0.0, 1.0}
        # the window is random_crop's for the batch's seed
        gen = torch.Generator().manual_seed(0)
        seeds = [int(torch.randint(0, 2 ** 31 - 1, (1,), generator=gen)) for _ in range(2)]
        c1, = augment.random_crop([f1], [12, 16, 3], seed=seeds[k])
        assert torch.equal(c1, im1[k])


def test_train_gt_and_2015_evaluation_split(tmp_path):
    """input_train_gt(40) leaves out exactly the 2015 pairs input_train_2015(40) evaluates on."""
    from unflow_b200.e2eflow.kitti.input import KITTIInput
    n = 45
    for top, img in (('data_scene_flow', 'image_2'), ('data_stereo_flow', 'colored_0')):
        for sub, names in ((img, ['%06d_%d.png' % (i, j) for i in range(n) for j in (10, 11)]),
                           ('flow_occ', ['%06d_10.png' % i for i in range(n)]),
                           ('flow_noc', ['%06d_10.png' % i for i in range(n)])):
            os.makedirs(tmp_path / top / 'training' / sub)
            for name in names:
                (tmp_path / top / 'training' / sub / name).touch()
    inp = KITTIInput(_Data(tmp_path), batch_size=1, dims=(4, 6), normalize=False)
    train = {(a, b) for a, b, _ in inp.train_gt_files(40) if 'data_scene_flow' in a}
    held = set(inp.image_pairs('data_scene_flow/training/image_2', 40))
    occ, _ = inp._flow_files('data_scene_flow/training', 40)
    every = set(inp.image_pairs('data_scene_flow/training/image_2'))
    assert len(train) == n - 40 and len(held) == 40
    assert not (train & held) and (train | held) == every
    # the ground truth of each training pair is its own frame's file; evaluation pairs line up the same way
    for a, b, g in inp.train_gt_files(40):
        assert os.path.basename(a)[:6] == os.path.basename(b)[:6] == os.path.basename(g)[:6]
    for (a, _), g in zip(inp.image_pairs('data_scene_flow/training/image_2', 40), occ):
        assert os.path.basename(a)[:6] == os.path.basename(g)[:6]


CONFIG = """
[dirs]
log = ../log
[run]
batch_size = 4
dataset = kitti_ft
[train]
learning_rate = 1.0e-4
decay_interval = 100000
height = 384
width = 1280
flownet = CSS
train_all = True
save_interval = 5000
[train_kitti]
height = 384
[train_kitti_ft]
height = 320
width = 768
manual_decay_iters = 45000,20000
manual_decay_lrs = 0.5e-5,0.25e-5
"""


def test_kitti_ft_config_resolution(tmp_path):
    """[train] updated by [train_kitti_ft], manual decay lists parsed, num_iters their sum, and the
    manual schedule in force (run.py:175-180, train.py:225-236)."""
    from unflow_b200 import run as R
    from unflow_b200.e2eflow.core.train import learning_rate_at
    ini = tmp_path / 'config.ini'
    ini.write_text(CONFIG)
    cfg = R.config_dict(str(ini))
    params = dict(cfg['train'])
    params.update(cfg.get('train_' + cfg['run']['dataset'], {}))
    R.convert_input_strings(params, cfg['dirs'])
    assert (params['height'], params['width'], params['flownet'], params['train_all']) == (320, 768, 'CSS', True)
    assert params['manual_decay_iters'] == [45000, 20000] and params['manual_decay_lrs'] == [0.5e-5, 0.25e-5]
    assert params['num_iters'] == 65000 and params['save_interval'] == 5000
    assert learning_rate_at(0, params) == 0.5e-5 and learning_rate_at(45000, params) == 0.5e-5
    assert learning_rate_at(45001, params) == 0.25e-5 and learning_rate_at(65000, params) == 0.25e-5


def test_run_rejects_unimplemented_datasets():
    from unflow_b200 import run as R
    with pytest.raises(SystemExit):
        R.kitti_inputs({'data': '/nonexistent'}, {}, {}, 'chairs', 1, 1, 0, 1)


def test_supervised_loss_kernel_ptxas_no_spills(tmp_path):
    from unflow_b200 import build
    nvcc = build._nvcc()
    nvcc = nvcc if os.path.isabs(nvcc) and os.path.exists(nvcc) else shutil.which(nvcc)
    if not nvcc:
        pytest.skip("nvcc not found")
    cmd = [nvcc] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.CSRC, "supervised_loss.cu"),
                                       "-o", str(tmp_path / "supervised_loss.o")]
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert p.returncode == 0, p.stdout
    name, seen = None, set()
    for line in p.stdout.splitlines():
        m = re.search(r"Function properties for (\S+)", line)
        if m:
            name = m.group(1)
            continue
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and name and "supervised_loss" in name:
            assert m.group(1) == "0" and m.group(2) == "0", "%s spills: %s" % (name, line.strip())
            seen.add("fwd" if "fwd" in name else "bwd")
    assert seen == {"fwd", "bwd"}
