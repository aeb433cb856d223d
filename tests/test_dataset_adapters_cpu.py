"""FlyingChairs, Sintel, Middlebury, SYNTHIA and Cityscapes adapters (reference
src/e2eflow/{chairs,sintel,middlebury,synthia,cityscapes}/, core/input.py), the multi-threaded batch
decode, and the dataset branches of ``unflow_b200.run`` / ``unflow_b200.eval`` on the CPU.

The file lists are compared with what the reference's own adapters made of the same tree
(tests/golden/reference_datasets.json, written by tests/golden/make_reference_datasets.py)."""
import argparse
import json
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from unflow_b200 import eval as E
from unflow_b200 import run as R
from unflow_b200.e2eflow.chairs.data import ChairsData
from unflow_b200.e2eflow.chairs.input import ChairsInput
from unflow_b200.e2eflow.cityscapes.data import CityscapesData
from unflow_b200.e2eflow.core import flow_io
from unflow_b200.e2eflow.core.input import resize_image_with_crop_or_pad
from unflow_b200.e2eflow.kitti.input import KITTIInput
from unflow_b200.e2eflow.middlebury.data import MiddleburyData
from unflow_b200.e2eflow.middlebury.input import MiddleburyInput
from unflow_b200.e2eflow.sintel.data import SintelData
from unflow_b200.e2eflow.sintel.input import SintelInput
from unflow_b200.e2eflow.synthia.data import SynthiaData

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(HERE, "golden", "reference_datasets.json")) as f:
        return json.load(f)


def _write_ppm(path, i):
    px = np.random.default_rng(i).integers(0, 256, (5, 7, 3), dtype=np.uint8)
    with open(path, 'wb') as f:
        f.write(b'P6\n7 5\n255\n' + px.tobytes())


def _golden_tree(root, spec):
    for rel in spec['files']:
        os.makedirs(os.path.dirname(os.path.join(root, rel)), exist_ok=True)
        open(os.path.join(root, rel), 'w').close()
    for i, rel in enumerate(spec['ppm']):
        os.makedirs(os.path.dirname(os.path.join(root, rel)), exist_ok=True)
        _write_ppm(os.path.join(root, rel), i)
    with open(os.path.join(root, 'flying_chairs', 'FlyingChairs_train_val.txt'), 'w') as f:
        f.write(''.join('%d\n' % t for t in spec['chairs_labels']))


def test_file_lists_match_the_reference_adapters(golden, tmp_path):
    root = str(tmp_path)
    _golden_tree(root, golden['tree'])
    dims = tuple(golden['dims'])
    rel = lambda files: [os.path.relpath(f, root) for f in files]
    unzip = lambda pairs: [rel(a for a, _ in pairs), rel(b for _, b in pairs)]

    cdata = ChairsData(root)
    g = golden['chairs']
    for d in ('image', 'test_image', 'flow'):
        assert sorted(os.listdir(os.path.join(root, 'flying_chairs', d))) == g[d], d
    for shift in (0, 3):
        pairs = ChairsInput(cdata, 2, dims, normalize=False).raw_pairs(swap_images=False, sequence=False, shift=shift)
        assert unzip(pairs) == g['raw_shift%d' % shift], shift
    ci = ChairsInput(cdata, 1, dims, normalize=False)
    assert unzip(ci.image_pairs('flying_chairs/test_image')) + [rel(ci.flow_files())] == g['test']

    si = SintelInput(SintelData(root), 1, dims, normalize=False)
    truth = [rel(x) for x in si.truth_files()]
    for variant in ('train_clean', 'train_final', 'test_clean', 'test_final'):
        pas = variant.split('_')[1]
        top = 'training' if variant.startswith('train') else 'test'
        got = unzip(si.sequence_pairs('sintel/%s/%s' % (top, pas)))
        assert got + (truth if top == 'training' else []) == golden['sintel'][variant], variant
    assert sorted(rel(SintelData(root).get_raw_dirs())) == golden['sintel']['raw_dirs']

    mi = MiddleburyInput(MiddleburyData(root), 1, dims, normalize=False)
    from unflow_b200.e2eflow.middlebury.data import NO_GROUND_TRUTH
    assert unzip(mi.sequence_pairs('middlebury/other-data', exclude=NO_GROUND_TRUTH)) + [rel(mi.flow_files())] \
        == golden['middlebury']['train']
    assert unzip(mi.sequence_pairs('middlebury/eval-data')) == golden['middlebury']['test']
    assert os.path.isdir(os.path.join(root, 'middlebury', 'other-data', 'Beanbags'))     # skipped, not deleted

    assert sorted(rel(SynthiaData(root).get_raw_dirs())) == golden['synthia']['raw_dirs']
    cs_dirs = CityscapesData(root).get_raw_dirs()
    assert sorted(rel(cs_dirs)) == golden['cityscapes']['raw_dirs']

    class Data:
        current_dir = root

        def get_raw_dirs(self):
            return sorted(cs_dirs)

    for shift in (0, 5):
        pairs = KITTIInput(Data(), 2, dims, normalize=False, skipped_frames=False).raw_pairs(
            swap_images=False, skip=[0, 1], shift=shift)
        assert unzip(pairs) == golden['cityscapes']['raw_skip01_shift%d' % shift], shift


def test_missing_directories_name_the_layout(tmp_path):
    for cls, what in ((SynthiaData, 'Stereo_Left'), (CityscapesData, 'leftImg8bit_sequence_trainvaltest'),
                      (ChairsData, 'FlyingChairs_release'), (SintelData, 'occlusions'),
                      (MiddleburyData, 'other-gt-flow')):
        with pytest.raises(FileNotFoundError, match=what):
            cls(str(tmp_path))
    assert os.listdir(str(tmp_path)) == []           # nothing created, nothing fetched


def test_chairs_conversion_is_lossless_and_keeps_the_release(tmp_path):
    root = tmp_path / "flying_chairs"
    data = root / "FlyingChairs_release" / "data"
    data.mkdir(parents=True)
    rng = np.random.default_rng(3)
    labels = [2, 1, 1, 2]
    ims = {}
    for i in range(len(labels)):
        for j in (1, 2):
            im = rng.integers(0, 256, (384, 512, 3), dtype=np.uint8)
            name = '%05d_img%d' % (i + 1, j)
            assert cv2.imwrite(str(data / (name + '.ppm')), im)
            ims[name] = im
        flow = rng.standard_normal((384, 512, 2)).astype(np.float32)
        flow_io.write_flo(str(data / ('%05d_flow.flo' % (i + 1))), flow)
    (root / "FlyingChairs_train_val.txt").write_text(''.join('%d\n' % t for t in labels))
    ChairsData(str(tmp_path))
    assert sorted(os.listdir(root / "image")) == ['00002_img1.png', '00002_img2.png', '00003_img1.png', '00003_img2.png']
    assert sorted(os.listdir(root / "test_image")) == ['00001_img1.png', '00001_img2.png', '00004_img1.png', '00004_img2.png']
    assert sorted(os.listdir(root / "flow")) == ['00001_flow.flo', '00004_flow.flo']
    for d in ('image', 'test_image'):
        for f in os.listdir(root / d):
            png = cv2.imread(str(root / d / f), cv2.IMREAD_UNCHANGED)
            ppm = cv2.imread(str(data / f.replace('.png', '.ppm')), cv2.IMREAD_UNCHANGED)
            assert np.array_equal(png, ppm) and np.array_equal(png, ims[f[:-4]]), f
    assert (data / "00001_flow.flo").read_bytes() == (root / "flow" / "00001_flow.flo").read_bytes()
    assert len(os.listdir(data)) == 12                    # the release is kept
    # converted once: a second construction leaves the converted files alone
    stamp = os.path.getmtime(root / "image" / "00002_img1.png")
    ChairsData(str(tmp_path))
    assert os.path.getmtime(root / "image" / "00002_img1.png") == stamp


def _sintel_tree(root, h=20, w=36, frames=3):
    """One training sequence; masks stored as 0/255.  Returns (flow, invalid, occ) of every pair."""
    rng = np.random.default_rng(1)
    truth = []
    for pas in ('clean', 'final'):
        for top, seq in (('training', 'alley_1'), ('test', 'cave_3')):
            d = os.path.join(root, 'sintel', top, pas, seq)
            os.makedirs(d)
            for i in range(frames):
                cv2.imwrite(os.path.join(d, 'frame_%04d.png' % (i + 1)), rng.integers(0, 255, (h, w, 3), dtype=np.uint8))
    for sub in ('flow', 'invalid', 'occlusions'):
        os.makedirs(os.path.join(root, 'sintel', 'training', sub, 'alley_1'))
    for i in range(frames):
        inv = np.zeros((h, w), np.uint8)
        inv[:, :4 + i] = 255
        cv2.imwrite(os.path.join(root, 'sintel', 'training', 'invalid', 'alley_1', 'frame_%04d.png' % (i + 1)), inv)
        if i == frames - 1:
            break
        occ = np.zeros((h, w), np.uint8)
        occ[:5 + 2 * i] = 255
        cv2.imwrite(os.path.join(root, 'sintel', 'training', 'occlusions', 'alley_1', 'frame_%04d.png' % (i + 1)), occ)
        flow = np.stack([np.full((h, w), 2.5 + i), np.full((h, w), -1.0)], 2).astype(np.float32)
        flow_io.write_flo(os.path.join(root, 'sintel', 'training', 'flow', 'alley_1', 'frame_%04d.flo' % (i + 1)), flow)
        truth.append((flow, inv > 0, occ > 0))
    return truth


def test_sintel_masks_from_0_255_files_binarise(tmp_path):
    truth = _sintel_tree(str(tmp_path))
    si = SintelInput(SintelData(str(tmp_path)), 1, (32, 48), normalize=False)
    items = list(si.input_train_clean())
    assert len(items) == len(truth) == 2
    for item, (flow, inv, occ) in zip(items, truth):
        assert len(item) == 7 and tuple(item[2][0].tolist()) == (20, 36, 3)
        flow_occ, mask_occ, flow_noc, mask_noc = [resize_image_with_crop_or_pad(t[0], 20, 36).numpy() for t in item[3:]]
        assert set(np.unique(mask_occ)) <= {0.0, 1.0} and set(np.unique(mask_noc)) <= {0.0, 1.0}
        assert np.array_equal(mask_occ[..., 0], (~inv).astype(np.float32))
        assert np.array_equal(mask_noc[..., 0], ((~inv) & (~occ)).astype(np.float32))
        assert np.array_equal(flow_occ, flow)
        assert np.array_equal(flow_noc, flow * (~occ)[..., None])
    assert len(list(si.input_test_final())) == 2 and len(list(si.input_test_final())[0]) == 3


def test_middlebury_flo_unknowns_are_masked(tmp_path):
    root = str(tmp_path)
    rng = np.random.default_rng(2)
    flow = rng.standard_normal((30, 40, 2)).astype(np.float32)
    flow[3:6, 7:9, 0] = 1e10
    flow[10, :, 1] = 1.7e9
    for seq in ('Grove2', 'Beanbags'):
        d = os.path.join(root, 'middlebury', 'other-data', seq)
        os.makedirs(d)
        for n in (10, 11):
            cv2.imwrite(os.path.join(d, 'frame%d.png' % n), rng.integers(0, 255, (30, 40, 3), dtype=np.uint8))
    os.makedirs(os.path.join(root, 'middlebury', 'other-gt-flow', 'Grove2'))
    flow_io.write_flo(os.path.join(root, 'middlebury', 'other-gt-flow', 'Grove2', 'flow10.flo'), flow)
    items = list(MiddleburyInput(MiddleburyData(root), 1, (32, 48), normalize=False).input_train())
    assert len(items) == 1                                       # Beanbags (no ground truth) skipped
    mask = resize_image_with_crop_or_pad(items[0][4][0], 30, 40)[..., 0].numpy()
    want = np.ones((30, 40), np.float32)
    want[3:6, 7:9] = 0
    want[10, :] = 0
    assert np.array_equal(mask, want)


def _synthia_tree(root, frames=5, h=40, w=60):
    rng = np.random.default_rng(4)
    for seq, views in (('SYNTHIA-SEQS-01-SUMMER', ('Omni_F', 'Omni_B')), ('SYNTHIA-SEQS-02-WINTER', ('Omni_L',))):
        for view in views:
            d = os.path.join(root, 'synthia', seq, seq, 'RGB', 'Stereo_Left', view)
            os.makedirs(d)
            for i in range(frames):
                cv2.imwrite(os.path.join(d, '%06d.png' % i), rng.integers(0, 255, (h, w, 3), dtype=np.uint8))


def test_threaded_decode_gives_the_same_batches(tmp_path):
    _synthia_tree(str(tmp_path))
    data = SynthiaData(str(tmp_path))
    streams = [KITTIInput(data, 3, (24, 32), normalize=n, num_threads=t).input_raw(swap_images=False, shift=2, pin=False)
               for t, n in ((1, False), (4, False), (4, True))]
    try:
        for _ in range(5):                        # 15 pairs of 12: wraps around
            one, four, four_norm = [next(s) for s in streams]
            assert all(torch.equal(a, b) for a, b in zip(one, four))
            assert not torch.equal(one[0], four_norm[0])
    finally:
        for s in streams:
            s.close()


def _ckpt_config(tmp_path, data_dir):
    from unflow_b200.e2eflow.core import tf_checkpoint as ck
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    ini = tmp_path / "config.ini"
    ini.write_text("[dirs]\nlog = %s/log\ncheckpoints = %s/ckpts\ndata = %s\n[run]\nbatch_size = 4\n[train]\n"
                   "flownet = s\nternary_weight = 1.0\n" % (tmp_path, tmp_path, data_dir))
    ck.save_variables(FlowNetVariables("s", False, seed=5), str(tmp_path / "ckpts" / "exE" / "model.ckpt-3"))
    return str(ini)


def _truth_stub(flows, dims):
    """An estimator that returns the (constant) ground-truth flow of each pair in turn, at the network
    size, scaled so that ``resize_output_flow`` brings it back to the file size exactly."""
    it = iter(flows)

    def make(params, normalization, variables):
        def fn(im1, im2):
            assert tuple(im1.shape) == (1,) + dims + (3,)
            (u, v), (h, w) = next(it)
            out = torch.zeros(1, dims[0], dims[1], 2)
            out[..., 0], out[..., 1] = u * dims[1] / w, v * dims[0] / h
            return out, -out
        return fn
    return make


def _args(ini, dataset, variant, out, num=-1):
    return argparse.Namespace(dataset=dataset, variant=variant, ex='exE', num=num, gpu='0', output_benchmark=True,
                              output_visual=False, output_backward=False, output_png=True, config=ini, out=out)


def test_run_eval_on_chairs_sintel_and_middlebury(tmp_path, capsys, monkeypatch):
    data = tmp_path / "data"
    ini = _ckpt_config(tmp_path, str(data))
    # FlyingChairs: two validation pairs at the network size 384x512, constant flows
    ch = data / "flying_chairs"
    for d in ('image', 'test_image', 'flow'):
        (ch / d).mkdir(parents=True)
    rng = np.random.default_rng(5)
    for i, (u, v) in enumerate(((1.5, -2.0), (0.25, 3.0))):
        for j in (1, 2):
            cv2.imwrite(str(ch / 'test_image' / ('%05d_img%d.png' % (i, j))), rng.integers(0, 255, (384, 512, 3), dtype=np.uint8))
        f = np.stack([np.full((384, 512), u), np.full((384, 512), v)], 2).astype(np.float32)
        f[:2, :3, 0] = 1e10                     # unknown: masked out
        flow_io.write_flo(str(ch / 'flow' / ('%05d_flow.flo' % i)), f)
    res = E.run_eval(_args(ini, 'chairs', 'test', str(tmp_path / "out_c")), torch.device('cpu'),
                     make_flow_fn=_truth_stub([((1.5, -2.0), (384, 512)), ((0.25, 3.0), (384, 512))], (384, 512)))
    assert abs(res['exE']['EPE_all']) < 1e-4 and set(res['exE']) == {'EPE_all'}
    assert sorted(os.listdir(tmp_path / "out_c" / "exE")) == ['000000_10.png', '000001_10.png', 'config.ini']
    # Sintel: 0/255 masks, 20x36 frames evaluated at 512x1024
    truth = _sintel_tree(str(data))
    stub = _truth_stub([((float(f[0, 0, 0]), float(f[0, 0, 1])), (20, 36)) for f, _, _ in truth], (512, 1024))
    res = E.run_eval(_args(ini, 'sintel', 'train_clean', str(tmp_path / "out_s")), torch.device('cpu'), make_flow_fn=stub)
    assert set(res['exE']) == {'EPE_noc', 'EPE_all', 'outliers_noc', 'outliers_all'}
    assert all(abs(v) < 1e-4 for v in res['exE'].values()), res
    assert sorted(os.listdir(tmp_path / "out_s" / "exE")) == ['000000_10.png', '000001_10.png', 'config.ini']
    flow, _ = flow_io.read_kitti_flow(str(tmp_path / "out_s" / "exE" / "000001_10.png"))
    assert flow.shape == (20, 36, 2) and np.allclose(flow[..., 0], 3.5, atol=1 / 64)
    # Middlebury: test variant (no ground truth) at 512x640, --num -1 = all pairs (the reference's 12 at most)
    for seq in ('Army', 'Mequon'):
        d = data / "middlebury" / "eval-data" / seq
        d.mkdir(parents=True)
        for n in (10, 11):
            cv2.imwrite(str(d / ('frame%d.png' % n)), rng.integers(0, 255, (388, 584, 3), dtype=np.uint8))
    nums = []
    loop = E.evaluate_examples
    monkeypatch.setattr(E, 'evaluate_examples', lambda *a, **k: nums.append(k['num']) or loop(*a, **k))
    res = E.run_eval(_args(ini, 'mdb', 'test', str(tmp_path / "out_m")), torch.device('cpu'),
                     make_flow_fn=_truth_stub([((0.0, 0.0), (388, 584))] * 2, (512, 640)))
    assert res['exE'] == {} and nums == [12]
    assert sorted(os.listdir(tmp_path / "out_m" / "exE")) == ['000000_10.png', '000001_10.png', 'config.ini']
    assert "-- evaluating: on -1 pairs from mdb/test" in capsys.readouterr().out


def test_eval_rejects_bad_dataset_variant_combinations():
    for dataset, variant in (('chairs', 'train_2012'), ('sintel', 'test'), ('mdb', 'train_clean'),
                             ('kitti', 'test'), ('synthia', 'train')):
        with pytest.raises(SystemExit):
            E.check_variant(dataset, variant)
        with pytest.raises(SystemExit):
            E.main(['--dataset', dataset, '--variant', variant])
    E.check_variant('sintel', 'test_final')
    E.check_variant('mdb', 'train')


def test_run_dispatcher_builds_each_dataset_input(tmp_path, capsys):
    data = tmp_path / "data"
    _synthia_tree(str(data), frames=4, h=40, w=60)
    rng = np.random.default_rng(6)
    for city, snippets in (('aachen', 2), ('bochum', 1)):
        d = data / "cs" / "leftImg8bit_sequence_trainvaltest" / "train" / city
        d.mkdir(parents=True)
        for s in range(snippets):
            for f in range(3):
                cv2.imwrite(str(d / ('%s_%06d_%06d_leftImg8bit.png' % (city, s, 17 + f))),
                            rng.integers(0, 255, (40, 60, 3), dtype=np.uint8))
    ch = data / "flying_chairs"
    for d in ('image', 'test_image', 'flow'):
        (ch / d).mkdir(parents=True)
    chairs_ims = []
    for i in range(6):
        im = rng.integers(0, 255, (24, 32, 3), dtype=np.uint8)
        cv2.imwrite(str(ch / 'image' / ('%05d_img%d.png' % (i // 2, i % 2 + 1))), im)
        chairs_ims.append(im)
    dirs = {'data': str(data)}
    run_config = {'batch_size': 2, 'num_input_threads': 2}
    params = {'height': 24, 'width': 32}
    # cityscapes, skip=[0, 1]: aachen's 6 frames give 5 pairs at step 1 and 2 at step 2, bochum's 3 give 2 + 1
    expected = {'chairs': 3, 'synthia': 9, 'cityscapes': 5 + 2 + 2 + 1}
    for ds in ('chairs', 'synthia', 'cityscapes'):
        batches, eval_input = R.dataset_inputs(dirs, run_config, params, ds, 2, 1, 0, 1)
        try:
            a, b = next(batches)
        finally:
            batches.close()
        assert a.shape == b.shape == (2, 24, 32, 3) and eval_input is None
        assert "Training on {} frame pairs.".format(expected[ds]) in capsys.readouterr().out, ds
        if ds == 'chairs':                       # no crop: the pair's own pixels (RGB)
            pairs = ChairsInput(ChairsData(str(data)), 2, (24, 32)).raw_pairs(swap_images=False, sequence=False)
            capsys.readouterr()
            want = cv2.imread(pairs[0][0])[:, :, ::-1].astype(np.float32)
            assert np.array_equal(a[0].numpy(), want)
    # the KITTI 2012 training set under [dirs] data is the evaluation input of every dataset
    (data / "data_stereo_flow" / "training" / "flow_occ").mkdir(parents=True)
    batches, eval_input = R.dataset_inputs(dirs, run_config, params, 'synthia', 2, 1, 0, 1)
    batches.close()
    assert isinstance(eval_input, KITTIInput) and eval_input.dims == (384, 1280)
    with pytest.raises(SystemExit):
        R.dataset_inputs(dirs, run_config, params, 'sintel', 2, 1, 0, 1)
    with pytest.raises(FileNotFoundError):
        R.dataset_inputs({'data': str(tmp_path / "empty")}, run_config, params, 'chairs', 2, 1, 0, 1)
