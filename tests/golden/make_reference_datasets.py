#!/usr/bin/env python
"""Run the reference's OWN dataset adapters (src/e2eflow/{chairs,sintel,middlebury,synthia,
cityscapes}/ and core/input.py, unmodified) on a synthetic directory tree under the TensorFlow-API
stand-in of tests/golden/tf_shim.py and store which files they pair, in which order, in
tests/golden/reference_datasets.json.

    python tests/golden/make_reference_datasets.py      (needs the reference source tree)

Stub queues record the file lists (``string_input_producer``); ``WholeFileReader``, ``substr`` and
``decode_raw`` only carry shapes.  ``rarfile`` and ``matplotlib.image`` (imported by the reference's
``core/data.py``, not installed) are empty stand-ins.  Nothing can reach a network: every
``urllib.request`` entry point the reference uses, ``Data._download_and_extract`` and socket
connections raise, and the tree holds every directory whose absence would make the reference
download (``SYNTHIA-SEQS-01-SUMMER`` for ``development=True`` included).

Stored: the tree itself (``files``: relative paths; ``ppm``: the FlyingChairs release images, which
must be real images for the conversion), and
  chairs      the conversion (names in ``image``, ``test_image``, ``flow``), ``input_raw`` pairs
              (``sequence=False``, shifts 0 and 3), ``input_test`` image and flow lists;
  sintel      train (clean, final) and test (clean, final) pairs; flow / invalid / occlusion lists;
  middlebury  train and test pairs, train flows (after the reference deleted the sequences without
              ground truth);
  synthia, cityscapes  ``get_raw_dirs`` (as sorted lists: the reference keeps ``os.listdir``
              order); Cityscapes ``input_raw(skip=[0, 1])`` pairs (shifts 0 and 5) over a stub
              ``Data`` listing the city directories sorted.
tests/test_dataset_adapters_cpu.py compares the product's adapters with these lists.
"""
import importlib
import json
import os
import socket
import sys
import tempfile
import types
import urllib.request

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_reference_run import load_reference  # noqa: E402
import tf_shim  # noqa: E402

DIMS = (4, 6)


def _no_network(*a, **k):
    raise RuntimeError("make_reference_datasets: the reference tried to reach a network")


class _NoNetworkOpener:
    def __init__(self, *a, **k):
        _no_network()


def seal_network():
    for name in ('urlretrieve', 'urlopen', 'build_opener'):
        setattr(urllib.request, name, _no_network)
    urllib.request.FancyURLopener = urllib.request.URLopener = _NoNetworkOpener
    socket.socket.connect = socket.socket.connect_ex = _no_network
    socket.create_connection = _no_network


def tree_spec():
    """Relative file paths of the fixture tree; the chairs release images are listed apart."""
    files = []
    synthia = {'SYNTHIA-SEQS-01-SUMMER': {'Omni_F': 4, 'Omni_B': 3}, 'SYNTHIA-SEQS-04-WINTER': {'Omni_L': 3}}
    for seq, views in synthia.items():
        for view, n in views.items():
            files += ['synthia/%s/%s/RGB/Stereo_Left/%s/%06d.png' % (seq, seq, view, i) for i in range(n)]
    cities = {'train/aachen': (2, 3), 'train/bochum': (1, 4), 'val/frankfurt': (2, 2)}
    for path, (snippets, frames) in cities.items():
        city = path.split('/')[1]
        files += ['cs/leftImg8bit_sequence_trainvaltest/%s/%s_%06d_%06d_leftImg8bit.png' % (path, city, s, 17 + f)
                  for s in range(snippets) for f in range(frames)]
    labels = [1, 2, 1, 1, 2, 1, 2]
    ppm = ['flying_chairs/FlyingChairs_release/data/%05d_img%d.ppm' % (i + 1, j)
           for i in range(len(labels)) for j in (1, 2)]
    files += ['flying_chairs/FlyingChairs_release/data/%05d_flow.flo' % (i + 1) for i in range(len(labels))]
    sintel_train = {'alley_1': 4, 'bamboo_2': 3, 'market_5': 2}
    for pas in ('clean', 'final'):
        for seq, n in sintel_train.items():
            files += ['sintel/training/%s/%s/frame_%04d.png' % (pas, seq, i + 1) for i in range(n)]
        for seq, n in {'ambush_1': 3, 'cave_3': 2}.items():
            files += ['sintel/test/%s/%s/frame_%04d.png' % (pas, seq, i + 1) for i in range(n)]
    for seq, n in sintel_train.items():
        files += ['sintel/training/flow/%s/frame_%04d.flo' % (seq, i + 1) for i in range(n - 1)]
        files += ['sintel/training/invalid/%s/frame_%04d.png' % (seq, i + 1) for i in range(n)]
        files += ['sintel/training/occlusions/%s/frame_%04d.png' % (seq, i + 1) for i in range(n - 1)]
    for seq in ('Dimetrodon', 'Grove2', 'Beanbags', 'RubberWhale'):
        files += ['middlebury/other-data/%s/frame%02d.png' % (seq, i) for i in (10, 11)]
    files += ['middlebury/other-data/Hydrangea/frame%02d.png' % i for i in (9, 10, 11)]
    for seq in ('Dimetrodon', 'Grove2', 'Hydrangea', 'RubberWhale'):
        files += ['middlebury/other-gt-flow/%s/flow%02d.flo' % (seq, i) for i in
                  ((9, 10) if seq == 'Hydrangea' else (10,))]
    for seq in ('Army', 'Mequon'):
        files += ['middlebury/eval-data/%s/frame%02d.png' % (seq, i) for i in (10, 11)]
    return {'files': files, 'ppm': ppm, 'chairs_labels': labels}


def build_tree(root, spec, write_ppm):
    """Empty files for ``spec['files']``, ``write_ppm(path, index)`` for the chairs images, the
    train / val list."""
    for rel in spec['files']:
        os.makedirs(os.path.dirname(os.path.join(root, rel)), exist_ok=True)
        open(os.path.join(root, rel), 'w').close()
    for i, rel in enumerate(spec['ppm']):
        os.makedirs(os.path.dirname(os.path.join(root, rel)), exist_ok=True)
        write_ppm(os.path.join(root, rel), i)
    with open(os.path.join(root, 'flying_chairs', 'FlyingChairs_train_val.txt'), 'w') as f:
        f.write(''.join('%d\n' % t for t in spec['chairs_labels']))


def write_ppm(path, i):
    """A small binary PPM (P6) of seeded pixels."""
    px = np.random.default_rng(i).integers(0, 256, (5, 7, 3), dtype=np.uint8)
    with open(path, 'wb') as f:
        f.write(b'P6\n7 5\n255\n' + px.tobytes())


def extend_shim(tf):
    """What the ``.flo`` / mask readers call beyond the stand-in: ``substr`` / ``decode_raw`` carry
    the header fields and payload size, ``to_float``."""
    def substr(value, pos, length):
        return ('substr', int(pos), length)

    def decode_raw(s, out_type=None):
        _, pos, length = s
        h, w, _ = tf_shim.STATE.decode_shape
        if pos == 4:
            return tf_shim._t([w], 'int32')
        if pos == 8:
            return tf_shim._t([h], 'int32')
        return tf_shim._t(np.zeros(int(length) // 4, np.float32))

    tf.substr, tf.decode_raw = substr, decode_raw
    tf.to_float = lambda x: tf_shim.cast(x, 'float32')
    tf.int32 = 'int32'


def main():
    seal_network()
    for name in ('rarfile', 'matplotlib', 'matplotlib.image'):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules['matplotlib'].image = sys.modules['matplotlib.image']
    tf, ref = load_reference()
    extend_shim(tf)
    mods = {n: importlib.import_module('e2eflow.' + n) for n in
            ('core.data', 'chairs.data', 'chairs.input', 'sintel.data', 'sintel.input', 'middlebury.data',
             'middlebury.input', 'synthia.data', 'cityscapes.data')}
    for m in mods.values():
        assert os.path.realpath(m.__file__).startswith(os.path.realpath(os.path.dirname(os.path.dirname(
            ref['losses'].__file__)))), m.__file__
        for attr in ('urlretrieve', 'FancyURLopener'):
            if hasattr(m, attr):
                setattr(m, attr, _NoNetworkOpener if attr == 'FancyURLopener' else _no_network)
    mods['core.data'].Data._download_and_extract = _no_network

    spec = tree_spec()
    out = {'tree': spec, 'dims': list(DIMS)}
    with tempfile.TemporaryDirectory() as root:
        build_tree(root, spec, write_ppm)
        rel = lambda files: [os.path.relpath(str(f), root) for f in files]

        def queues():
            return [rel(q) for q in tf_shim.STATE.queues]

        def reset(shape=(DIMS[0], DIMS[1], 3)):
            tf_shim.STATE.reset({})
            tf_shim.STATE.decode_shape = shape

        # ---- FlyingChairs --------------------------------------------------------------------------
        cdata = mods['chairs.data'].ChairsData(root, development=True)
        chairs = {d: sorted(os.listdir(os.path.join(root, 'flying_chairs', d))) for d in ('image', 'test_image', 'flow')}
        for shift in (0, 3):
            reset()
            mods['chairs.input'].ChairsInput(cdata, batch_size=2, dims=DIMS, normalize=False).input_raw(
                swap_images=False, shift=shift)
            chairs['raw_shift%d' % shift] = queues()[:2]
        reset()
        mods['chairs.input'].ChairsInput(cdata, batch_size=1, dims=DIMS, normalize=False).input_test()
        chairs['test'] = queues()[:3]                   # frame 1, frame 2, flow
        out['chairs'] = chairs

        # ---- Sintel -----------------------------------------------------------------------------------
        sdata = mods['sintel.data'].SintelData(root, development=True)
        sintel = {}
        for variant in ('train_clean', 'train_final', 'test_clean', 'test_final'):
            reset()
            getattr(mods['sintel.input'].SintelInput(sdata, batch_size=1, dims=DIMS, normalize=False),
                    'input_' + variant)()
            sintel[variant] = queues()                  # frame 1, frame 2[, flow, invalid, occlusions]
        sintel['raw_dirs'] = sorted(rel(sdata.get_raw_dirs()))
        out['sintel'] = sintel

        # ---- Middlebury (its Data deletes the sequences without ground truth) ------------------------
        mdata = mods['middlebury.data'].MiddleburyData(root, development=True)
        mdb = {}
        for variant in ('train', 'test'):
            reset()
            getattr(mods['middlebury.input'].MiddleburyInput(mdata, batch_size=1, dims=DIMS, normalize=False),
                    'input_' + variant)()
            mdb[variant] = queues()                     # frame 1, frame 2[, flow]
        out['middlebury'] = mdb

        # ---- SYNTHIA, Cityscapes ---------------------------------------------------------------------
        out['synthia'] = {'raw_dirs': sorted(rel(mods['synthia.data'].SynthiaData(root, development=True).get_raw_dirs()))}
        cs_dirs = mods['cityscapes.data'].CityscapesData(root, development=True).get_raw_dirs()
        out['cityscapes'] = {'raw_dirs': sorted(rel(cs_dirs))}

        class Data:
            current_dir = root

            def get_raw_dirs(self):
                return sorted(cs_dirs)

        for shift in (0, 5):
            reset()
            ref['kitti_input'].KITTIInput(Data(), batch_size=2, dims=DIMS, normalize=False, skipped_frames=False) \
                .input_raw(swap_images=False, center_crop=True, skip=[0, 1], shift=shift, needs_crop=False)
            out['cityscapes']['raw_skip01_shift%d' % shift] = queues()[:2]

    path = os.path.join(HERE, 'reference_datasets.json')
    with open(path, 'w') as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write('\n')
    print("wrote %s (%.1f KB)" % (path, os.path.getsize(path) / 1024.0))


if __name__ == '__main__':
    main()
