"""FlyingChairs layout (reference src/e2eflow/chairs/data.py).

Training reads ``flying_chairs/image`` (the training pairs as PNG), evaluation
``flying_chairs/test_image`` (the validation pairs) with ``flying_chairs/flow`` (their ``.flo``
ground truth).  When the release layout is there (``flying_chairs/FlyingChairs_release/data/
*_img{1,2}.ppm, *_flow.flo`` and ``flying_chairs/FlyingChairs_train_val.txt``, one line per pair:
1 = training, 2 = validation) it is converted on construction as ``ChairsData._fetch_if_missing``
does: every ``.ppm`` written losslessly as a ``.png`` into ``image`` or ``test_image`` by its
pair's label, the validation ``.flo`` files copied into ``flow``.  The reference converts on every
construction; here a marker file records a finished conversion, so it runs once (an interrupted
one runs again).  Nothing is deleted, the release directory included."""
import os
import re
import shutil

from ..core.data import Data

OUTPUT_DIRS = ('image', 'test_image', 'flow')
CONVERTED_MARKER = '.converted_from_release'


class ChairsData(Data):
    dirs = ['flying_chairs']
    layout = ('flying_chairs/{image,test_image}/*.png + flying_chairs/flow/*.flo, or the release: '
              'flying_chairs/FlyingChairs_release/data/*.{ppm,flo} + flying_chairs/FlyingChairs_train_val.txt')

    def _check(self):
        self._require('flying_chairs')
        local_path = os.path.join(self.current_dir, 'flying_chairs')
        release = (os.path.isdir(os.path.join(local_path, 'FlyingChairs_release', 'data'))
                   and os.path.isfile(os.path.join(local_path, 'FlyingChairs_train_val.txt')))
        if release and not os.path.isfile(os.path.join(local_path, CONVERTED_MARKER)):
            convert_release(local_path)
        self._require(*(os.path.join('flying_chairs', d) for d in OUTPUT_DIRS))

    def get_raw_dirs(self):
        return [os.path.join(self.current_dir, 'flying_chairs', 'image')]


def convert_release(local_path):
    """chairs/data.py:35-70 on ``local_path`` = ``<data>/flying_chairs``."""
    import cv2
    print('>> converting chairs data to .png')
    data_path = os.path.join(local_path, 'FlyingChairs_release', 'data')
    with open(os.path.join(local_path, 'FlyingChairs_train_val.txt')) as f:
        train_val = [int(line.strip()) == 1 for line in f if line.strip()]
    for d in OUTPUT_DIRS:
        os.makedirs(os.path.join(local_path, d), exist_ok=True)
    im_files = sorted(f for f in os.listdir(data_path) if re.match(r'[0-9]+.*\.ppm', f))
    flow_files = sorted(f for f in os.listdir(data_path) if re.match(r'[0-9]+.*\.flo', f))
    train_val_repeated = [t for t in train_val for _ in range(2)]
    for t, f in zip(train_val_repeated, im_files):
        im = cv2.imread(os.path.join(data_path, f), cv2.IMREAD_UNCHANGED)
        if im is None:
            raise IOError("cannot read image " + os.path.join(data_path, f))
        out = os.path.join(local_path, 'image' if t else 'test_image', os.path.splitext(f)[0] + '.png')
        if not cv2.imwrite(out, im):
            raise IOError("cannot write " + out)
    for t, f in zip(train_val, flow_files):
        if not t:
            shutil.copyfile(os.path.join(data_path, f), os.path.join(local_path, 'flow', f))
    open(os.path.join(local_path, CONVERTED_MARKER), 'w').close()
    print('>> processed chairs data')
