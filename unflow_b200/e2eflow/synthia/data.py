"""SYNTHIA-SEQS layout (reference src/e2eflow/synthia/data.py)."""
import os

from ..core.data import Data


class SynthiaData(Data):
    dirs = ['synthia']
    layout = 'synthia/<SEQ>/<SEQ>/RGB/Stereo_Left/<view>/*.png, e.g. SEQ = SYNTHIA-SEQS-01-SUMMER, view = Omni_F'

    def _check(self):
        self._require('synthia')

    def get_raw_dirs(self):
        """Every view of every sequence present, in ``os.listdir`` order as the reference lists them."""
        root_dir = os.path.join(self.current_dir, 'synthia')
        dirs = []
        for seq in os.listdir(root_dir):
            seq_dir = os.path.join(root_dir, seq, seq, 'RGB', 'Stereo_Left')
            for view in os.listdir(seq_dir):
                dirs.append(os.path.join(seq_dir, view))
        return dirs
