"""Cityscapes sequence layout (reference src/e2eflow/cityscapes/data.py)."""
import os

from ..core.data import Data


class CityscapesData(Data):
    dirs = ['cs']
    layout = ("cs/leftImg8bit_sequence_trainvaltest/<split>/<city>/*.png (the unpacked "
              "leftImg8bit_sequence_trainvaltest.zip of the Cityscapes release)")

    def _check(self):
        self._require(os.path.join('cs', 'leftImg8bit_sequence_trainvaltest'))

    def get_raw_dirs(self):
        """One directory per city of every split, in ``os.listdir`` order as the reference lists them."""
        top_dir = os.path.join(self.current_dir, 'cs', 'leftImg8bit_sequence_trainvaltest')
        dirs = []
        for split in os.listdir(top_dir):
            split_path = os.path.join(top_dir, split)
            for city in os.listdir(split_path):
                dirs.append(os.path.join(split_path, city))
        return dirs
