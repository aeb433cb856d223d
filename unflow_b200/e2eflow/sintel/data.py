"""MPI Sintel layout (reference src/e2eflow/sintel/data.py)."""
import os

from ..core.data import Data


class SintelData(Data):
    dirs = ['sintel']
    layout = ('sintel/{training,test}/{clean,final}/<seq>/frame_*.png, '
              'sintel/training/{flow,invalid,occlusions}/<seq>/frame_*.{flo,png} (the unpacked MPI-Sintel-complete.zip)')

    def _check(self):
        self._require('sintel')

    def get_raw_dirs(self):
        dirs = []
        for folder in ['training/clean', 'training/final', 'test/clean', 'test/final']:
            top_dir = os.path.join(self.current_dir, 'sintel', folder)
            for sub_dir in os.listdir(top_dir):
                dirs.append(os.path.join(top_dir, sub_dir))
        return dirs
