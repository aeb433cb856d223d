"""Middlebury flow layout (reference src/e2eflow/middlebury/data.py)."""
from ..core.data import Data

# sequences of other-data without ground truth; the reference deletes them after downloading, here
# they are left on disk and skipped by MiddleburyInput
NO_GROUND_TRUTH = ['Beanbags', 'DogDance', 'MiniCooper', 'Walking']


class MiddleburyData(Data):
    dirs = ['middlebury']
    layout = ('middlebury/{other-data,eval-data}/<seq>/frame*.png, middlebury/other-gt-flow/<seq>/flow10.flo '
              '(the unpacked other-gt-flow.zip, other-color-twoframes.zip, eval-color-twoframes.zip)')

    def _check(self):
        self._require('middlebury')

    def get_raw_dirs(self):
        raise NotImplementedError("Can not train on middlebury")
