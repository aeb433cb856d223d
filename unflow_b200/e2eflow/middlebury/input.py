"""Middlebury inputs (reference src/e2eflow/middlebury/input.py): per sequence frame k paired with
frame k + 1; ``input_train`` over ``other-data`` with the ``.flo`` ground truth of ``other-gt-flow``
(mask: both components < 1e9), ``input_test`` over ``eval-data``.  The sequences of ``other-data``
without ground truth (``data.NO_GROUND_TRUTH``) are skipped, which is what the reference's deleting
them amounts to."""
import os

from ..core.flow_io import read_flo
from ..core.input import Input, sequence_files
from .data import NO_GROUND_TRUTH


class MiddleburyInput(Input):
    def __init__(self, data, batch_size, dims, *, num_threads=1, normalize=True):
        super().__init__(data, batch_size, dims, num_threads=num_threads, normalize=normalize)

    def flow_files(self):
        return sequence_files(os.path.join(self.data.current_dir, 'middlebury', 'other-gt-flow'))

    def input_train(self):
        """One pass, batch 1: ``(im1, im2, input_shape, flow, mask)`` cropped / padded to ``dims``."""
        flows = self.flow_files()
        pairs = self.sequence_pairs('middlebury/other-data', exclude=NO_GROUND_TRUTH)
        assert len(pairs) == len(flows), "%d pairs, %d flow files" % (len(pairs), len(flows))
        for item, path in zip(self._input_sequence_test('middlebury/other-data', exclude=NO_GROUND_TRUTH), flows):
            flow, mask = read_flo(path)
            yield item + (self._preprocess_truth(flow), self._preprocess_truth(mask))

    def input_test(self):
        return self._input_sequence_test('middlebury/eval-data')
