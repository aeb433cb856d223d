"""MPI Sintel inputs (reference src/e2eflow/sintel/input.py): per sequence frame k paired with
frame k + 1 of ``{training,test}/{clean,final}``; the training variants add the ground truth of
``training/{flow,invalid,occlusions}`` (sorted per sequence; the last ``invalid`` file of every
sequence dropped, it belongs to the last frame, which starts no pair):

    flow_occ = flow, mask_occ = 1 - invalid, flow_noc = flow * (1 - occ), mask_noc = mask_occ * (1 - occ)

Deliberate deviation: ``invalid`` / ``occlusions`` PNGs are binarised (value > 0).  The reference
casts the decoded byte to float unscaled (``_read_binary``), which for masks stored as 0/255 makes
``1 - occ`` no mask at all; for 0/1 files both give the same numbers."""
import os

import numpy as np
import torch

from ..core.flow_io import read_flo
from ..core.input import Input, sequence_files

GT_DIRS = ('flow', 'invalid', 'occlusions')


def read_binary(path):
    """A mask PNG -> float32 [h,w,1], 1 where the (grey) value is > 0."""
    import cv2
    im = cv2.imread(path, cv2.IMREAD_GRAYSCALE)
    if im is None:
        raise IOError("cannot read image " + path)
    return torch.from_numpy((im > 0).astype(np.float32)[:, :, None])


class SintelInput(Input):
    def __init__(self, data, batch_size, dims, *, num_threads=1, normalize=True):
        super().__init__(data, batch_size, dims, num_threads=num_threads, normalize=normalize)

    def truth_files(self):
        """(flow, invalid, occlusion) file lists, one entry per training pair (sintel/input.py:86-94)."""
        top = os.path.join(self.data.current_dir, 'sintel', 'training')
        lists = [sequence_files(os.path.join(top, d), ignore_last=(d == 'invalid')) for d in GT_DIRS]
        assert len(lists[0]) == len(lists[1]) == len(lists[2]), [len(x) for x in lists]
        return lists

    def _input_train(self, image_dir):
        """One pass, batch 1: ``(im1, im2, input_shape, flow_occ, mask_occ, flow_noc, mask_noc)``
        cropped / padded to ``dims``."""
        flows, invalids, occs = self.truth_files()
        for item, f_flow, f_inv, f_occ in zip(self._input_sequence_test(image_dir), flows, invalids, occs):
            flow = torch.from_numpy(read_flo(f_flow)[0])
            occ = read_binary(f_occ)
            mask_occ = 1 - read_binary(f_inv)
            yield item + tuple(self._preprocess_truth(t) for t in
                               (flow, mask_occ, flow * (1 - occ), mask_occ * (1 - occ)))

    def input_train_clean(self):
        return self._input_train('sintel/training/clean')

    def input_train_final(self):
        return self._input_train('sintel/training/final')

    def input_test_clean(self):
        return self._input_sequence_test('sintel/test/clean')

    def input_test_final(self):
        return self._input_sequence_test('sintel/test/final')
