"""FlyingChairs inputs (reference src/e2eflow/chairs/input.py): unrelated training pairs
(sorted files of ``flying_chairs/image``, (2i, 2i+1) a pair, no crop: frames are 384x512) and the
validation pairs of ``flying_chairs/test_image`` with the i-th sorted ``.flo`` of
``flying_chairs/flow`` (mask: both components < 1e9)."""
import os

from ..core.flow_io import read_flo
from ..core.input import Input


class ChairsInput(Input):
    def __init__(self, data, batch_size, dims, *, num_threads=1, normalize=True):
        super().__init__(data, batch_size, dims, num_threads=num_threads, normalize=normalize)

    def flow_files(self):
        flow_dir = os.path.join(self.data.current_dir, 'flying_chairs', 'flow')
        return [os.path.join(flow_dir, fn) for fn in sorted(os.listdir(flow_dir))]

    def input_test(self):
        """One pass, batch 1: ``(im1, im2, input_shape, flow, mask)`` cropped / padded to ``dims``."""
        flows = self.flow_files()
        for item, path in zip(self._input_test('flying_chairs/test_image'), flows):
            flow, mask = read_flo(path)
            yield item + (self._preprocess_truth(flow), self._preprocess_truth(mask))

    def input_raw(self, swap_images=True, shift=0, **kw):
        """chairs/input.py:39-43; ``kw`` takes the rank / world_size / crop_seed / pin of
        ``Input.input_raw``."""
        return super().input_raw(sequence=False, swap_images=swap_images, needs_crop=False, shift=shift, **kw)
