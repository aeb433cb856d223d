"""KITTI inputs (reference src/e2eflow/kitti/input.py): image pairs with the occluded /
non-occluded ground-truth flow of the 2012 and 2015 training sets for evaluation, and the
ground-truth training batches of the supervised fine-tune (``input_train_gt``)."""
import os
import random

import torch

from ..core import augment
from ..core.flow_io import read_kitti_flow
from ..core.input import DecodeAhead, Input, read_png_image, resize_image_with_crop_or_pad

# (image directory, ground-truth directory) of the two training sets input_train_gt draws from
TRAIN_GT_SETS = [('data_scene_flow/training/image_2', 'data_scene_flow/training/flow_occ'),
                 ('data_stereo_flow/training/colored_0', 'data_stereo_flow/training/flow_occ')]


class KITTIInput(Input):
    def _flow_files(self, flow_dir, hold_out_inv):
        """kitti/input.py:35-70: sorted flow_occ / flow_noc files; ``hold_out_inv`` keeps the first k
        of a ``random.seed(0)`` shuffle of each list (the same permutation, the lists being equally
        long)."""
        out = []
        for sub in ('flow_occ', 'flow_noc'):
            d = os.path.join(self.data.current_dir, flow_dir, sub)
            files = os.listdir(d)
            files.sort()
            if hold_out_inv is not None:
                random.seed(0)
                random.shuffle(files)
                files = files[:hold_out_inv]
            out.append([os.path.join(d, f) for f in files])
        assert len(out[0]) == len(out[1])
        return out

    def _input_train(self, image_dir, flow_dir, hold_out_inv=None):
        """One pass, batch 1: ``(im1, im2, input_shape, flow_occ, mask_occ, flow_noc, mask_noc)``,
        everything cropped / padded to ``dims`` like the reference's queues deliver it."""
        height, width = self.dims
        occ, noc = self._flow_files(flow_dir, hold_out_inv)
        for (fn1, fn2), f_occ, f_noc in zip(self.image_pairs(image_dir, hold_out_inv), occ, noc):
            raw1, raw2 = read_png_image(fn1), read_png_image(fn2)
            item = [self._preprocess_image(raw1).unsqueeze(0), self._preprocess_image(raw2).unsqueeze(0),
                    torch.tensor(raw1.shape).unsqueeze(0)]
            for path in (f_occ, f_noc):
                flow, mask = read_kitti_flow(path)
                flow, mask = torch.as_tensor(flow).float(), torch.as_tensor(mask).float()
                if mask.dim() == 2:
                    mask = mask.unsqueeze(-1)
                item += [resize_image_with_crop_or_pad(flow, height, width).unsqueeze(0),
                         resize_image_with_crop_or_pad(mask, height, width).unsqueeze(0)]
            yield tuple(item)

    def input_train_2015(self, hold_out_inv=None):
        return self._input_train('data_scene_flow/training/image_2', 'data_scene_flow/training', hold_out_inv)

    def input_test_2015(self, hold_out_inv=None):
        return self._input_test('data_scene_flow/testing/image_2', hold_out_inv)

    def input_train_2012(self, hold_out_inv=None):
        return self._input_train('data_stereo_flow/training/colored_0', 'data_stereo_flow/training', hold_out_inv)

    def input_test_2012(self, hold_out_inv=None):
        return self._input_test('data_stereo_flow/testing/colored_0', hold_out_inv)

    # -- supervised fine-tuning ------------------------------------------------------------------
    def train_gt_files(self, hold_out):
        """kitti/input.py:82-119: the ordered ``(im1, im2, flow_occ)`` file triples ``input_train_gt``
        trains on.  Per set (2015 ``image_2``, 2012 ``colored_0``): sorted files, (2i, 2i+1) are a pair
        with the i-th ground-truth file, a ``random.seed(0)`` shuffle, the first ``hold_out`` dropped
        (the pairs ``input_train_2015(hold_out)`` / ``input_train_2012(hold_out)`` evaluate on); then
        both sets together shuffled again with ``random.seed(0)``."""
        filenames = []
        for img_dir, gt_dir in TRAIN_GT_SETS:
            img_dir = os.path.join(self.data.current_dir, img_dir)
            gt_dir = os.path.join(self.data.current_dir, gt_dir)
            img_files = sorted(os.listdir(img_dir))
            gt_files = sorted(os.listdir(gt_dir))
            assert len(img_files) % 2 == 0 and len(img_files) // 2 == len(gt_files)
            triples = [(os.path.join(img_dir, img_files[2 * i]), os.path.join(img_dir, img_files[2 * i + 1]),
                        os.path.join(gt_dir, gt_files[i])) for i in range(len(gt_files))]
            random.seed(0)
            random.shuffle(triples)
            filenames.extend(triples[hold_out:])
        random.seed(0)
        random.shuffle(filenames)
        return filenames

    def input_train_gt(self, hold_out, rank=0, world_size=1, crop_seed=0, pin=None):
        """Infinite iterator of ``(im1, im2, flow_gt, mask_gt)`` batches ``[B,H,W,3]``, ``[B,H,W,3]``,
        ``[B,H,W,2]``, ``[B,H,W,1]`` float32 (pinned host memory when CUDA is available), cycling
        through ``train_gt_files(hold_out)``.  One random crop window of ``dims`` is shared by both
        frames and the ground truth (kitti/input.py:126-131); the flow decodes as (v - 2**15) / 64 and
        the mask is the third channel.  With ``rank`` / ``world_size`` each rank takes every
        world_size-th batch, as ``input_raw`` does: batches rank, rank + world_size, ... of the stream
        (a resumed run passes a larger ``rank`` to skip the batches already trained on)."""
        triples = self.train_gt_files(hold_out)
        if not triples:
            raise ValueError("input_train_gt: no training pairs left after holding out %d per set" % hold_out)
        height, width = self.dims
        B = self.batch_size
        pin = torch.cuda.is_available() if pin is None else pin

        def read_gt(path):
            flow, mask = read_kitti_flow(path)
            return torch.cat([torch.as_tensor(flow), torch.as_tensor(mask)], 2).float()

        def plan(batch_index):
            gen = torch.Generator().manual_seed(crop_seed * 1000003 + batch_index)
            seeds = [int(torch.randint(0, 2 ** 31 - 1, (1,), generator=gen)) for _ in range(B)]
            out = [torch.empty((B, height, width, c), dtype=torch.float32, pin_memory=pin) for c in (3, 3, 2, 1)]

            def item(k):
                fn1, fn2, fn_gt = triples[(batch_index * B + k) % len(triples)]

                def finish(im1, im2, gt):
                    im1, im2, gt = augment.random_crop([im1, im2, gt], [height, width, 3], seed=seeds[k])
                    if self.normalize:
                        im1, im2 = self._normalize_image(im1), self._normalize_image(im2)
                    for dst, src in zip(out, (im1, im2, gt[:, :, 0:2], gt[:, :, 2:3])):
                        dst[k].copy_(src)
                return (lambda: read_png_image(fn1), lambda: read_png_image(fn2), lambda: read_gt(fn_gt)), finish

            return tuple(out), [item(k) for k in range(B)]

        return DecodeAhead(plan, rank, world_size, self.num_threads)
