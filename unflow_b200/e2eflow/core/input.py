"""Host-side input pipeline with the reference's file-pairing rules (src/e2eflow/core/input.py).

The reference builds TF queue runners (``string_input_producer`` -> ``WholeFileReader`` ->
``decode_png`` -> ``tf.train.batch``); the pairing / ordering logic in front of the queues is plain
Python and is what decides WHICH frames are trained on.  That logic is kept verbatim in behaviour:

* ``input_raw`` (:121-196): per directory the sorted frame list, consecutive frames paired
  (``sequence``) for every ``skip`` distance, pairs whose frame numbers are not consecutive dropped
  when ``skipped_frames``; ``random.seed(seed)`` shuffle; optional swapped duplicates; the resume
  ``shift`` applied with ``np.roll`` on the pair array WITHOUT an axis (i.e. on the flattened list
  of file names, as the reference does -- an odd shift re-pairs neighbouring entries);
  one random crop offset shared by both frames of a pair (``random_crop``), batches of
  ``batch_size`` consecutive pairs, cycling forever.
* ``_input_images`` (:78-107): sorted files, (2i, 2i+1) are a pair; ``hold_out_inv`` keeps the first
  k pairs of a ``random.seed(0)`` shuffle.

Instead of TF queues a batch iterator with a small prefetch thread decodes PNGs (OpenCV) into
pinned host tensors ``[B,H,W,3]`` float32 in [0,255], RGB like ``tf.image.decode_png``; with
``num_threads`` > 1 the pairs of a batch are decoded on a pool of that many threads, into the same
slots with the same crop seeds (bit-identical batches).
* ``sequence_pairs`` / ``sequence_files`` (sintel/input.py, middlebury/input.py): per sorted
  sequence directory frame k paired with frame k + 1, and the sorted per-sequence ground-truth lists.
With ``rank`` / ``world_size`` each rank takes every world_size-th batch: distinct shards per GPU
(the reference's towers all dequeue the same batch, SURVEY.md R4).
"""
import os
import queue
import random
import threading

import numpy as np
import torch

from . import augment


def frame_name_to_num(name):
    stripped = name.split('.')[0].lstrip('0')
    if stripped == '':
        return 0
    return int(stripped)


def read_png_image(path):
    """RGB float32 [h,w,3] in [0,255] (tf.image.decode_png(channels=3) + cast)."""
    import cv2
    im = cv2.imread(path, cv2.IMREAD_COLOR)
    if im is None:
        raise IOError("cannot read image " + path)
    return torch.from_numpy(np.ascontiguousarray(im[:, :, ::-1])).float()


def resize_image_with_crop_or_pad(t, height, width):
    """tf.image.resize_image_with_crop_or_pad for [h,w,c] or [b,h,w,c]: centre crop / zero pad."""
    hd, wd = t.dim() - 3, t.dim() - 2
    h, w = t.shape[hd], t.shape[wd]
    if h > height:
        t = t.narrow(hd, (h - height) // 2, height)
    if w > width:
        t = t.narrow(wd, (w - width) // 2, width)
    h, w = t.shape[hd], t.shape[wd]
    if h < height or w < width:
        top, left = (height - h) // 2, (width - w) // 2
        pad = [0, 0, left, width - w - left, top, height - h - top]
        t = torch.nn.functional.pad(t, pad)
    return t


def resize_input(t, height, width, resized_h, resized_w):
    """core/input.py:10-14: undo the crop-or-pad to (resized_h, resized_w), then bilinear."""
    from . import tf_image
    t = t.reshape(resized_h, resized_w, 3)
    t = resize_image_with_crop_or_pad(t, height, width).unsqueeze(0)
    return tf_image.resize_bilinear(t, [resized_h, resized_w])


def resize_output_crop(t, height, width, channels):
    """core/input.py:17-21: centre crop / zero pad a [1,h,w,c] result back to the file size."""
    return resize_image_with_crop_or_pad(t[0], height, width).reshape(1, height, width, channels)


def resize_output(t, height, width, channels):
    """core/input.py:24-25."""
    from . import tf_image
    return tf_image.resize_bilinear(t, [height, width])


def resize_output_flow(t, height, width, channels=2):
    """core/input.py:28-34 (implemented in core/flow_io.py)."""
    from .flow_io import resize_output_flow as impl
    return impl(t, height, width, channels)


class _Prefetcher:
    """Iterator over ``make(i)`` for i = first, first+step, ... produced by a daemon thread."""

    def __init__(self, make, first, step, depth=4, pool=None):
        self._q = queue.Queue(maxsize=depth)
        self._stop = threading.Event()
        self._pool = pool

        def work():
            i = first
            while not self._stop.is_set():
                try:
                    item = make(i)
                except BaseException as e:   # surfaced in the consumer
                    item = e
                while not self._stop.is_set():
                    try:
                        self._q.put(item, timeout=0.1)
                        break
                    except queue.Full:
                        continue
                if isinstance(item, BaseException):
                    return
                i += step

        self._t = threading.Thread(target=work, daemon=True)
        self._t.start()

    def __iter__(self):
        return self

    def __next__(self):
        item = self._q.get()
        if isinstance(item, StopIteration):
            raise StopIteration
        if isinstance(item, BaseException):
            raise item
        return item

    def close(self):
        self._stop.set()
        if self._pool is not None:
            self._pool.shutdown(wait=False)


class Input():
    mean = [104.920005, 110.1753, 114.785955]
    stddev = 1 / 0.0039216

    def __init__(self, data, batch_size, dims, *,
                 num_threads=1, normalize=True,
                 skipped_frames=False):
        assert len(dims) == 2
        self.data = data
        self.dims = dims
        self.batch_size = batch_size
        self.num_threads = num_threads
        self.normalize = normalize
        self.skipped_frames = skipped_frames

    def get_normalization(self):
        return self.mean, self.stddev

    def _normalize_image(self, image):
        return (image - torch.tensor(self.mean)) / self.stddev

    def _preprocess_image(self, image):
        height, width = self.dims
        image = resize_image_with_crop_or_pad(image, height, width)
        if self.normalize:
            image = self._normalize_image(image)
        return image

    def _decode_pool(self):
        """A pool of ``num_threads`` decode threads ([run] num_input_threads; OpenCV releases the GIL),
        None for one thread."""
        if self.num_threads <= 1:
            return None
        from concurrent.futures import ThreadPoolExecutor
        return ThreadPoolExecutor(self.num_threads, thread_name_prefix='decode')

    @staticmethod
    def _fill(pool, load, n):
        """``load(k)`` for k < n: in order on the calling thread, or spread over ``pool``.  Each
        ``load`` writes only its own slot k of the batch, so both give the same batch."""
        if pool is None:
            for k in range(n):
                load(k)
        else:
            list(pool.map(load, range(n)))

    # -- which files ---------------------------------------------------------------------------
    def raw_pairs(self, swap_images=True, sequence=True, shift=0, seed=0, skip=0):
        """The ordered list of (frame 1, frame 2) file names ``input_raw`` trains on."""
        if not isinstance(skip, list):
            skip = [skip]
        filenames = []
        for dir_path in self.data.get_raw_dirs():
            files = os.listdir(dir_path)
            files.sort()
            if sequence:
                steps = [1 + s for s in skip]
                stops = [len(files) - s for s in steps]
            else:
                steps = [2]
                stops = [len(files)]
                assert len(files) % 2 == 0
            for step, stop in zip(steps, stops):
                for i in range(0, stop, step):
                    if self.skipped_frames and sequence:
                        assert step == 1
                        if frame_name_to_num(files[i]) + 1 != frame_name_to_num(files[i + 1]):
                            continue
                    filenames.append((os.path.join(dir_path, files[i]),
                                      os.path.join(dir_path, files[i + 1])))
        random.seed(seed)
        random.shuffle(filenames)
        print("Training on {} frame pairs.".format(len(filenames)))
        extended = []
        for fn1, fn2 in filenames:
            extended.append((fn1, fn2))
            if swap_images:
                extended.append((fn2, fn1))
        shift = shift % len(extended)
        rolled = np.roll(np.array(extended, dtype=object), shift)     # no axis: flattened, like the reference
        return [(str(a), str(b)) for a, b in rolled]

    def image_pairs(self, image_dir, hold_out_inv=None):
        """Sorted files of ``image_dir``; (2i, 2i+1) belong together (core/input.py:78-107)."""
        image_dir = os.path.join(self.data.current_dir, image_dir)
        image_files = os.listdir(image_dir)
        image_files.sort()
        assert len(image_files) % 2 == 0, 'expected pairs of images'
        pairs = [(os.path.join(image_dir, image_files[2 * i]), os.path.join(image_dir, image_files[2 * i + 1]))
                 for i in range(len(image_files) // 2)]
        if hold_out_inv is not None:
            random.seed(0)
            random.shuffle(pairs)
            pairs = pairs[:hold_out_inv]
        return pairs

    def sequence_pairs(self, image_dir, exclude=()):
        """Per sorted sub-directory of ``image_dir`` (one sequence each), frame k paired with frame
        k + 1 (sintel/input.py:63-84, middlebury/input.py:66-87); sub-directories named in
        ``exclude`` are skipped."""
        image_dir = os.path.join(self.data.current_dir, image_dir)
        pairs = []
        for sub_name in sorted(os.listdir(image_dir)):
            if sub_name in exclude:
                continue
            sub_dir = os.path.join(image_dir, sub_name)
            files = sorted(os.listdir(sub_dir))
            pairs += [(os.path.join(sub_dir, files[i]), os.path.join(sub_dir, files[i + 1]))
                      for i in range(len(files) - 1)]
        return pairs

    def _input_sequence_test(self, image_dir, exclude=()):
        """``_input_test`` over ``sequence_pairs``: ``(im1, im2, input_shape)``, batch 1."""
        for fn1, fn2 in self.sequence_pairs(image_dir, exclude):
            raw1, raw2 = read_png_image(fn1), read_png_image(fn2)
            yield (self._preprocess_image(raw1).unsqueeze(0), self._preprocess_image(raw2).unsqueeze(0),
                   torch.tensor(raw1.shape).unsqueeze(0))

    def _preprocess_truth(self, t):
        """A ground-truth map [h,w,c] -> [1,H,W,c] cropped / padded to ``dims`` (``_preprocess_flow``)."""
        height, width = self.dims
        t = torch.as_tensor(t).float()
        if t.dim() == 2:
            t = t.unsqueeze(-1)
        return resize_image_with_crop_or_pad(t, height, width).unsqueeze(0)

    # -- batches -------------------------------------------------------------------------------
    def input_raw(self, swap_images=True, sequence=True,
                  needs_crop=True, shift=0, seed=0,
                  center_crop=False, skip=0, rank=0, world_size=1, crop_seed=0, pin=None):
        """Infinite iterator of ``(image_1, image_2)`` batches ``[B,H,W,3]`` (pinned host memory when
        CUDA is available)."""
        pairs = self.raw_pairs(swap_images, sequence, shift, seed, skip)
        height, width = self.dims
        B = self.batch_size
        pin = torch.cuda.is_available() if pin is None else pin

        pool = self._decode_pool()

        def make(batch_index):
            gen = torch.Generator().manual_seed(crop_seed * 1000003 + batch_index)
            # the crop seeds of the whole batch are drawn first, in order, so they do not depend on
            # which thread decodes which pair
            seeds = [int(torch.randint(0, 2 ** 31 - 1, (1,), generator=gen)) for _ in range(B)] if needs_crop else None
            a = torch.empty((B, height, width, 3), dtype=torch.float32, pin_memory=pin)
            b = torch.empty((B, height, width, 3), dtype=torch.float32, pin_memory=pin)

            def load(k):
                fn1, fn2 = pairs[(batch_index * B + k) % len(pairs)]
                im1, im2 = read_png_image(fn1), read_png_image(fn2)
                if needs_crop:
                    im1, im2 = augment.random_crop([im1, im2], [height, width, 3], seed=seeds[k])
                else:
                    im1, im2 = im1.reshape(height, width, 3), im2.reshape(height, width, 3)
                if self.normalize:
                    im1, im2 = self._normalize_image(im1), self._normalize_image(im2)
                a[k].copy_(im1)
                b[k].copy_(im2)

            self._fill(pool, load, B)
            return a, b

        return _Prefetcher(make, rank, world_size, pool=pool)

    def _input_test(self, image_dir, hold_out_inv=None):
        """One pass over the pairs of ``image_dir``: ``(im1, im2, input_shape)`` with batch 1
        (``allow_smaller_final_batch`` makes larger batches ragged; evaluation uses 1)."""
        for fn1, fn2 in self.image_pairs(image_dir, hold_out_inv):
            raw1, raw2 = read_png_image(fn1), read_png_image(fn2)
            yield (self._preprocess_image(raw1).unsqueeze(0), self._preprocess_image(raw2).unsqueeze(0),
                   torch.tensor(raw1.shape).unsqueeze(0))


def sequence_files(parent_dir, ignore_last=False):
    """sintel/input.py:38-49 ``_get_filenames``: the sorted files of every sorted sub-directory,
    each sub-directory's last file dropped with ``ignore_last``."""
    filenames = []
    for sub_name in sorted(os.listdir(parent_dir)):
        sub_dir = os.path.join(parent_dir, sub_name)
        files = sorted(os.listdir(sub_dir))
        if ignore_last:
            files = files[:-1]
        filenames += [os.path.join(sub_dir, f) for f in files]
    return filenames
