"""The decode-ahead input pipeline (``core.input.DecodeAhead``) without a GPU: ``input_raw`` and
``input_train_gt`` batches bit-identical to one decode thread for any thread count (wraparound, rank
shards), more than a batch's decodes in flight across batch boundaries, memory bounded to a fixed number
of batches ahead, decode errors surfaced in the consumer, and a prompt ``close()``."""
import threading
import time

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from unflow_b200.e2eflow.core import input as core_input
from unflow_b200.e2eflow.core.flow_io import write_kitti_flow
from unflow_b200.e2eflow.kitti import input as kitti_input
from unflow_b200.e2eflow.kitti.input import KITTIInput
from unflow_b200.e2eflow.synthia.data import SynthiaData

B = 3


class _Data:
    def __init__(self, root):
        self.current_dir = str(root)


def _synthia_tree(root, frames=5, h=40, w=60):
    """Two sequences, three views, ``frames`` frames each: 3 * (frames - 1) pairs."""
    rng = np.random.default_rng(4)
    for seq, views in (('SYNTHIA-SEQS-01-SUMMER', ('Omni_F', 'Omni_B')), ('SYNTHIA-SEQS-02-WINTER', ('Omni_L',))):
        for view in views:
            d = root / 'synthia' / seq / seq / 'RGB' / 'Stereo_Left' / view
            d.mkdir(parents=True)
            for i in range(frames):
                cv2.imwrite(str(d / ('%06d.png' % i)), rng.integers(0, 255, (h, w, 3), dtype=np.uint8))


def _kitti_gt_tree(root, n=4, h=20, w=30):
    """Both KITTI training sets with n pairs each and their flow_occ ground truth."""
    rng = np.random.default_rng(1)
    for top, img in (('data_scene_flow', 'image_2'), ('data_stereo_flow', 'colored_0')):
        tr = root / top / 'training'
        for sub in (img, 'flow_occ'):
            (tr / sub).mkdir(parents=True)
        for i in range(n):
            for j in (10, 11):
                cv2.imwrite(str(tr / img / ('%06d_%d.png' % (i, j))), rng.integers(0, 255, (h, w, 3), dtype=np.uint8))
            flow = rng.integers(-3000, 3000, (h, w, 2)).astype(np.float32) / 64.0
            valid = (rng.random((h, w)) < 0.5).astype(np.float32)
            write_kitti_flow(str(tr / 'flow_occ' / ('%06d_10.png' % i)), flow, valid)


def _take(stream, n):
    try:
        return [tuple(t.clone() for t in next(stream)) for _ in range(n)]
    finally:
        stream.close()


def _same(a, b):
    return len(a) == len(b) and all(all(torch.equal(x, y) for x, y in zip(p, q)) for p, q in zip(a, b))


@pytest.mark.parametrize("rank,world", [(0, 1), (1, 2)])
def test_input_raw_bit_identical_for_any_thread_count(tmp_path, rank, world):
    _synthia_tree(tmp_path)
    data = SynthiaData(str(tmp_path))

    def batches(threads):
        inp = KITTIInput(data, B, (24, 32), normalize=False, num_threads=threads)
        # 12 pairs, shift 5: six batches of 3 wrap around the list twice (rank shard: every other batch)
        return _take(inp.input_raw(swap_images=False, shift=5, rank=rank, world_size=world, crop_seed=3, pin=False), 6)

    want = batches(1)
    assert not all(torch.equal(want[0][0], w[0]) for w in want[1:])
    for threads in (2, B, 16):
        assert _same(batches(threads), want), threads
    # the shard is the rank's batches of the one-rank stream
    if world == 2:
        full = KITTIInput(data, B, (24, 32), normalize=False, num_threads=1).input_raw(
            swap_images=False, shift=5, crop_seed=3, pin=False)
        assert _same(_take(full, 12)[1::2], want)


@pytest.mark.parametrize("rank,world", [(0, 1), (1, 2)])
def test_input_train_gt_bit_identical_for_any_thread_count(tmp_path, rank, world):
    _kitti_gt_tree(tmp_path)

    def batches(threads):
        inp = KITTIInput(_Data(tmp_path), B, (12, 16), normalize=True, num_threads=threads)
        # 2 x (4 - 1) = 6 triples: five batches of 3 wrap around
        return _take(inp.input_train_gt(1, rank=rank, world_size=world, pin=False), 5)

    want = batches(1)
    assert [tuple(t.shape) for t in want[0]] == [(B, 12, 16, 3), (B, 12, 16, 3), (B, 12, 16, 2), (B, 12, 16, 1)]
    for threads in (2, B, 16):
        assert _same(batches(threads), want), threads


class _SlowReader:
    """A stand-in for read_png_image that takes ``delay`` seconds and records how many reads overlap,
    which threads ran them and how many have started."""

    def __init__(self, real, delay, fail=None):
        self.real, self.delay, self.fail = real, delay, fail
        self.lock = threading.Lock()
        self.active = self.peak = self.started = 0
        self.threads = set()

    def __call__(self, path):
        with self.lock:
            self.active += 1
            self.started += 1
            self.peak = max(self.peak, self.active)
            self.threads.add(threading.current_thread())
        try:
            time.sleep(self.delay)
            if self.fail is not None and self.fail in path:
                raise IOError("cannot read image " + path)
            return self.real(path)
        finally:
            with self.lock:
                self.active -= 1


def _slow_stream(tmp_path, monkeypatch, threads, delay, fail=None, batch=2):
    _synthia_tree(tmp_path)
    reader = _SlowReader(core_input.read_png_image, delay, fail)
    monkeypatch.setattr(core_input, 'read_png_image', reader)
    inp = KITTIInput(SynthiaData(str(tmp_path)), batch, (24, 32), normalize=False, num_threads=threads)
    return inp.input_raw(swap_images=False, pin=False), reader


def test_more_than_a_batch_of_decodes_in_flight(tmp_path, monkeypatch):
    stream, reader = _slow_stream(tmp_path, monkeypatch, threads=8, delay=0.2, batch=2)
    try:
        for _ in range(6):
            next(stream)
    finally:
        stream.close()
    # a batch of 2 pairs is 4 frame decodes; 8 threads keep reads of the following batches going
    assert reader.peak > 2 * 2, reader.peak
    assert reader.peak <= 8


def test_train_gt_decodes_every_file_as_its_own_task(tmp_path, monkeypatch):
    _kitti_gt_tree(tmp_path)
    reader = _SlowReader(core_input.read_png_image, 0.2)
    monkeypatch.setattr(kitti_input, 'read_png_image', reader)
    stream = KITTIInput(_Data(tmp_path), 1, (12, 16), normalize=False, num_threads=6).input_train_gt(1, pin=False)
    try:
        for _ in range(3):
            next(stream)
    finally:
        stream.close()
    assert reader.peak > 2, reader.peak       # both frames of a pair and frames of later pairs together


def test_memory_is_bounded_to_a_fixed_number_of_batches_ahead(tmp_path, monkeypatch):
    stream, reader = _slow_stream(tmp_path, monkeypatch, threads=4, delay=0.0, batch=2)
    try:
        assert stream.depth == 4
        next(stream)
        time.sleep(0.5)                 # the pool catches up and then has nothing more to do
        assert reader.started == (1 + stream.depth) * 2 * 2, reader.started
        # many threads per batch: enough batches ahead to keep them all busy, no more
        wide = core_input.DecodeAhead(lambda i: (None, [((lambda: 0,) * 2, lambda a, b: None)] * 2), 0, 1, 40)
        assert wide.depth == 10
        wide.close()
    finally:
        stream.close()


def _numbered_plan(fail_at=None):
    """Batch i is ``[i]``, written by its one item; planning batch ``fail_at`` raises once."""
    failed = []

    def plan(i):
        if i == fail_at and not failed:
            failed.append(i)
            raise MemoryError("cannot allocate batch %d" % i)
        out = [None]

        def finish(v):
            out[0] = v
        return out, [((lambda: i,), finish)]
    return plan


def test_a_failing_plan_loses_no_batch(tmp_path):
    # depth 4: batches 0..4 are planned at construction; taking batch 1 needs batch 5 planned first
    stream = core_input.DecodeAhead(_numbered_plan(fail_at=5), 0, 1, 2)
    try:
        assert next(stream) == [0]
        with pytest.raises(MemoryError):
            next(stream)
        # batch 1 was not taken: the next call plans batch 5 again and returns batch 1, then the rest in order
        assert [next(stream)[0] for _ in range(8)] == list(range(1, 9))
    finally:
        stream.close()


def test_a_failing_constructor_leaves_no_thread():
    before = set(threading.enumerate())
    with pytest.raises(MemoryError):
        core_input.DecodeAhead(_numbered_plan(fail_at=2), 0, 1, 4)
    assert not [t for t in set(threading.enumerate()) - before if t.is_alive()]


def test_close_is_prompt_and_leaves_no_busy_worker(tmp_path, monkeypatch):
    stream, reader = _slow_stream(tmp_path, monkeypatch, threads=8, delay=0.3, batch=2)
    next(stream)
    time.sleep(0.1)                     # reads of the next batches are running
    assert reader.active > 0
    t0 = time.perf_counter()
    stream.close()
    elapsed = time.perf_counter() - t0
    assert elapsed < 2.0, elapsed       # the running reads finish (one delay), the queued ones are cancelled
    assert reader.active == 0
    assert not any(t.is_alive() for t in reader.threads)
    started = reader.started
    time.sleep(0.5)
    assert reader.started == started


def test_a_decode_error_reaches_the_consumer(tmp_path, monkeypatch):
    # 12 pairs in listing order (seed 0 shuffle); fail every read of one file that the stream reaches
    stream, reader = _slow_stream(tmp_path, monkeypatch, threads=4, delay=0.0, fail='Omni_L', batch=2)
    with pytest.raises(IOError, match='Omni_L'):
        for _ in range(12):
            next(stream)
    with pytest.raises(IOError):
        next(stream)                    # the stream stays failed
    stream.close()
    assert not any(t.is_alive() for t in reader.threads)
