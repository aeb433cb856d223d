#!/usr/bin/env python
"""The training loop as users run it: ``unflow_b200.run.main`` on a generated PNG tree of each dataset,
augmentation on, in both conv arithmetic modes, with and without ``--graph``.

    python tools/bench_train_loop.py [--steps 100] [--warmup 20] [--batches 16] [--threads N]
                                     [--datasets chairs,synthia,cityscapes,kitti] [--modes fp32,3xtf32]
                                     [--graph both|on|off]

Prints the card's name, power limit and SM clock limit, then one JSON line per dataset:
  loop   per (conv_precision, graph): ms per training iteration and pairs/s, from a host clock read after a
         device synchronise at the end of iteration ``--warmup`` and at the end of iteration
         ``--warmup + --steps``.  Between the two it is run.py's own loop: the next batch from the input
         pipeline ([run] num_input_threads = ``--threads``, default os.cpu_count()), the host-to-device
         copy, the step (captured once and replayed with ``--graph``).  The mode is set the way users set
         it, with ``[run] conv_precision``.  ``input_wait_ms_per_step`` is the part of it the loop spent
         waiting for its next batch (0: the input keeps up).  The pipeline decodes a few batches ahead
         while the first steps run (and the graph is captured), so an input-bound loop starts with that
         lead; the ``--warmup`` iterations are there to use it up, and the timed window is steady state;
  input  the same input pipeline alone (``run.dataset_inputs``: PNG decode, crop, pinned batch), in pairs/s
         at 1, B and os.cpu_count() decode threads, over ``--batches`` batches taken after the pipeline's
         lead (its ``depth`` batches decoded ahead, and the first) has been used up.
Geometries, batch 4 and loss parameters are those of tools/bench_datasets.py (FlowNetC, one GPU).  The
frames are smooth synthetic images, which compress better than photographs, so they decode somewhat
faster than a real dataset's.  Everything it writes goes to a temporary directory.
"""
import argparse
import contextlib
import io
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from bench_datasets import BATCH, DATASETS, card  # noqa: E402
from unflow_b200 import synthetic as synth  # noqa: E402

N_FRAMES = 16


def _write_frames(d, frame_hw, names, seed):
    import cv2
    os.makedirs(d, exist_ok=True)
    for i in range(0, len(names), 2):
        a, b, _ = synth.image_pair(1, frame_hw[0], frame_hw[1], seed=seed + i)
        for name, im in zip(names[i:i + 2], (a, b)):
            if not cv2.imwrite(os.path.join(d, name), im[0].clamp(0, 255).byte().numpy()[:, :, ::-1].copy()):
                raise IOError("cannot write " + os.path.join(d, name))


def make_tree(data, dataset, frame_hw):
    """``N_FRAMES`` frames at ``frame_hw`` in the layout ``run.dataset_inputs`` reads for ``dataset``."""
    j = os.path.join
    if dataset == 'chairs':
        _write_frames(j(data, 'flying_chairs', 'image'), frame_hw,
                      ['%05d_img%d.png' % (i // 2, i % 2 + 1) for i in range(N_FRAMES)], 0)
        for d in ('test_image', 'flow'):
            os.makedirs(j(data, 'flying_chairs', d))
    elif dataset == 'synthia':
        seq = 'SYNTHIA-SEQS-01-SUMMER'
        _write_frames(j(data, 'synthia', seq, seq, 'RGB', 'Stereo_Left', 'Omni_F'), frame_hw,
                      ['%06d.png' % i for i in range(N_FRAMES)], 0)
    elif dataset == 'cityscapes':
        _write_frames(j(data, 'cs', 'leftImg8bit_sequence_trainvaltest', 'train', 'aachen'), frame_hw,
                      ['aachen_000000_%06d_leftImg8bit.png' % (17 + i) for i in range(N_FRAMES)], 0)
    elif dataset == 'kitti':
        drive = j(data, 'kitti_raw', '2011_09_26', '2011_09_26_drive_0001_extract')
        for cam in ('image_02', 'image_03'):
            _write_frames(j(drive, cam, 'data'), frame_hw, ['%010d.png' % i for i in range(N_FRAMES)], 0)
    else:
        raise SystemExit("unknown dataset " + dataset)


def write_config(path, root, dataset, net_hw, params, precision, threads):
    lines = ["[dirs]", "log = %s/log" % root, "checkpoints = %s/log/checkpoints" % root, "data = %s/data" % root,
             "[run]", "batch_size = %d" % BATCH, "gpu_list = 0", "num_input_threads = %d" % threads,
             "dataset = %s" % dataset, "development = True", "conv_precision = %s" % precision,
             "[train]", "decay_interval = 100000", "save_interval = 100000", "display_interval = 100000",
             "[train_%s]" % dataset, "height = %d" % net_hw[0], "width = %d" % net_hw[1],
             "num_iters = 100000", "decay_after = 100000"]
    lines += ["%s = %s" % (k, v) for k, v in params.items()]
    with open(path, 'w') as f:
        f.write("\n".join(lines) + "\n")


@contextlib.contextmanager
def step_clock(warmup, steps):
    """Patches Trainer.step: a device synchronise and a host clock reading after iteration ``warmup`` and
    after iteration ``warmup + steps``."""
    from unflow_b200.e2eflow.core.train import Trainer
    orig = Trainer.step
    marks = []
    count = [0]

    def step(self, *args, **kwargs):
        out = orig(self, *args, **kwargs)
        count[0] += 1
        if count[0] in (warmup, warmup + steps):
            torch.cuda.synchronize()
            marks.append(time.perf_counter())
        return out

    Trainer.step = step
    try:
        yield marks
    finally:
        Trainer.step = orig


class _TimedStream:
    """A batch stream whose ``next`` calls are timed: ``waits`` gets the seconds of each."""

    def __init__(self, stream, waits):
        self.stream, self.waits = stream, waits

    def __iter__(self):
        return self

    def __next__(self):
        t0 = time.perf_counter()
        item = next(self.stream)
        self.waits.append(time.perf_counter() - t0)
        return item

    def close(self):
        self.stream.close()


@contextlib.contextmanager
def input_clock():
    """Patches run.dataset_inputs so that the training loop's batch stream is a ``_TimedStream``."""
    from unflow_b200 import run as R
    orig = R.dataset_inputs
    waits = []

    def dataset_inputs(*args, **kwargs):
        batches, eval_input = orig(*args, **kwargs)
        return _TimedStream(batches, waits), eval_input

    R.dataset_inputs = dataset_inputs
    try:
        yield waits
    finally:
        R.dataset_inputs = orig


def time_loop(root, dataset, net_hw, params, precision, graph, threads, steps, warmup):
    from unflow_b200 import run as R
    ini = os.path.join(root, 'config_%s_%s_%d.ini' % (dataset, precision, graph))
    write_config(ini, root, dataset, net_hw, params, precision, threads)
    argv = ["--ex", "bench_%s" % dataset, "--config", ini, "--debug", "--ow", "--max-iters", str(warmup + steps)]
    log = io.StringIO()
    with step_clock(warmup, steps) as marks, input_clock() as waits, contextlib.redirect_stdout(log):
        R.main(argv + (["--graph"] if graph else []))
    if "-- rank 0: conv precision %s" % precision not in log.getvalue():
        raise SystemExit("run did not train in %s:\n%s" % (precision, log.getvalue()))
    ms = (marks[1] - marks[0]) * 1e3 / steps
    # iteration i takes its batch before its step: the timed iterations warmup + 1 .. warmup + steps
    wait = sum(waits[warmup:warmup + steps]) * 1e3 / steps
    return {"ms_per_step": round(ms, 2), "pairs_per_s": round(BATCH / (ms * 1e-3), 2),
            "input_wait_ms_per_step": round(wait, 2)}


def time_input(root, dataset, net_hw, threads, batches):
    from unflow_b200 import run as R
    run_config = {'batch_size': BATCH, 'num_input_threads': threads, 'development': True}
    with contextlib.redirect_stdout(io.StringIO()):
        stream, _ = R.dataset_inputs({'data': os.path.join(root, 'data')}, run_config,
                                     {'height': net_hw[0], 'width': net_hw[1]}, dataset, BATCH, 1, 0, 1)
    try:
        for _ in range(stream.depth + 1):
            next(stream)
        t0 = time.perf_counter()
        for _ in range(batches):
            next(stream)
        dt = time.perf_counter() - t0
    finally:
        stream.close()
    return round(batches * BATCH / dt, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batches", type=int, default=16, help="timed input batches per thread count")
    ap.add_argument("--threads", type=int, default=os.cpu_count() or 1,
                    help="[run] num_input_threads of the timed loops")
    ap.add_argument("--datasets", default=",".join(DATASETS))
    ap.add_argument("--modes", default="fp32,3xtf32")
    ap.add_argument("--graph", choices=("both", "on", "off"), default="both")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_loop needs a CUDA device")
    graphs = {"both": (False, True), "on": (True,), "off": (False,)}[args.graph]
    print(json.dumps({"card": card(), "host_cpus": os.cpu_count(), "loop_threads": args.threads}), flush=True)
    for name in args.datasets.split(","):
        net_hw, frame_hw, params, _ = DATASETS[name]
        line = {"dataset": name, "network_hw": list(net_hw), "frame_hw": list(frame_hw), "batch": BATCH,
                "flownet": params["flownet"], "augment": True}
        with tempfile.TemporaryDirectory() as root:
            make_tree(os.path.join(root, 'data'), name, frame_hw)
            line["input_pairs_per_s"] = {str(t): time_input(root, name, net_hw, t, args.batches)
                                         for t in sorted({1, BATCH, os.cpu_count() or 1})}
            line["loop"] = {}
            for precision in args.modes.split(","):
                for graph in graphs:
                    key = "%s%s" % (precision, "+graph" if graph else "")
                    line["loop"][key] = time_loop(root, name, net_hw, params, precision, graph, args.threads,
                                                  args.steps, args.warmup)
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
