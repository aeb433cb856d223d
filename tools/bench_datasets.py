#!/usr/bin/env python
"""Training-step time and host input rate at the FlyingChairs, SYNTHIA and Cityscapes geometries
(and KITTI's, for comparison).

    python tools/bench_datasets.py [--steps 20] [--warmup 3] [--batches 12]

Prints the card's name and power limit, then one JSON line per dataset:
  step   the unsupervised FlowNetC training step (bidirectional forward, 5-level loss with that
         dataset's [train_<dataset>] loss parameters of config_template/config.ini, backward, Adam) on
         4 synthetic pairs at the network size, one GPU, 3xTF32 convs, replayed as one CUDA graph --
         bench.py's headline rules: ``--warmup`` eager steps, capture, two replays, ``--steps`` timed
         between CUDA events;
  input  the host pipeline (PNG decode, crop, pinned batch of 4) on a generated PNG tree at the
         dataset's frame size, in pairs/s, with 1 decode thread and with os.cpu_count() threads
         ([run] num_input_threads); the first batch is not timed.
Everything it writes goes to a temporary directory.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from unflow_b200 import synthetic as synth  # noqa: E402

BATCH = 4
BASE = dict(flownet='C', pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0)
# dataset -> (network height x width, frame height x width, loss parameters, input_raw arguments)
DATASETS = {
    'chairs': ((384, 512), (384, 512), dict(BASE, learning_rate=1.0e-4), dict(sequence=False, needs_crop=False)),
    'synthia': ((512, 768), (760, 1280), dict(BASE, learning_rate=1.0e-4), dict()),
    'cityscapes': ((512, 1024), (1024, 2048),
                   dict(BASE, learning_rate=1.0e-5, fb_weight=0.2, mask_occlusion='fb', occ_weight=12.4),
                   dict(skip=[0, 1])),
    # for comparison: KITTI raw at [train_kitti]'s crop
    'kitti': ((320, 1152), (375, 1242),
              dict(BASE, learning_rate=1.0e-5, fb_weight=0.2, mask_occlusion='fb', occ_weight=12.4), dict()),
}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the card's name still comes from CUDA
        q = "nvidia-smi unavailable (%s)" % e
    return {"cuda_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def time_step(hw, params, steps, warmup):
    from unflow_b200.e2eflow.core.train import Trainer
    from unflow_b200.e2eflow.core import conv_ops
    assert conv_ops.get_mode() == "3xtf32"
    dev = torch.device("cuda", 0)
    trainer = Trainer(params, synth.KITTI_NORMALIZATION, dev, seed=1234)
    im1, im2, _ = synth.image_pair(BATCH, hw[0], hw[1], seed=1234)
    im1, im2 = im1.to(dev), im2.to(dev)
    for _ in range(warmup):
        trainer.step(im1, im2)
    trainer.capture(im1, im2)
    for _ in range(2):
        trainer.step(im1, im2)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        loss = trainer.step(im1, im2)
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / steps
    return {"ms_per_step": round(ms, 3), "pairs_per_s": round(BATCH / (ms * 1e-3), 2),
            "final_loss": float(loss)}


def make_tree(root, frame_hw, n_frames=16):
    """One sequence directory of ``n_frames`` PNG frames (smooth synthetic images)."""
    import cv2
    d = os.path.join(root, 'seq')
    os.makedirs(d)
    for i in range(0, n_frames, 2):
        a, b, _ = synth.image_pair(1, frame_hw[0], frame_hw[1], seed=i)
        for k, im in enumerate((a, b)):
            cv2.imwrite(os.path.join(d, '%06d.png' % (i + k)), im[0].clamp(0, 255).byte().numpy())
    return [d]


def time_input(dirs, net_hw, raw_kw, threads, batches):
    from unflow_b200.e2eflow.kitti.input import KITTIInput

    class Data:
        current_dir = os.path.dirname(dirs[0])

        def get_raw_dirs(self):
            return dirs

    stream = KITTIInput(Data(), BATCH, net_hw, normalize=False, num_threads=threads).input_raw(
        swap_images=False, **raw_kw)
    try:
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
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batches", type=int, default=12, help="timed input batches per thread count")
    ap.add_argument("--datasets", default=",".join(DATASETS), help="comma separated; a name may repeat")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_datasets needs a CUDA device")
    from unflow_b200 import _native
    from unflow_b200.e2eflow.core import conv_ops
    import unflow_b200.e2eflow.core.train  # noqa: F401  (importing flownet sets the conv mode from the environment)
    _native.lib()
    conv_ops.set_mode("3xtf32")
    torch.backends.cudnn.benchmark = True
    print(json.dumps({"card": card(), "host_cpus": os.cpu_count()}), flush=True)
    for name in args.datasets.split(","):
        net_hw, frame_hw, params, raw_kw = DATASETS[name]
        line = {"dataset": name, "network_hw": list(net_hw), "frame_hw": list(frame_hw), "batch": BATCH,
                "flownet": "C", "conv": "3xtf32", "cuda_graph": True,
                "loss": {k: v for k, v in params.items() if k not in ('flownet', 'learning_rate')}}
        line["step"] = time_step(net_hw, params, args.steps, max(args.warmup, 3))
        with tempfile.TemporaryDirectory() as root:
            dirs = make_tree(root, frame_hw)
            line["input_pairs_per_s"] = {str(t): time_input(dirs, net_hw, raw_kw, t, args.batches)
                                         for t in sorted({1, os.cpu_count() or 1})}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
