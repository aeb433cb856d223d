#!/usr/bin/env python
"""Training-step time with TensorBoard summaries, against the same step without them.

    python tools/bench_summary.py [--steps 100] [--rounds 3] [--images]

The unsupervised FlowNetC step of run.py (augmentation on, [train_kitti]'s loss, 4 synthetic pairs at
320x1152, one GPU, 3xTF32 convs) is captured as one CUDA graph and replayed in three settings, which
alternate within every round:
  none   the loss is printed every 50 steps (run.py's default display_interval), no writer;
  50     summaries written every 50 steps, as run.py writes them;
  1      summaries written every step.
``--images`` also writes the image summaries (run.py does with ``--debug``).  Each window is
``--steps`` replays timed with the host clock between device synchronisations.  Prints the card's
name and power limit, then one JSON line per setting with the ms/step of every round.  The event
files go to a temporary directory.
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

import torch  # noqa: E402

from unflow_b200 import synthetic as synth  # noqa: E402

BATCH, HW = 4, (320, 1152)
PARAMS = dict(flownet='C', pyramid_loss=True, border_mask=True, ternary_weight=1.0, smooth_2nd_weight=3.0,
              learning_rate=1.0e-5, decay_interval=100000, decay_after=100000, fb_weight=0.2,
              mask_occlusion='fb', occ_weight=12.4)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as e:          # the card's name still comes from CUDA
        q = "nvidia-smi unavailable (%s)" % e
    return {"cuda_name": torch.cuda.get_device_name(0), "nvidia_smi": q}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", action="store_true", help="also write the image summaries (run.py --debug)")
    args = ap.parse_args()
    from unflow_b200 import run as R
    from unflow_b200.e2eflow.core import augment
    from unflow_b200.e2eflow.core.summary import SummaryWriter
    from unflow_b200.e2eflow.core.train import Trainer, learning_rate_at
    print(json.dumps(card()))
    dev = torch.device("cuda", 0)
    tr = Trainer(PARAMS, synth.KITTI_NORMALIZATION, dev, seed=1234, augment=True)
    tr.track_images = args.images
    augment.seed(4321)
    im1, im2, _ = synth.image_pair(BATCH, HW[0], HW[1], seed=1234)
    im1, im2 = im1.to(dev), im2.to(dev)
    tr.capture(im1, im2)
    for _ in range(3):
        tr.step(im1, im2)
    torch.cuda.synchronize()
    settings = {"none": (50, False), "50": (50, True), "1": (1, True)}
    times = {k: [] for k in settings}
    with tempfile.TemporaryDirectory() as tmp:
        writer = SummaryWriter(os.path.join(tmp, "train"))
        for _ in range(args.rounds):
            for name, (interval, write) in settings.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for k in range(1, args.steps + 1):
                    loss = tr.step(im1, im2)
                    if k % interval == 0:
                        float(loss)                         # run.py prints the loss at a display step
                        if write:
                            R.write_train_summaries(writer, tr, tr.iteration,
                                                    learning_rate_at(tr.iteration - 1, PARAMS), images=args.images)
                torch.cuda.synchronize()
                times[name].append(round((time.perf_counter() - t0) * 1e3 / args.steps, 3))
        writer.close()
    for name, (interval, write) in settings.items():
        print(json.dumps({"setting": name, "display_interval": interval, "summaries": write, "images": args.images
                          and write, "steps": args.steps, "ms_per_step": times[name]}))


if __name__ == "__main__":
    main()
