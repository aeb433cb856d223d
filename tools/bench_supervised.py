#!/usr/bin/env python
"""Time the supervised KITTI fine-tune step (dataset = kitti_ft) on one H100.

    python tools/bench_supervised.py [--spec C|CSS] [--steps K] [--warmup W] [--batch B] [--dump-outputs DIR]

Step: forward of the network stack (forward flow only), the fused Charbonnier loss of
csrc/supervised_loss.cu against seeded ground truth with a sparse mask (synthetic.supervised_batch),
backward and Adam, on B pairs of 320x768 (the [train_kitti_ft] crop).  A stacked --spec trains
every network (train_all), so every network adds a loss term.  The conv stacks run in bench.py's
default 3xTF32 mode (--conv fp32: cuDNN float32).

One JSON line: ``value`` frame-pairs/s with the inputs resident in HBM and the step replayed as one
CUDA graph (CUDA events around the timed steps, synchronised on both sides); ``e2e`` the same through
Trainer.step with the four tensors in pinned host memory; ``rooflines`` the two supervised-loss
kernels, per-launch CUDA-event time from an eager pass against their algorithmic bytes and the
H100 SXM data-sheet HBM rate; ``clocks`` nvidia-smi samples of the timed region (bench.py's sampler).
--dump-outputs DIR writes the loss of the last timed step and a seeded sample of the parameters and
Adam moments (bench.py's format).  Nothing is written to the tree.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from unflow_b200 import synthetic as synth  # noqa: E402

H, W = 320, 768        # config_template [train_kitti_ft] height x width


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--spec", default="C", help="network stack; a stacked spec trains every network (train_all)")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=4, help="image pairs per step")
    ap.add_argument("--conv", default=os.environ.get("UNFLOW_CONV_PRECISION", "3xtf32"), choices=["fp32", "3xtf32"],
                    help="arithmetic of the conv stacks, as in bench.py: 3xtf32 = tensor cores at fp32-level "
                         "accuracy, fp32 = plain cuDNN float32")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_supervised.py needs a CUDA device")

    from unflow_b200 import _native
    from unflow_b200.e2eflow import ops
    from unflow_b200.e2eflow.core import conv_ops
    from unflow_b200.e2eflow.core.train import Trainer
    _native.lib()
    conv_ops.set_mode(args.conv)
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda", 0)
    params = dict(flownet=args.spec, learning_rate=1.0e-5, train_all=len(args.spec) > 1)
    trainer = Trainer(params, synth.KITTI_NORMALIZATION, dev, seed=1234, supervised=True)
    h_batch = tuple(t.pin_memory() for t in synth.supervised_batch(args.batch, H, W, seed=1234))
    d_batch = tuple(t.to(dev) for t in h_batch)
    loss_host = torch.zeros((), dtype=torch.float32).pin_memory()
    sampler = bench.ClockSampler(0)
    sampler.start()

    def timed(fn, steps, hook=False):
        torch.cuda.synchronize()
        if hook:
            ops.kernel_timer.enable()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        start.record()
        for _ in range(steps):
            last = fn()
        end.record()
        torch.cuda.synchronize()
        t1 = time.time()
        ktimes = ops.kernel_timer.collect() if hook else {}
        return start.elapsed_time(end), ktimes, sampler.window(t0, t1), last

    for _ in range(max(args.warmup, 3)):
        trainer.step(*d_batch)
    eager_steps = min(args.steps, 5)
    ms_eager, ktimes, _, _ = timed(lambda: trainer.step(*d_batch), eager_steps, hook=True)
    kbytes = dict(ops.kernel_timer.bytes)

    trainer.capture(*d_batch)
    for _ in range(2):
        trainer.step(*d_batch)
    ms, _, clocks, last = timed(lambda: trainer.step(*d_batch), args.steps)
    if args.dump_outputs:
        bench.dump_outputs(args.dump_outputs, trainer, last)

    def e2e_step():
        loss = trainer.step(*h_batch)
        loss_host.copy_(loss, non_blocking=True)
        return loss

    for _ in range(2):
        e2e_step()
    ms_e2e, _, _, _ = timed(e2e_step, args.steps)
    torch.cuda.synchronize()
    sampler.close()

    peaks = bench.load_peaks()
    roofs = []
    for name in ("supervised_loss_fwd_%dx%d" % (H, W), "supervised_loss_bwd_%dx%d" % (H, W)):
        t = ktimes.get(name)
        if not t:
            continue
        avg = sum(t) / len(t) * 1e-3
        nbytes = kbytes.get(name, 0) / len(t)
        roofs.append({"kernel": name, "bound": "hbm", "launches_timed": len(t), "avg_us": round(avg * 1e6, 2),
                      "achieved": round(nbytes / avg / 1e9, 1), "peak": peaks["hbm_gbs"], "unit": "GB/s",
                      "frac": round(nbytes / avg / 1e9 / peaks["hbm_gbs"], 4), "peak_source": peaks["_source"],
                      "algorithmic_bytes": nbytes})
    line = {
        "metric": "frame-pairs/s at %dx%d FlowNet%s supervised fine-tune" % (H, W, args.spec),
        "value": round(args.batch * args.steps / (ms * 1e-3), 3), "unit": "frame-pairs/s",
        "ms_per_step": round(ms / args.steps, 3), "steps": args.steps, "warmup": args.warmup,
        "ms_per_step_eager": round(ms_eager / eager_steps, 3),
        "config": {"flownet": args.spec, "conv_precision": args.conv, "train_all": len(args.spec) > 1,
                   "batch": args.batch, "cuda_graph": True,
                   "data": "synthetic (seeded pairs, true flow, 40 % valid mask, -512 elsewhere; random-init weights)"},
        "e2e": {"value": round(args.batch * args.steps / (ms_e2e * 1e-3), 3), "unit": "frame-pairs/s",
                "ms_per_step": round(ms_e2e / args.steps, 3),
                "h2d_bytes_per_step": sum(t.numel() for t in h_batch) * 4, "d2h_bytes_per_step": 4},
        "rooflines": roofs,
        "clocks": clocks,
        "final_loss": float(loss_host.item()),
    }
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
