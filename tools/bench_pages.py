#!/usr/bin/env python
"""What the evaluation pages cost: ``eval --output_pages`` and ``[run] interactive_plot``, each against the
same run without them.

    python tools/bench_pages.py [--pairs 100] [--rounds 2] [--chunk 500] [--eval-pairs 194] [--skip-train]

eval   ``python -m unflow_b200.eval --dataset kitti --variant train_2015 --num <pairs>`` on a generated KITTI
       2015 tree at the real frame size (375x1242), FlowNetC experiments with 3xTF32 convs, for 1 and 3
       experiments, without and with ``--output_pages`` (``--num_vis`` = pairs).  The settings alternate
       within every round.  Wall time of ``eval.main`` from the host clock (it ends with the metrics'
       device-to-host reads); ``pages_write_s`` is the part spent rendering and encoding the pages.
train  ``run.main`` on a generated KITTI tree as ``[train_kitti]`` configures it (320x1152, batch 4,
       augmentation on, 3xTF32, ``--graph``), evaluating after every ``--chunk`` iterations on a KITTI 2012
       training set of ``--eval-pairs`` pairs at 375x1242 (the real set has 194), without and with
       ``interactive_plot = True``.  Two chunks run; ``chunk_s`` is the second one, from the end of the
       first evaluation to the end of the second, so it holds the page writing of the first evaluation
       on the background thread; ``eval_s`` the evaluations; ``final_join_s`` how long the end of the run
       waited for the last pages.  The default ``save_interval`` is 5000 iterations, which hides the page
       writing further.
The generated frames are smooth synthetic images; the trees repeat 10 distinct pairs.  Prints the card's
name and power limit, then one JSON line per measurement.  Everything it writes goes to a temporary
directory.
"""
import argparse
import contextlib
import io
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_datasets import card  # noqa: E402
from bench_train_loop import make_tree  # noqa: E402
from unflow_b200 import synthetic as synth  # noqa: E402

LOSS = ["flownet = C", "pyramid_loss = True", "border_mask = True", "ternary_weight = 1.0",
        "smooth_2nd_weight = 3.0", "fb_weight = 0.2", "mask_occlusion = fb", "occ_weight = 12.4"]
FRAME_HW = (375, 1242)
DISTINCT = 10


def write_gt_set(image_dir, flow_dir, n):
    """``n`` pairs ``%06d_10.png`` / ``_11.png`` with flow_occ / flow_noc ground truth, 10 distinct ones."""
    import cv2
    from unflow_b200.e2eflow.core import flow_io
    for d in (image_dir, flow_dir + '/flow_occ', flow_dir + '/flow_noc'):
        os.makedirs(d, exist_ok=True)
    for i in range(n):
        names = [os.path.join(image_dir, '%06d_1%d.png' % (i, k)) for k in (0, 1)]
        flows = [os.path.join(flow_dir, sub, '%06d_10.png' % i) for sub in ('flow_occ', 'flow_noc')]
        if i >= DISTINCT:
            for src, dst in zip([p.replace('%06d_' % i, '%06d_' % (i % DISTINCT)) for p in names + flows],
                                names + flows):
                shutil.copyfile(src, dst)
            continue
        a, b, f = synth.image_pair(1, FRAME_HW[0], FRAME_HW[1], seed=1000 + i)
        for path, im in zip(names, (a, b)):
            if not cv2.imwrite(path, im[0].clamp(0, 255).byte().numpy()[:, :, ::-1].copy()):
                raise IOError("cannot write " + path)
        for path in flows:
            flow_io.write_kitti_flow(path, f[0].numpy(), np.ones(FRAME_HW))


@contextlib.contextmanager
def timed(module, name, log, sync=True):
    """Patches ``module.name`` so that every call appends (start, end) to ``log``; with ``sync`` after a
    device synchronise at both ends (not for host-only work on another thread, which would wait for the
    training loop's kernels)."""
    orig = getattr(module, name)

    def wrapper(*args, **kwargs):
        if sync:
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = orig(*args, **kwargs)
        if sync:
            torch.cuda.synchronize()
        log.append((t0, time.perf_counter()))
        return out

    setattr(module, name, wrapper)
    try:
        yield log
    finally:
        setattr(module, name, orig)


def bench_eval(root, pairs, rounds):
    from unflow_b200 import eval as E
    from unflow_b200.e2eflow.core import pages, tf_checkpoint
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    tr = os.path.join(root, 'data', 'data_scene_flow', 'training')
    write_gt_set(os.path.join(tr, 'image_2'), tr, pairs)
    ini = os.path.join(root, 'eval.ini')
    with open(ini, 'w') as f:
        f.write("\n".join(["[dirs]", "log = %s/log" % root, "checkpoints = %s/ckpts" % root,
                           "data = %s/data" % root, "[run]", "batch_size = 4", "conv_precision = 3xtf32",
                           "[train]"] + LOSS) + "\n")
    names = ['e%d' % k for k in range(3)]
    for k, name in enumerate(names):
        tf_checkpoint.save_variables(FlowNetVariables('C', False, seed=20 + k),
                                     os.path.join(root, 'ckpts', name, 'model.ckpt-1'))

    def run(n_ex, with_pages, num):
        argv = ["--dataset", "kitti", "--variant", "train_2015", "--ex", ",".join(names[:n_ex]), "--num", str(num),
                "--config", ini, "--out", os.path.join(root, 'out')]
        if with_pages:
            argv += ["--output_pages", "--num_vis", str(num)]
        writes = []
        with timed(pages, 'write_pages', writes, sync=False), contextlib.redirect_stdout(io.StringIO()):
            t0 = time.perf_counter()
            E.main(argv)
            dt = time.perf_counter() - t0
        return dt, sum(b - a for a, b in writes)

    run(1, True, 5)       # warm-up: modules, conv plans, the resize tables of this size
    settings = [(n, p) for n in (1, 3) for p in (False, True)]
    results = {s: [] for s in settings}
    for _ in range(rounds):
        for s in settings:
            results[s].append(run(s[0], s[1], pairs))
    for (n, p), runs in results.items():
        print(json.dumps({"bench": "eval", "experiments": n, "output_pages": p, "pairs": pairs,
                          "wall_s": [round(t, 2) for t, _ in runs],
                          "ms_per_pair_per_experiment": [round(t * 1e3 / pairs / n, 1) for t, _ in runs],
                          "pages_write_s": [round(w, 2) for _, w in runs]}))


def bench_train(root, chunk, eval_pairs):
    from unflow_b200 import run as R
    from unflow_b200.e2eflow.core import pages
    data = os.path.join(root, 'data')
    make_tree(data, 'kitti', FRAME_HW)
    tr = os.path.join(data, 'data_stereo_flow', 'training')
    write_gt_set(os.path.join(tr, 'colored_0'), tr, eval_pairs)
    for plot in (False, True):
        ini = os.path.join(root, 'train_%d.ini' % plot)
        with open(ini, 'w') as f:
            f.write("\n".join(["[dirs]", "log = %s/log" % root, "checkpoints = %s/log/checkpoints" % root,
                               "data = %s" % data, "[run]", "batch_size = 4", "gpu_list = 0",
                               "num_input_threads = %d" % (os.cpu_count() or 1), "dataset = kitti",
                               "development = True", "conv_precision = 3xtf32",
                               "interactive_plot = %s" % plot, "[train]", "decay_interval = 100000",
                               "save_interval = %d" % chunk, "display_interval = 100000"] + LOSS +
                              ["[train_kitti]", "height = 320", "width = 1152", "num_iters = 500000",
                               "learning_rate = 1.0e-5", "decay_after = 100000"]) + "\n")
        evals, writes = [], []
        with timed(R, 'evaluate_kitti', evals), timed(pages, 'write_pages', writes, sync=False), \
                contextlib.redirect_stdout(io.StringIO()):
            R.main(["--ex", "bench_pages", "--config", ini, "--debug", "--ow", "--graph",
                    "--max-iters", str(2 * chunk)])
            end = time.perf_counter()
        out = {"bench": "train", "interactive_plot": plot, "chunk_iterations": chunk, "eval_pairs": eval_pairs,
               "chunk_s": round(evals[1][1] - evals[0][1], 2),
               "eval_s": [round(b - a, 2) for a, b in evals]}
        if plot:
            out["pages_write_s"] = [round(b - a, 2) for a, b in writes]
            out["final_join_s"] = round(end - evals[1][1], 2)
        print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--chunk", type=int, default=500, help="save_interval of the timed training run")
    ap.add_argument("--eval-pairs", type=int, default=194)
    ap.add_argument("--skip-train", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pages needs a CUDA device")
    print(json.dumps(card()))
    with tempfile.TemporaryDirectory() as root:
        bench_eval(os.path.join(root, 'eval'), args.pairs, args.rounds)
        if not args.skip_train:
            bench_train(os.path.join(root, 'train'), args.chunk, args.eval_pairs)


if __name__ == '__main__':
    main()
