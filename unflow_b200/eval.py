"""Evaluate experiments on a dataset variant and write benchmark / visualisation files -- the
non-interactive part of the reference's ``eval_gui.py`` (src/eval_gui.py:96-352):

    python -m unflow_b200.eval --dataset kitti --variant train_2012 --ex my_experiment --num 10
    python -m unflow_b200.eval --variant test_2015 --ex C,CSS --num -1 --output_benchmark
    python -m unflow_b200.eval --dataset sintel --variant train_final --ex C --num -1

Datasets and variants: kitti (train_2012, train_2015, test_2012, test_2015), chairs (test),
sintel (train_clean, train_final, test_clean, test_final), mdb (train, test); with ``--num -1``
the Sintel test variants evaluate 552 pairs and Middlebury test 12, as the reference does.

For every experiment in ``--ex`` the newest checkpoint is looked up under [dirs] log /ex/<name>, then
[dirs] checkpoints/<name> (eval_gui.py:100-108; TensorFlow checkpoints of the reference and this
implementation's ``.pt`` files are both accepted), the networks are restored, and every example is
run at the dataset's fixed size (KITTI 384x1280, FlyingChairs 384x512, Sintel 512x1024,
Middlebury 512x640): ``resize_input`` -> ``unsupervised_loss(...,
augment=False, return_flow=True)`` -> ``resize_output_flow`` back to the file size.  Printed per
experiment: ``EPE_noc, EPE_all, outliers_noc, outliers_all`` (eval_gui.py:175-178), or ``EPE_all`` /
nothing for variants with other / no ground truth.  ``--output_benchmark`` writes
``<out>/<ex>/%06d_10.png`` 16-bit KITTI flow files (``flow_to_int16``: u*64+2^15 clamped and
truncated, validity 1 -- eval_gui.py:67-73) or ``.flo`` with ``--no-output_png``;
``--output_backward`` adds ``_01`` files; ``--output_visual`` writes overlay / flow-colour / error
images.  The GUI pages (``e2eflow.gui.display``) are out of scope.
"""
import argparse
import os
import shutil
import sys

import numpy as np
import torch

from .run import config_dict, convert_input_strings, latest_checkpoint

KITTI_VARIANTS = ('train_2012', 'train_2015', 'test_2012', 'test_2015')
# dataset -> (variants, network input height x width) (eval_gui.py:298-322)
DATASETS = {'kitti': (KITTI_VARIANTS, (384, 1280)),
            'chairs': (('test',), (384, 512)),
            'sintel': (('train_clean', 'train_final', 'test_clean', 'test_final'), (512, 1024)),
            'mdb': (('train', 'test'), (512, 640))}
# pairs evaluated with --num -1 where the reference sets a number (eval_gui.py:315-322)
ALL_PAIRS = {('sintel', 'test_clean'): 552, ('sintel', 'test_final'): 552, ('mdb', 'test'): 12}


def check_variant(dataset, variant):
    if dataset not in DATASETS:
        raise SystemExit("--dataset %s: must be one of %s" % (dataset, ', '.join(DATASETS)))
    if variant not in DATASETS[dataset][0]:
        raise SystemExit("--variant %s: %s has %s" % (variant, dataset, ', '.join(DATASETS[dataset][0])))


def dataset_input(dataset, variant, data_dir):
    """The input object of ``dataset`` at its network size (batch 1, unnormalised) and the iterator of
    ``variant``: ``(im1, im2, input_shape[, ground truth])`` per pair."""
    check_variant(dataset, variant)
    dims = DATASETS[dataset][1]
    if dataset == 'kitti':
        from .e2eflow.kitti.data import KITTIData
        from .e2eflow.kitti.input import KITTIInput
        need = 'data_stereo_flow' if variant.endswith('2012') else 'data_scene_flow'
        data_input = KITTIInput(KITTIData(data_dir, development=True, require=(need,)), batch_size=1,
                                normalize=False, dims=dims)
    elif dataset == 'chairs':
        from .e2eflow.chairs.data import ChairsData
        from .e2eflow.chairs.input import ChairsInput
        data_input = ChairsInput(ChairsData(data_dir), batch_size=1, normalize=False, dims=dims)
    elif dataset == 'sintel':
        from .e2eflow.sintel.data import SintelData
        from .e2eflow.sintel.input import SintelInput
        data_input = SintelInput(SintelData(data_dir), batch_size=1, normalize=False, dims=dims)
    else:
        from .e2eflow.middlebury.data import MiddleburyData
        from .e2eflow.middlebury.input import MiddleburyInput
        data_input = MiddleburyInput(MiddleburyData(data_dir), batch_size=1, normalize=False, dims=dims)
    return data_input, getattr(data_input, 'input_' + variant)


def flow_to_int16(flow):
    """eval_gui.py:67-73: [1,h,w,2] float -> [h,w,3] uint16 (u, v, 1), clamped, truncated."""
    f = np.asarray(flow, dtype=np.float32)[0]
    enc = np.maximum(np.float32(0.0), np.minimum(f * np.float32(64.0) + np.float32(32768.0), np.float32(65535.0)))
    out = np.ones(f.shape[:2] + (3,), dtype=np.uint16)
    out[..., 0:2] = enc.astype(np.uint16)
    return out


def write_rgb_png(z, path, bitdepth=8):
    """eval_gui.py:59-64: first image of a batch as an RGB PNG (8 or 16 bit)."""
    from .e2eflow.core import flow_io
    z = np.asarray(z)
    if z.ndim == 4:
        z = z[0]
    if bitdepth == 16:
        flow_io.write_png16(path, z.astype(np.uint16))
        return
    import cv2
    z = np.clip(z, 0, 255).astype(np.uint8)
    if z.shape[2] == 1:
        z = np.repeat(z, 3, 2)
    if not cv2.imwrite(path, np.ascontiguousarray(z[:, :, ::-1])):
        raise IOError("cannot write " + path)


def network_flow_fn(params, normalization, variables):
    """The flow estimator of an experiment: frames [1,H,W,3] in [0,255] -> (flow_fw, flow_bw) in pixels."""
    from .e2eflow.core.unsupervised import unsupervised_loss

    def fn(im1, im2):
        with torch.no_grad():
            _, fw, bw = unsupervised_loss((im1, im2), params, normalization, augment=False,
                                          return_flow=True, variables=variables)
        return fw, bw
    return fn


def evaluate_examples(name, items, dims, flow_fn, device, num=10, out_dir=None, output_benchmark=False,
                      output_visual=False, output_backward=False, output_png=True, log=sys.stdout):
    """The per-example loop of ``_evaluate_experiment`` (eval_gui.py:110-310).  ``items`` yields what
    the input classes deliver: ``(im1, im2, input_shape[, flow_occ, mask_occ, flow_noc, mask_noc |
    flow_gt, mask])`` padded / cropped to ``dims``.  Returns ``{scalar name: average}``."""
    from .e2eflow.core import flow_util
    from .e2eflow.core.flow_io import resize_output_flow, write_flo
    from .e2eflow.core.input import resize_image_with_crop_or_pad, resize_input
    from .e2eflow.core import tf_image
    rh, rw = dims
    sums, n = {}, 0
    max_iter = num if num > 0 else None
    for item in items:
        if max_iter is not None and n == max_iter:
            break
        h, w = int(item[2][0, 0]), int(item[2][0, 1])
        im1 = resize_input(item[0].to(device), h, w, rh, rw)
        im2 = resize_input(item[1].to(device), h, w, rh, rw)
        flow, flow_bw = flow_fn(im1, im2)
        flow = resize_output_flow(flow, h, w).contiguous()
        flow_bw = resize_output_flow(flow_bw, h, w).contiguous()
        truth = [resize_image_with_crop_or_pad(t[0].to(device), h, w).unsqueeze(0) for t in item[3:]]
        scalars = {}
        if len(truth) == 4:
            flow_occ, mask_occ, flow_noc, mask_noc = truth
            scalars = {'EPE_noc': flow_util.flow_error_avg(flow_noc, flow, mask_noc),
                       'EPE_all': flow_util.flow_error_avg(flow_occ, flow, mask_occ),
                       'outliers_noc': flow_util.outlier_pct(flow_noc, flow, mask_noc),
                       'outliers_all': flow_util.outlier_pct(flow_occ, flow, mask_occ)}
        elif len(truth) == 2:
            scalars = {'EPE_all': flow_util.flow_error_avg(truth[0], flow, truth[1])}
        for k, v in scalars.items():
            sums[k] = sums.get(k, 0.0) + float(v)
        iterstr = str(n).zfill(6)
        if output_visual and out_dir:
            im1_o = tf_image.resize_bilinear(im1, [h, w])
            im2_o = tf_image.resize_bilinear(im2, [h, w])
            write_rgb_png(((im1_o * 0.5 + im2_o * 0.5)).cpu().numpy(), os.path.join(out_dir, iterstr + '_img.png'))
            write_rgb_png((flow_util.flow_to_color(flow) * 255).cpu().numpy(), os.path.join(out_dir, iterstr + '_flow.png'))
            if len(truth) == 4:
                err = flow_util.flow_error_image(flow, truth[0], truth[1], truth[3])
                write_rgb_png((err * 255).cpu().numpy(), os.path.join(out_dir, iterstr + '_err.png'))
        if output_benchmark and out_dir:
            targets = [(flow, '_10')] + ([(flow_bw, '_01')] if output_backward else [])
            for f, suffix in targets:
                if output_png:
                    write_rgb_png(flow_to_int16(f.cpu().numpy()), os.path.join(out_dir, iterstr + suffix + '.png'),
                                  bitdepth=16)
                else:
                    write_flo(os.path.join(out_dir, iterstr + suffix + '.flo'), f[0].cpu().numpy())
        n += 1
        log.write("-- evaluating '{}': {}/{}\n".format(name, n, max_iter))
    averages = {k: v / max(n, 1) for k, v in sums.items()}
    for k in ('EPE_noc', 'EPE_all', 'outliers_noc', 'outliers_all'):
        if k in averages:
            log.write("({}) {} = {}\n".format(name, k, averages[k]))
    return averages


def experiment_setup(name, default_config_path, dataset):
    """eval_gui.py:97-116: experiment directory, its config and its newest checkpoint."""
    current = config_dict(default_config_path)
    exp_dir = os.path.join(current['dirs'].get('log', ''), 'ex', name)
    config_path = os.path.join(exp_dir, 'config.ini')
    if not os.path.isfile(config_path):
        config_path = default_config_path
    ckpt = latest_checkpoint(exp_dir) if os.path.isdir(exp_dir) else None
    if ckpt is None:
        exp_dir = os.path.join(current['dirs'].get('checkpoints', ''), name)
        ckpt = latest_checkpoint(exp_dir)
    if ckpt is None:
        raise RuntimeError("Error: experiment must contain a checkpoint")
    config = config_dict(config_path)
    params = config['train']
    convert_input_strings(params, current['dirs'])
    if 'train_' + dataset in config:
        params.update(config['train_' + dataset])
    return params, ckpt, config_path


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--dataset', default='kitti', choices=tuple(DATASETS))
    ap.add_argument('--variant', default='train_2012',
                    help='; '.join('%s: %s' % (d, ', '.join(v)) for d, (v, _) in DATASETS.items()))
    ap.add_argument('--ex', default='', help='Experiment name(s) (can be comma separated list).')
    ap.add_argument('--num', type=int, default=10, help='Number of examples to evaluate. -1 = all.')
    ap.add_argument('--gpu', default='0',
                    help='GPU id(s), comma separated; evaluation runs on the first listed id (eval_gui.py '
                         'sets CUDA_VISIBLE_DEVICES to the list and uses its first device)')
    ap.add_argument('--output_benchmark', action='store_true', help='Output raw flow files.')
    ap.add_argument('--output_visual', action='store_true', help='Output flow visualization files.')
    ap.add_argument('--output_backward', action='store_true', help='Output backward flow files.')
    ap.add_argument('--output_png', dest='output_png', action='store_true', default=True)
    ap.add_argument('--no-output_png', dest='output_png', action='store_false', help='write .flo instead')
    ap.add_argument('--config', default=os.environ.get('UNFLOW_CONFIG', '../config.ini'))
    ap.add_argument('--out', default='../out')
    args = ap.parse_args(argv)
    check_variant(args.dataset, args.variant)
    if not torch.cuda.is_available():
        raise SystemExit("unflow_b200.eval needs a CUDA device (no CPU fallback)")
    device = torch.device('cuda', int(args.gpu.split(',')[0]))
    torch.cuda.set_device(device)
    return run_eval(args, device)


def run_eval(args, device, make_flow_fn=network_flow_fn):
    """``main`` after argument parsing; ``make_flow_fn(params, normalization, variables)`` builds the
    estimator (the tests substitute a stub to exercise everything around the network on the CPU)."""
    print("-- evaluating: on {} pairs from {}/{}".format(args.num, args.dataset, args.variant))

    from .e2eflow.core.flownet import FlowNetVariables
    from .run import restore_checkpoint
    dirs = config_dict(args.config)['dirs']
    data_input, input_fn = dataset_input(args.dataset, args.variant, dirs['data'])
    num = args.num
    if num == -1:
        num = ALL_PAIRS.get((args.dataset, args.variant), num)
    results = {}
    for name in [n for n in args.ex.split(',') if n]:
        params, ckpt, config_path = experiment_setup(name, args.config, args.dataset)
        variables = FlowNetVariables(params.get('flownet', 'S'), params.get('full_res'), seed=0).to(device)

        class _Holder:       # restore_checkpoint only touches .variables unless optimiser state is asked for
            pass
        holder = _Holder()
        holder.variables = variables
        restore_checkpoint(holder, ckpt[1])
        out_dir = None
        if args.output_visual or args.output_benchmark:
            out_dir = os.path.join(args.out, name)
            if os.path.isdir(out_dir):
                shutil.rmtree(out_dir)
            os.makedirs(out_dir)
            shutil.copyfile(config_path, os.path.join(out_dir, 'config.ini'))
        results[name] = evaluate_examples(
            name, input_fn(), data_input.dims, make_flow_fn(params, data_input.get_normalization(), variables),
            device, num=num, out_dir=out_dir, output_benchmark=args.output_benchmark,
            output_visual=args.output_visual, output_backward=args.output_backward, output_png=args.output_png)
    return results


if __name__ == '__main__':
    main()
