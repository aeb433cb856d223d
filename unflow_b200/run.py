"""Training entry point with the reference's flags and config.ini semantics
(/root/reference/src/run.py:21-33, src/e2eflow/util.py:37-62, src/e2eflow/core/train.py:116-145):

    python -m unflow_b200.run --ex NAME [--debug] [--ow] [--config PATH] [--synthetic]
    python -m torch.distributed.run --nproc-per-node N -m unflow_b200.run --ex NAME   (alternative launcher)

* ``config.ini`` sections [dirs] [run] [train] [train_<dataset>] are parsed with the same type
  coercion (int -> float -> bool -> str); the dataset section overrides [train]
  (run.py:91-92); ``manual_decay_*`` strings become lists and define ``num_iters``.
* [run] gpu_list (run.py:40-49, ``launch.py``): ``gpu_list = 3`` trains in this process on GPU 3;
  ``gpu_list = 0,1,2,3`` trains data parallel from the one command above -- it starts one worker per
  listed GPU (worker k on the k-th listed GPU, ``CUDA_VISIBLE_DEVICES`` set to the list), waits on them and
  stops them all when one fails or the command is interrupted.  Ids count the devices the command sees;
  duplicate, negative or absent ids are rejected before anything starts.  Without the key the run trains
  on ``cuda:LOCAL_RANK``; under an external launcher (``WORLD_SIZE`` set) gpu_list is not used and the
  launcher's processes train.
* [run] batch_size is the TOTAL batch, divided by the number of GPUs (run.py:48).
* training runs in chunks of ``save_interval`` iterations; after each chunk a checkpoint is
  written and training resumes from the newest checkpoint by parsing the iteration from the file
  name (train.py:124-135, 258-259).  ``--ckpt-format pt`` (default) writes ``model.ckpt-<iter>.pt``
  (variables under their TF names, TF layout); ``--ckpt-format tf`` writes the reference's own
  format (``model.ckpt-<iter>.index`` / ``.data-00000-of-00001`` + the ``checkpoint`` state file,
  core/tf_checkpoint.py), which the reference's Saver can restore.  Either kind is accepted on
  resume and for ``finetune``.  ``--ow`` discards an existing experiment, ``--debug`` disables
  checkpoint writing.
* experiment directories (experiment.py): when training ends -- also when there was nothing left to
  train ("max_iter reached") -- rank 0 concludes the experiment (run.py:204-205): the newest checkpoint
  of [dirs] checkpoints /<name> is copied into [dirs] log /ex/<name>, the directory meant to be backed
  up, next to the earlier concluded ones; not with ``--debug``.  At start-up, when [dirs] checkpoints
  /<name> holds no checkpoint (missing or emptied) and log/ex/<name> does -- a concluded run or a
  pretrained model extracted there -- that one is copied back and training continues from it, with the
  reference's "Warning: intermediate checkpoints could not be restored."  Copies go through a temporary
  name and a rename, so a half-copied checkpoint is never visible under its final name.  ``--ow`` also
  removes the concluded checkpoints.
* [dirs] fast: before reading a dataset, local rank 0 of each node copies the KITTI directories and
  those of the training dataset from [dirs] data into [dirs] fast where they are missing there (a
  FlyingChairs release is converted in [dirs] data first), while the other ranks wait; the run then
  reads [dirs] fast.  An interrupted copy is redone by the next run; staged copies are kept.
* ``finetune = exA,exB`` ([train*] sections): network i of the stack is initialised from the
  newest checkpoint of experiment i -- looked up in [dirs] checkpoints, then [dirs] log /ex --
  with the reference's rules (util.py:75-85, train.py:23-62): when the experiment has no
  checkpoint of its own all listed networks are restored; when it resumes and ``train_all`` is off,
  the fixed networks (all but the last) are restored again from their sources; a checkpoint that
  lacks the ``full_res`` layers restores the rest.
* ``dataset = kitti`` with an existing [dirs] data directory trains on the KITTI raw sequences
  through the reference's pairing / shuffling / resume-shift rules (core/input.py, kitti/) and
  evaluates on the KITTI 2012 training set after every ``save_interval`` chunk; each rank reads
  its own shard of the batch stream.  With ``--synthetic`` (or when [dirs] data does not exist)
  batches are seeded synthetic pairs of the configured height x width.
* ``dataset = kitti_ft`` fine-tunes with ground truth (run.py:175-197): ``Trainer(supervised=True)``
  on ``input_train_gt(40)`` -- KITTI 2015 + 2012 training pairs with their flow_occ ground truth,
  the 40 held-out pairs of each set left out -- and evaluates after every ``save_interval`` chunk on
  those 40 held-out pairs of the 2015 training set.  Parameters are [train] updated by
  [train_kitti_ft].  With ``--synthetic`` the batches are seeded synthetic pairs with their true
  flow and a sparse validity mask (``synthetic.supervised_batch``).
* ``dataset = chairs | synthia | cityscapes`` trains unsupervised on FlyingChairs (unrelated 384x512
  pairs of ``flying_chairs/image``, converted from the release layout when needed), the SYNTHIA
  sequences (consecutive frames, random crop) or the Cityscapes sequences (frame distances 1 and 2,
  random crop) with the reference's arguments (run.py:62-173, ``dataset_inputs``), and like
  ``kitti`` evaluates on the KITTI 2012 training set after every chunk when it is under [dirs] data.
  [run] num_input_threads threads decode frames a few batches ahead (bit-identical batches for any count).
  With ``--synthetic`` every dataset trains on seeded synthetic pairs of its height x width.
  Datasets are never downloaded: a missing directory is an error naming the expected layout.
* [run] conv_precision = fp32 | 3xtf32: the arithmetic of the conv / deconv layers (core/conv_ops.py),
  set before the first network is built, for training and the in-training evaluation.  ``3xtf32`` runs
  them on the project's wgmma tensor-core kernels, ``fp32`` on cuDNN float32 (the reference's
  arithmetic).  Without the key the environment variable ``UNFLOW_CONV_PRECISION`` decides, else fp32.
  Workers started for ``gpu_list`` read the same config, so every rank uses the same mode, and
  ``eval.py`` evaluates an experiment in the mode of its copied config.
* TensorBoard summaries (train.py:66-86,187-261,314-370; experiment.py:14-25), from rank 0 only, also
  with ``--debug``: ``<[dirs] log>/ex/<name>/train`` gets the learning rate, every tracked loss and the
  weights of the weighted terms at i = 1 and every ``display_interval`` steps (the steps the loss is
  printed at); with ``--debug`` also the tracked images, as the reference adds image summaries in debug
  mode only.  ``<[dirs] log>/ex/<name>/eval`` gets the AEE / outlier averages and every tracked loss
  averaged over the evaluation set after every ``save_interval`` chunk, at that iteration.  ``--ow``
  removes both.  View them with ``tensorboard --logdir <[dirs] log>/ex``.
* [run] interactive_plot = True (train.py:287-308, 378-384): after every in-training evaluation rank 0 writes
  its pages to ``<[dirs] log>/ex/<name>/eval_pages/%06d.png``, one per evaluated pair, titled
  ``<name> (i=<iteration>)``, with the rows warped image, flow, occ, reverse disocc and flow error
  (``core/pages.py``); they replace the previous evaluation's pages, as the reference replaces its plot
  window.  Also with ``--debug``.  The PNGs are encoded on a background thread while training continues.
"""
import argparse
import configparser
import copy
import datetime
import filecmp
import glob
import os
import shutil
import sys

import torch
import torch.distributed as dist

KITTI_NORMALIZATION = ([104.920005, 110.1753, 114.785955], 1 / 0.0039216)  # core/input.py:45-46
FT_HOLD_OUT = 40    # pairs of each KITTI training set kept out of the fine-tune for evaluation (run.py:187-188)
STAGING_TIMEOUT = datetime.timedelta(hours=24)     # how long ranks wait for [dirs] fast to be filled
CONV_PRECISIONS = ('fp32', '3xtf32')                # core/conv_ops.py


def config_dict(config_path):
    """util.py:37-62: the config as a dict of sections with intuitively typed values."""
    config = configparser.ConfigParser()
    if not config.read(config_path):
        raise FileNotFoundError(config_path)
    d = dict()
    for section_key in config.sections():
        sd = dict()
        section = config[section_key]
        for key in section:
            val = section[key]
            try:
                sd[key] = int(val)
            except ValueError:
                try:
                    sd[key] = float(val)
                except ValueError:
                    try:
                        sd[key] = section.getboolean(key)
                    except ValueError:
                        sd[key] = val
        d[section_key] = sd
    return d


def convert_input_strings(config_dct, dirs=None):
    """util.py:65-85: the manual decay lists and, given ``dirs``, the ``finetune`` experiment names
    resolved to their newest checkpoints (``(iteration, path)`` as ``latest_checkpoint`` returns)."""
    if 'manual_decay_iters' in config_dct and 'manual_decay_lrs' in config_dct:
        iters_lst = [int(i) for i in str(config_dct['manual_decay_iters']).split(',')]
        lrs_lst = [float(l) for l in str(config_dct['manual_decay_lrs']).split(',')]
        config_dct['manual_decay_iters'] = iters_lst
        config_dct['manual_decay_lrs'] = lrs_lst
        config_dct['num_iters'] = sum(iters_lst)

    if 'finetune' in config_dct and dirs is not None:
        found = []
        for name in str(config_dct['finetune']).split(','):
            name = name.strip()
            ckpt = latest_checkpoint(os.path.join(dirs.get('checkpoints', ''), name))
            if ckpt is None:
                ckpt = latest_checkpoint(os.path.join(dirs.get('log', ''), 'ex', name))
            assert ckpt, "Could not load experiment " + name
            found.append(ckpt)
        config_dct['finetune'] = found


def conv_precision(run_config, default):
    """The conv arithmetic ``[run] conv_precision`` asks for: ``fp32`` (cuDNN float32, the reference's
    arithmetic) or ``3xtf32`` (the wgmma tensor-core kernels at fp32-level accuracy); ``default`` when
    the key is absent.  Any other value ends the command (SystemExit) naming both."""
    if 'conv_precision' not in run_config:
        return default
    value = run_config['conv_precision']
    if value not in CONV_PRECISIONS:
        raise SystemExit('[run] conv_precision = %s: must be %s' % (value, ' or '.join(CONV_PRECISIONS)))
    return value


def latest_checkpoint(ckpt_dir):
    """Newest checkpoint of an experiment directory as ``(iteration, path)``: a ``.pt`` file of
    this implementation or the prefix of a TF checkpoint named by the ``checkpoint`` state file
    (tf.train.get_checkpoint_state); None when there is none."""
    from .e2eflow.core import tf_checkpoint
    best = None
    for p in glob.glob(os.path.join(ckpt_dir, "model.ckpt-*.pt")):
        try:
            it = int(os.path.basename(p)[len("model.ckpt-"):-3])
        except ValueError:
            continue
        if best is None or it > best[0]:
            best = (it, p)
    state = tf_checkpoint.get_checkpoint_state(ckpt_dir)
    if state is not None and os.path.exists(state[0] + '.index'):
        try:
            it = tf_checkpoint.checkpoint_iteration(state[0])
        except ValueError:
            it = 0
        if best is None or it > best[0]:
            best = (it, state[0])
    return best


def external_restores(params, has_own_checkpoint):
    """restore_networks (train.py:23-37): which entries of ``finetune`` (one per network of the
    stack, in order) are loaded from their source experiments."""
    finetune = params.get('finetune', [])
    n_nets = len(params.get('flownet', 'S'))
    assert len(finetune) <= n_nets
    if params.get('train_all'):
        return finetune if not has_own_checkpoint else []
    return finetune if not has_own_checkpoint else finetune[:n_nets - 1]


def restore_checkpoint(trainer, path, nets=None, with_optimizer=False):
    """Load network variables (and optionally Adam's moments) from either checkpoint kind."""
    from .e2eflow.core import tf_checkpoint
    variables = trainer.variables
    if path.endswith('.pt'):
        state = torch.load(path, map_location='cpu')
        tensors = state['variables']
        if nets is not None:
            keep = {s for i in nets for s in variables.scopes_of_net(i)}
            tensors = {k: v for k, v in tensors.items() if k.rsplit('/', 1)[0] in keep}
        missing = [n for n in variables.variable_names()
                   if n not in tensors and (nets is None or n.rsplit('/', 1)[0] in keep)]
        if any('full_res' not in n for n in missing):
            raise KeyError("checkpoint %s lacks %s" % (path, missing[0]))
        variables.load_tf_dict(tensors, strict=False)
        if with_optimizer and 'adam_slots' in state:
            trainer.load_adam_slots(state['adam_slots'])
        return
    tf_checkpoint.restore_variables(variables, path, nets=nets)
    if with_optimizer:
        reader = tf_checkpoint.BundleReader(path)
        slots = {n: (reader.tensor(n + '/Adam'), reader.tensor(n + '/Adam_1'))
                 for n in trainer.trainable_names if n + '/Adam' in reader and n + '/Adam_1' in reader}
        trainer.load_adam_slots(slots)


def save_checkpoint(trainer, ckpt_dir, iteration, fmt='pt'):
    """train.py:258-259 ``saver.save(sess, save_path, global_step=i)``.  The reference's Saver
    holds only the trained networks unless ``train_all`` (train.py:32-37); here every network of
    the stack is written, so a checkpoint is self-contained (a superset of the reference's)."""
    from .e2eflow.core import tf_checkpoint
    prefix = os.path.join(ckpt_dir, 'model.ckpt-%d' % iteration)
    if fmt == 'tf':
        return tf_checkpoint.save_variables(trainer.variables, prefix, adam_slots=trainer.adam_slots())
    slots = {k: (torch.from_numpy(m), torch.from_numpy(v)) for k, (m, v) in trainer.adam_slots().items()}
    torch.save({'variables': trainer.variables.to_tf_dict(), 'adam_slots': slots}, prefix + '.pt')
    return prefix + '.pt'


def _replace_atomically(dst, write):
    """``write(tmp)`` fills ``dst + '.partial'``, which is flushed to disk and renamed to ``dst``; the
    directory is flushed after the rename, so the new name also survives a power loss.  Under its final
    name a file is complete or absent.  A failed write leaves no temporary file behind."""
    tmp = dst + '.partial'
    try:
        write(tmp)
        with open(tmp, 'rb+') as f:
            os.fsync(f.fileno())
        os.replace(tmp, dst)
    except BaseException:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise
    fd = os.open(os.path.dirname(os.path.abspath(dst)), os.O_RDONLY)
    try:
        os.fsync(fd)
    finally:
        os.close(fd)


def _write_text(path, text):
    with open(path, 'w') as f:
        f.write(text)


def copy_checkpoint(path, dst_dir):
    """experiment.py:61-74 (``_copy_latest_checkpoint``): the checkpoint ``path`` -- a ``.pt`` file or a TF
    prefix, as ``latest_checkpoint`` returns it -- copied into ``dst_dir`` under its own name.  A TF
    checkpoint's ``.data`` and ``.index`` files are followed by a ``checkpoint`` state file naming only
    this checkpoint, as the reference writes it.  Every file is replaced atomically and the state file
    comes last, so ``latest_checkpoint(dst_dir)`` finds the previous newest checkpoint or this complete
    one, never a part of it.  Files already there with the same bytes are left alone (a run concluded
    again).  A different TF checkpoint of the same name loses its ``.index`` before its ``.data`` is
    replaced, so no reader pairs the new data with the old index.  Returns the copy's path (or prefix)."""
    os.makedirs(dst_dir, exist_ok=True)
    src_dir, base = os.path.split(path)
    names = [base] if path.endswith('.pt') else [base + '.data-00000-of-00001', base + '.index']
    pending = [n for n in names if not (os.path.isfile(os.path.join(dst_dir, n)) and
                                        filecmp.cmp(os.path.join(src_dir, n), os.path.join(dst_dir, n),
                                                    shallow=False))]
    index = os.path.join(dst_dir, base + '.index')
    if not path.endswith('.pt') and pending and os.path.isfile(index):
        os.remove(index)
        pending = [n for n in names if n in pending or n.endswith('.index')]
    for name in pending:
        _replace_atomically(os.path.join(dst_dir, name),
                            lambda tmp, name=name: shutil.copyfile(os.path.join(src_dir, name), tmp))
    if not path.endswith('.pt'):
        state = 'model_checkpoint_path: "%s"\nall_model_checkpoint_paths: "%s"\n' % (base, base)
        _replace_atomically(os.path.join(dst_dir, 'checkpoint'), lambda tmp: _write_text(tmp, state))
    return os.path.join(dst_dir, base)


def conclude(ckpt_dir, ex_dir):
    """experiment.py:79-83 (``Experiment.conclude``): the newest checkpoint of ``ckpt_dir`` ([dirs]
    checkpoints /<name>, which need not be kept) copied into ``ex_dir`` ([dirs] log /ex/<name>, which
    should be backed up).  Earlier concluded checkpoints stay.  Returns the copy's path, or None when
    ``ckpt_dir`` holds no checkpoint."""
    ck = latest_checkpoint(ckpt_dir)
    if ck is None:
        print('Warning: no checkpoints written')
        return None
    return copy_checkpoint(ck[1], ex_dir)


def restore_concluded(ckpt_dir, ex_dir):
    """experiment.py:36-45 (``Experiment.__init__``): when ``ckpt_dir`` holds no checkpoint (missing or
    emptied) but ``ex_dir`` does -- a concluded experiment, or a pretrained model extracted there -- the
    newest one of ``ex_dir`` is copied into ``ckpt_dir``, so training continues from it.  Returns the
    copy's path, or None when nothing was copied."""
    if latest_checkpoint(ckpt_dir) is not None:
        return None
    ck = latest_checkpoint(ex_dir)
    if ck is None:
        return None
    path = copy_checkpoint(ck[1], ckpt_dir)
    print('Warning: intermediate checkpoints could not be restored.')
    return path


def remove_concluded(ex_dir):
    """``--ow``: the concluded checkpoints of ``ex_dir`` (``model.ckpt-*`` and the ``checkpoint`` state
    file) removed, so that a fresh run does not later restore the discarded model."""
    for p in glob.glob(os.path.join(ex_dir, 'model.ckpt-*')) + [os.path.join(ex_dir, 'checkpoint')]:
        if os.path.isfile(p):
            os.remove(p)


def kitti_inputs(dirs, run_config, params, train_dataset, gpu_batch_size, start_iter, rank, world):
    """The 'kitti' branch of the reference run.py (:31-58, :96-115): training batches from the raw
    sequences (``input_raw(swap_images=False, center_crop=True, shift=iterations_done * batch_size)``)
    and, when present, the KITTI 2012 training set with ground truth for evaluation at 384x1280.
    The 'kitti_ft' branch (:175-197): ground-truth batches from ``input_train_gt(40)`` and, when
    present, the KITTI 2015 training set for evaluation.  Returns (batches, eval_input)."""
    if train_dataset not in ('kitti', 'kitti_ft'):
        raise SystemExit("dataset '%s': kitti_inputs serves kitti and kitti_ft (dataset_inputs dispatches "
                         "the others)" % train_dataset)
    from .e2eflow.kitti.data import KITTIData
    from .e2eflow.kitti.input import KITTIInput
    if train_dataset == 'kitti_ft':
        kdata = KITTIData(dirs['data'], development=run_config.get('development', True),
                          fast_dir=dirs.get('fast'), require=('data_scene_flow', 'data_stereo_flow'))
        kinput = KITTIInput(data=kdata, batch_size=gpu_batch_size, normalize=False,
                            dims=(params['height'], params['width']), num_threads=run_config.get('num_input_threads', 1))
        # batch k of the stream is fixed (file order and crop seeds), and iteration i of rank r trains on
        # batch (i - 1) * world + r: a resumed run continues with the batches the interrupted one had
        # not reached (the reference's queue ignores the resume shift and starts over)
        batches = kinput.input_train_gt(FT_HOLD_OUT, rank=(start_iter - 1) * world + rank, world_size=world)
        eval_input = None
        if os.path.isdir(os.path.join(kdata.current_dir, 'data_scene_flow', 'training', 'flow_occ')):
            eval_input = KITTIInput(data=kdata, batch_size=1, normalize=False, dims=(384, 1280))
        return batches, eval_input
    kdata = KITTIData(dirs['data'], development=run_config.get('development', True),
                      fast_dir=dirs.get('fast'))
    kinput = KITTIInput(data=kdata, batch_size=gpu_batch_size, normalize=False, skipped_frames=True,
                        dims=(params['height'], params['width']), num_threads=run_config.get('num_input_threads', 1))
    batches = kinput.input_raw(swap_images=False, center_crop=True,
                               shift=(start_iter - 1) * run_config['batch_size'],
                               rank=rank, world_size=world)
    eval_input = None
    if os.path.isdir(os.path.join(kdata.current_dir, 'data_stereo_flow', 'training', 'flow_occ')):
        eval_input = KITTIInput(data=kdata, batch_size=1, normalize=False, dims=(384, 1280))
    return batches, eval_input


def dataset_inputs(dirs, run_config, params, train_dataset, gpu_batch_size, start_iter, rank, world):
    """The dataset branches of the reference run.py (:62-202): training batches of ``train_dataset``
    and the KITTI 2012 training set (at 384x1280) the run evaluates on after every chunk, or None when
    that set is not under [dirs] data.  kitti / kitti_ft: ``kitti_inputs``.

    * chairs: ``ChairsInput.input_raw(swap_images=False, shift=...)`` -- unrelated 384x512 pairs, no crop;
    * synthia: ``KITTIInput(SynthiaData).input_raw(swap_images=False, shift=...)`` -- consecutive frames of
      every sequence / view, random crop, no ``skipped_frames``;
    * cityscapes: ``KITTIInput(CityscapesData, skipped_frames=False).input_raw(swap_images=False,
      center_crop=True, skip=[0, 1], shift=...)`` -- ``center_crop`` is a no-op in the reference, which
      random-crops, and the pairs that span two snippets of a city directory are kept, as there.

    ``shift`` is the reference's resume shift (iterations done x [run] batch_size); each rank reads its
    own shard of the batch stream; [run] num_input_threads threads decode ahead of it."""
    if train_dataset in ('kitti', 'kitti_ft'):
        return kitti_inputs(dirs, run_config, params, train_dataset, gpu_batch_size, start_iter, rank, world)
    from .e2eflow.kitti.input import KITTIInput
    kw = dict(batch_size=gpu_batch_size, normalize=False, dims=(params['height'], params['width']),
              num_threads=run_config.get('num_input_threads', 1))
    data_kw = dict(development=run_config.get('development', True), fast_dir=dirs.get('fast'))
    stream = dict(swap_images=False, shift=(start_iter - 1) * run_config['batch_size'], rank=rank, world_size=world)
    if train_dataset == 'chairs':
        from .e2eflow.chairs.data import ChairsData
        from .e2eflow.chairs.input import ChairsInput
        batches = ChairsInput(ChairsData(dirs['data'], **data_kw), **kw).input_raw(**stream)
    elif train_dataset == 'synthia':
        from .e2eflow.synthia.data import SynthiaData
        batches = KITTIInput(SynthiaData(dirs['data'], **data_kw), **kw).input_raw(**stream)
    elif train_dataset == 'cityscapes':
        from .e2eflow.cityscapes.data import CityscapesData
        batches = KITTIInput(CityscapesData(dirs['data'], **data_kw), skipped_frames=False,
                             **kw).input_raw(center_crop=True, skip=[0, 1], **stream)
    else:
        raise SystemExit("dataset '%s': must be one of synthia, kitti, kitti_ft, cityscapes, chairs"
                         % train_dataset)
    from .e2eflow.kitti.data import KITTIData
    kdata = KITTIData(dirs['data'], fast_dir=dirs.get('fast'), require=())
    eval_input = None
    if os.path.isdir(os.path.join(kdata.current_dir, 'data_stereo_flow', 'training', 'flow_occ')):
        eval_input = KITTIInput(data=kdata, batch_size=1, normalize=False, dims=(384, 1280))
    return batches, eval_input


def stage_datasets(data_dir, fast_dir, train_dataset, local_rank=0):
    """[dirs] fast (core/data.py:27-36, run.py:53-56): the directories of the KITTI adapter, which the
    reference builds with ``fast_dir`` whatever it trains on, and of ``train_dataset``'s adapter, copied
    from ``data_dir`` into ``fast_dir`` where they are missing there (``data.stage``).  A FlyingChairs
    release is converted in ``data_dir`` first, so the converted tree is what is copied.  Only local
    rank 0 copies (the node's ranks share its disk); on other ranks this does nothing.  Returns the
    directories copied."""
    if local_rank != 0:
        return []
    from .e2eflow.core.data import stage
    from .e2eflow.kitti.data import KITTIData
    dirs = list(KITTIData.dirs)
    if train_dataset == 'chairs':
        from .e2eflow.chairs.data import ChairsData, convert_if_release
        if not os.path.isdir(os.path.join(fast_dir, 'flying_chairs')):
            convert_if_release(os.path.join(data_dir, 'flying_chairs'))
        dirs += ChairsData.dirs
    elif train_dataset == 'synthia':
        from .e2eflow.synthia.data import SynthiaData
        dirs += SynthiaData.dirs
    elif train_dataset == 'cityscapes':
        from .e2eflow.cityscapes.data import CityscapesData
        dirs += CityscapesData.dirs
    return stage(data_dir, fast_dir, dirs)


def evaluate_kitti(trainer, eval_input, device, hold_out_inv=None, dataset='2012', loss_averages=None,
                   pages=None):
    """train.py:265-385 on ``einput.input_train_2012()`` (``dataset='2012'``) or
    ``einput.input_train_2015()`` (``'2015'``): every pair is brought back to its file size (the
    queue pads to 384x1280), resized bilinearly to 384x1280 for the network, and the flow is resized
    back before AEE / outlier-% against the occluded and non-occluded ground truth.  ``loss_averages``:
    a dict that receives the tracked losses averaged over the pairs, ``pages`` a ``pages.Tiles`` that
    receives their visualisation tiles (core/train.py: evaluate)."""
    from .e2eflow.core.input import resize_image_with_crop_or_pad
    from .e2eflow.core.train import evaluate
    source = {'2012': eval_input.input_train_2012, '2015': eval_input.input_train_2015}[dataset]

    def examples():
        for item in source(hold_out_inv):
            h, w = int(item[2][0, 0]), int(item[2][0, 1])
            yield tuple(resize_image_with_crop_or_pad(t[0], h, w).unsqueeze(0).to(device)
                        for t in (item[0], item[1]) + item[3:])

    result, _ = evaluate(trainer.variables, trainer.params, trainer.normalization, examples(),
                         loss_averages=loss_averages, pages=pages)
    return result


def interactive_plot(run_config):
    """[run] interactive_plot (train.py:378-384): write the pages of every in-training evaluation.  Off
    when the key is absent or False."""
    return bool(run_config.get('interactive_plot', False))


def summary_writers(log_dir, name, rank, overwrite=False):
    """The train and eval event-file writers of experiment ``name`` (experiment.py:14-25), on rank 0
    only (None, None elsewhere).  ``overwrite`` (``--ow``) removes the earlier runs' files first."""
    if rank != 0:
        return None, None
    from .e2eflow.core.summary import SummaryWriter
    dirs = [os.path.join(log_dir, 'ex', name, d) for d in ('train', 'eval')]
    if overwrite:
        for d in dirs:
            if os.path.isdir(d):
                shutil.rmtree(d)
    return tuple(SummaryWriter(d) for d in dirs)


def write_train_summaries(writer, trainer, step, lr, images=False):
    """train.py:253-255 at a display step: the learning rate, the tracked losses (one device-to-host
    copy) and the weights under the reference's tags; with ``images`` the tracked images too."""
    from .e2eflow.core import summary
    from .e2eflow.core.train import read_scalars
    losses, params, tracked_images = trainer.tracked()
    tags = summary.train_tags(losses, params, tracked_images if images else ())
    writer.scalar(tags['learning_rate']['learning_rate'], lr, step)
    for kind, values in (('losses', read_scalars(losses)), ('params', params)):
        for name, value in values.items():
            writer.scalar(tags[kind][name], value, step)
    if images:
        for name, (t, to_image) in tracked_images.items():
            writer.image(tags['images'][name], to_image(t) if to_image is not None else t, step)
    writer.flush()


def write_eval_summaries(writer, step, result, loss_averages):
    """train.py:365-370: the evaluation averages under the reference's eval tags."""
    from .e2eflow.core import summary
    tags = summary.eval_tags(loss_averages)
    for name in summary.EVAL_METRICS:
        writer.scalar(tags[name], result[name], step)
    for name, value in loss_averages.items():
        writer.scalar(tags[summary.strip_tower(name)], value, step)
    writer.flush()


def synthetic_batch(batch, height, width, step, rank, device, supervised=False):
    from . import synthetic
    seed = 1234 + 7919 * step + rank
    if supervised:
        return tuple(t.to(device) for t in synthetic.supervised_batch(batch, height, width, seed=seed))
    im1, im2, _ = synthetic.image_pair(batch, height, width, seed=seed)
    return im1.to(device), im2.to(device)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--ex', default='default', help='Name of the experiment.')
    ap.add_argument('--debug', action='store_true', help='disable checkpoint writing for debugging')
    ap.add_argument('--ow', action='store_true', help='overwrite a previous experiment of the same name')
    ap.add_argument('--config', default=os.environ.get('UNFLOW_CONFIG', '../config.ini'))
    ap.add_argument('--synthetic', action='store_true')
    ap.add_argument('--max-iters', type=int, default=None, help='stop early (for smoke runs)')
    ap.add_argument('--graph', action='store_true',
                    help='capture the training step in one CUDA graph (Trainer.capture) and replay it')
    ap.add_argument('--no-augment', action='store_true',
                    help='train without the random affine / photometric augmentation (the reference '
                         'always trains with it, train.py:160,169)')
    ap.add_argument('--ckpt-format', choices=('pt', 'tf'), default='pt',
                    help="'tf' writes TensorFlow checkpoints the reference can restore")
    args = ap.parse_args(argv)

    cfg = config_dict(args.config)
    dirs, run_config = cfg.get('dirs', {}), cfg['run']
    # before any network exists; importing flownet first applies UNFLOW_CONV_PRECISION, which the key overrides
    from .e2eflow.core import conv_ops, flownet
    precision = flownet.set_conv_precision(conv_precision(run_config, conv_ops.get_mode()))
    train_dataset = run_config.get('dataset', 'kitti')
    params = copy.deepcopy(cfg['train'])
    params.update(cfg.get('train_' + train_dataset, {}))
    convert_input_strings(params, dirs)

    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    local_rank = int(os.environ.get('LOCAL_RANK', '0'))
    if not torch.cuda.is_available():
        raise SystemExit("unflow_b200.run needs a CUDA device (no CPU fallback)")
    from . import launch
    gpu_ids = launch.resolve(run_config, torch.cuda.device_count())
    if gpu_ids is not None and len(gpu_ids) > 1:
        # the workers do all the work, rank 0 the experiment directories; this process creates no CUDA context
        code = launch.launch(sys.argv[1:] if argv is None else argv, gpu_ids)
        if code:
            raise SystemExit(code)
        return
    local = gpu_ids[0] if gpu_ids is not None else local_rank
    torch.cuda.set_device(local)
    device = torch.device('cuda', local)
    if world > 1:
        dist.init_process_group('nccl', device_id=device)
    assert run_config['batch_size'] % world == 0, 'batch_size must be divisible by the number of GPUs'
    gpu_batch_size = int(run_config['batch_size'] / world)

    log_dir = dirs.get('log', '../log')
    ckpt_dir = os.path.join(dirs.get('checkpoints', os.path.join(log_dir, 'checkpoints')), args.ex)
    ex_dir = os.path.join(log_dir, 'ex', args.ex)
    if rank == 0:
        if args.ow:
            if os.path.isdir(ckpt_dir):
                shutil.rmtree(ckpt_dir)
            remove_concluded(ex_dir)
        os.makedirs(ckpt_dir, exist_ok=True)
        # before the barrier below: every rank's latest_checkpoint then finds the restored checkpoint
        restore_concluded(ckpt_dir, ex_dir)
        # experiment.py (Experiment.__init__): the run's config is kept in log/ex/<name>/config.ini -- where
        # eval.py (eval_gui.py:97-116) looks for the parameters a checkpoint was trained with
        if not args.debug and os.path.isfile(args.config):
            os.makedirs(ex_dir, exist_ok=True)
            if args.ow or not os.path.isfile(os.path.join(ex_dir, 'config.ini')):
                shutil.copyfile(args.config, os.path.join(ex_dir, 'config.ini'))
    # before any step: without the tensorboard package the run stops here
    train_writer, eval_writer = summary_writers(log_dir, args.ex, rank, overwrite=args.ow)
    if world > 1:
        dist.barrier()

    from .e2eflow.core.train import Trainer, learning_rate_at
    supervised = train_dataset == 'kitti_ft'
    tr = Trainer(params, KITTI_NORMALIZATION, device, seed=1234, augment=not args.no_augment,
                 supervised=supervised)
    tr.track_images = args.debug and train_writer is not None      # train.py:156
    if tr.augment:
        from .e2eflow.core import augment as _augment
        _augment.seed(4321 + rank)      # towers / ranks differ in their augmentation draws (train.py:169)

    num_iters = params.get('num_iters', 0)
    if args.max_iters is not None:
        num_iters = min(num_iters, args.max_iters)
    save_interval = min(params['save_interval'], max(num_iters, 1))
    start_iter = 1
    ck = latest_checkpoint(ckpt_dir)
    external = external_restores(params, ck is not None)
    if ck is not None:
        # continue training
        restore_checkpoint(tr, ck[1], with_optimizer=True)
        tr.iteration = ck[0]
        start_iter = ck[0] + 1
    for i, source in enumerate(external):
        if rank == 0:
            print('-- restore', 'network %d' % i, source[1])
        restore_checkpoint(tr, source[1], nets=[i])
    if start_iter > num_iters:
        print('-- train: max_iter reached')
        if rank == 0 and not args.debug:      # run.py:204-205 concludes after tr.run however it returned
            conclude(ckpt_dir, ex_dir)
        for w in (train_writer, eval_writer):
            if w is not None:
                w.close()
        return
    tr.broadcast_variables(0)
    if rank == 0:
        print('-- training from i = {} to {}'.format(start_iter, num_iters))
    print('-- rank {}: conv precision {}'.format(rank, precision))

    # rank 0 writes the pages of each evaluation on a background thread; the next evaluation and the end of
    # the run wait for it and raise its error
    plots = None
    if rank == 0 and interactive_plot(run_config):
        from .e2eflow.core import pages
        plots = pages.PageWriter()
    batches, eval_input = None, None
    data_dir = dirs.get('data', '')
    if not args.synthetic and os.path.isdir(data_dir):
        if dirs.get('fast'):
            # copying a dataset can outlast NCCL's collective timeout: the ranks wait for the copies on a gloo
            # group that allows for it
            group = dist.new_group(backend='gloo', timeout=STAGING_TIMEOUT) if world > 1 else None
            stage_datasets(data_dir, dirs['fast'], train_dataset, local_rank)
            if group is not None:
                dist.barrier(group=group)
        batches, eval_input = dataset_inputs(dirs, run_config, params, train_dataset, gpu_batch_size,
                                             start_iter, rank, world)
    # the decode pool is stopped however the loop ends (an error, Ctrl-C): its queued reads are cancelled
    try:
        for i in range(start_iter, num_iters + 1):
            if batches is None:
                batch = synthetic_batch(gpu_batch_size, params['height'], params['width'], i, rank, device,
                                        supervised=supervised)
            else:
                batch = tuple(t.to(device, non_blocking=True) for t in next(batches))
            if args.graph and tr._graph is None:
                tr.capture(*batch)       # leaves parameters, moments and the iteration counter untouched
            loss = tr.step(*batch)       # LR schedule inside (train.py:225-244)
            if rank == 0 and (i == 1 or i % params['display_interval'] == 0):
                print("-- train: i = {}, loss = {}".format(i, float(loss)))
                write_train_summaries(train_writer, tr, i, learning_rate_at(i - 1, params),
                                      images=tr.track_images)
            if i % save_interval == 0:
                if not args.debug and rank == 0:
                    save_checkpoint(tr, ckpt_dir, i, args.ckpt_format)
                if eval_input is not None and rank == 0:      # Trainer.run: self.eval(1) after every chunk
                    loss_averages, tiles = {}, None
                    if plots is not None:
                        plots.join()
                        tiles = pages.Tiles()
                    if supervised:      # the 2015 pairs input_train_gt held out
                        result = evaluate_kitti(tr, eval_input, device, FT_HOLD_OUT, dataset='2015',
                                                loss_averages=loss_averages, pages=tiles)
                    else:
                        result = evaluate_kitti(tr, eval_input, device, params.get('eval_hold_out_inv'),
                                                loss_averages=loss_averages, pages=tiles)
                    print("-- eval: i = {}".format(i))
                    for k in sorted(result):
                        print("   {} = {}".format(k, result[k]))
                    write_eval_summaries(eval_writer, i, result, loss_averages)
                    if plots is not None:       # the previous evaluation's pages are replaced (train.py:379-380)
                        title = "{} (i={})".format(args.ex, i)
                        plots.start(os.path.join(ex_dir, 'eval_pages'), lambda _, t=title: t, [args.ex], [tiles])
                if world > 1:
                    # rank 0 alone writes the checkpoint and evaluates: the others wait here instead of inside the
                    # next step's all-reduce (where the wait would run into the NCCL watchdog and count as step time)
                    dist.barrier()
    finally:
        if batches is not None:
            batches.close()
        if plots is not None:
            plots.join()
    if rank == 0 and not args.debug:      # after the last chunk's barrier; the other ranks need not wait
        conclude(ckpt_dir, ex_dir)
    for w in (train_writer, eval_writer):
        if w is not None:
            w.close()
    if world > 1:
        if args.graph:
            # ncclCommDestroy was observed to hang for minutes when the communicator had been used
            # inside a captured CUDA graph (bench.py:_finish): leave once every rank is done
            torch.cuda.synchronize()
            dist.barrier()
            sys.stdout.flush()
            sys.stderr.flush()
            os._exit(0)
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
