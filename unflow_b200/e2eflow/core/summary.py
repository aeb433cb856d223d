"""TensorBoard event files with the reference's summaries (src/e2eflow/core/train.py:66-86,193-213,
314-370), written through ``torch.utils.tensorboard`` -- no TensorFlow needed.

Tags.  The reference names a summary after the tracked op (``tf.identity(x, name=...)``,
unsupervised.py:18-24) with ``tower_N/`` removed.  ``tf.summary.scalar`` / ``tf.summary.image`` open a
name scope of that name, and TF makes a name scope unique against every op name already in the graph,
so the tag of a summary on the op ``loss2/ternary`` is ``loss2/ternary_1``; in the evaluation graph the
averaged value is fed through a placeholder of the same name first, which takes ``_1``, so the
evaluation tag is ``loss2/ternary_2``.  ``unique_name`` restates that rule (ops.py
``Graph.unique_name``); ``train_tags`` and ``eval_tags`` apply it in the order the reference creates
the ops.

Images.  ``image_uint8`` is the conversion of TF's ``ImageSummary`` kernel (summary_image_op.cc) for
float input, per image of the batch: over the pixels whose channels are all finite, if the minimum is
>= 0 scale by 255 / max (0 when max < 1e-6), else by 127 / max|x| (0 when that is < 1e-6) and add 128;
truncate to uint8; a pixel with a non-finite channel takes the bad colour (255, 0, 0).  At most
``max_outputs`` = 3 images, tagged ``<tag>/image/<i>``.  The conversion runs on the tensor's device;
only the uint8 result is copied to the host and PNG-encoded there (1 channel: grayscale PNG, 3: RGB).
"""
import io
import re

import torch

MAX_OUTPUTS = 3                   # tf.summary.image's default
_BAD_COLOR = (255, 0, 0, 255)     # ImageSummary's default bad_color
_ZERO_THRESHOLD = 1e-6


def unique_name(in_use, name):
    """TF 1.x ``Graph.unique_name``: ``name`` if unused, else ``name_<k>`` with the first free k;
    marks the result as used.  ``in_use``: {lower-case name: count}."""
    key = name.lower()
    i = in_use.get(key, 0)
    in_use[key] = i + 1
    if i == 0:
        return name
    base = key
    while key in in_use:
        key = '%s_%d' % (base, i)
        i += 1
    in_use[key] = 1
    return '%s_%d' % (name, i - 1)


def strip_tower(name):
    """train.py:71: the tower prefix of a multi-GPU graph is not part of the tag."""
    return re.sub('tower_[0-9]*/', '', name)


def train_tags(losses, params=(), images=()):
    """Summary tags of the training graph (train.py:68-86,193-202) as ``{kind: {op name: tag}}``.
    ``losses`` / ``params`` / ``images``: the op names of the 'losses', 'params' and 'train_images'
    collections in creation order.  ``learning_rate`` is the reference's own
    ``summarized_placeholder('learning_rate', 'train')`` under ``tf.name_scope('params')``."""
    in_use = {}
    for n in ('params/learning_rate',) + tuple(losses) + tuple(params) + tuple(images):
        unique_name(in_use, n)
    return {'learning_rate': {'learning_rate': unique_name(in_use, 'params/train/learning_rate')},
            'losses': {n: unique_name(in_use, strip_tower(n)) for n in losses},
            'params': {n: unique_name(in_use, strip_tower(n)) for n in params},
            'images': {n: unique_name(in_use, strip_tower(n)) for n in images}}


EVAL_METRICS = ('AEE/occluded', 'outliers/occluded', 'AEE/non-occluded', 'outliers/non-occluded')


def eval_tags(losses):
    """Summary tags of the evaluation graph (train.py:314-328): ``summarized_placeholder`` creates a
    placeholder named like the value, then the summary; ``{name: tag}`` for the four metrics and
    every tracked loss."""
    in_use = {}
    for n in losses:
        unique_name(in_use, n)
    out = {}
    for n in EVAL_METRICS + tuple(strip_tower(n) for n in losses):
        unique_name(in_use, n)                     # the placeholder
        out[n] = unique_name(in_use, n)            # tf.summary.scalar's name scope
    return out


def image_uint8(images, max_outputs=MAX_OUTPUTS):
    """[N,H,W,C] (C = 1 or 3) -> uint8 [min(N, max_outputs),H,W,C] with ImageSummary's float
    normalisation (module docstring), computed on the tensor's device."""
    x = images[:max_outputs].detach()
    if x.dim() != 4 or x.shape[-1] not in (1, 3):
        raise ValueError("image summary: [N,H,W,1|3] expected, got %s" % (tuple(x.shape),))
    if x.dtype == torch.uint8:
        return x
    x = x.float()
    n, c = x.shape[0], x.shape[-1]
    finite = torch.isfinite(x).all(dim=-1, keepdim=True)
    lo = torch.where(finite, x, float('inf')).reshape(n, -1).amin(dim=1)
    hi = torch.where(finite, x, float('-inf')).reshape(n, -1).amax(dim=1)
    negative = lo < 0
    max_abs = torch.maximum(lo.abs(), hi.abs())
    zero = torch.zeros_like(lo)
    scale = torch.where(negative, torch.where(max_abs < _ZERO_THRESHOLD, zero, 127.0 / max_abs),
                        torch.where(hi < _ZERO_THRESHOLD, zero, 255.0 / hi))
    offset = torch.where(negative, zero + 128.0, zero)
    y = x * scale.view(n, 1, 1, 1)
    y = (y + offset.view(n, 1, 1, 1)).clamp_(0, 255).to(torch.uint8)       # truncates, as Eigen's cast
    bad = torch.zeros(c, dtype=torch.uint8, device=x.device)
    for k in range(c):
        bad[k:k + 1].fill_(_BAD_COLOR[k])       # a fill kernel: indexed assignment would copy from the host
    return torch.where(finite, y, bad)


def _png(hwc):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(hwc[:, :, 0] if hwc.shape[2] == 1 else hwc, 'L' if hwc.shape[2] == 1 else 'RGB').save(buf, 'PNG')
    return buf.getvalue()


class SummaryWriter:
    """One event-file directory (a TensorBoard run)."""

    def __init__(self, logdir):
        try:
            from torch.utils.tensorboard import SummaryWriter as _Writer
            from tensorboard.compat.proto.summary_pb2 import Summary
        except ImportError as e:
            raise ImportError("writing TensorBoard summaries needs the tensorboard package: %s" % e) from e
        self._summary = Summary
        self._writer = _Writer(log_dir=logdir)
        self.logdir = logdir

    def scalar(self, tag, value, step):
        self._writer.add_scalar(tag, float(value), int(step))

    def image(self, tag, nhwc_batch, step):
        """``tf.summary.image(tag, nhwc_batch)``: the first three images as ``<tag>/image/<i>``."""
        batch = image_uint8(nhwc_batch).cpu().numpy()
        values = [self._summary.Value(tag='%s/image/%d' % (tag, i), image=self._summary.Image(
            height=im.shape[0], width=im.shape[1], colorspace=im.shape[2], encoded_image_string=_png(im)))
            for i, im in enumerate(batch)]
        self._writer._get_file_writer().add_summary(self._summary(value=values), int(step))

    def flush(self):
        self._writer.flush()

    def close(self):
        self._writer.close()
