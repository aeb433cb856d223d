"""Dataset directories (reference src/e2eflow/core/data.py).

The reference's ``Data`` downloads and unpacks a dataset whose directory is missing; here nothing is
ever fetched: a missing directory is a ``FileNotFoundError`` naming the layout the adapter expects.
``fast_dir``, when given, is read instead of ``data_dir``.  As the reference's ``Data.__init__``
(core/data.py:27-36) does, ``run`` first copies the adapter's ``dirs`` from ``data_dir`` into
``fast_dir`` where they are missing there (``stage``); staged copies are never removed."""
import os
import shutil


def stage(data_dir, fast_dir, dirs):
    """Copy every entry of ``dirs`` that is a directory under ``data_dir`` and missing under ``fast_dir``.
    A copy is made in ``<dst>.partial`` and renamed to ``<dst>`` once complete, so an interrupted copy
    is never taken for a dataset: the next call discards it and copies again.  Directories already
    under ``fast_dir`` are not touched.  Returns the entries copied."""
    copied = []
    for d in dirs:
        src, dst = os.path.join(data_dir, d), os.path.join(fast_dir, d)
        if os.path.isdir(dst) or not os.path.isdir(src):
            continue
        partial = dst + '.partial'
        if os.path.isdir(partial):
            shutil.rmtree(partial)
        print(">> Copying {} to {}".format(d, fast_dir))
        shutil.copytree(src, partial)
        os.rename(partial, dst)
        print(">> Copied {}".format(d))
        copied.append(d)
    return copied


class Data():
    layout = ''      # the expected directory layout, for the error message

    def __init__(self, data_dir, stat_log_dir=None, development=True, fast_dir=None):
        self.development = development
        self.data_dir = data_dir
        self.stat_log_dir = stat_log_dir
        self.fast_dir = fast_dir
        self.current_dir = fast_dir or data_dir
        self._check()

    def _check(self):
        """Raise ``FileNotFoundError`` unless the dataset is in place (subclasses)."""

    def _require(self, *rel):
        for r in rel:
            if not os.path.isdir(os.path.join(self.current_dir, r)):
                raise FileNotFoundError("%s not found under %s (expected layout: %s; datasets are not downloaded)"
                                        % (r, self.current_dir, self.layout))

    def get_raw_dirs(self):
        """Every directory of training frames (each one an ordered sequence or a list of pairs)."""
        raise NotImplementedError()

    def get_raw_files(self):
        return [os.path.join(d, p) for d in self.get_raw_dirs() for p in os.listdir(d)]
