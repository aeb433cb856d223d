"""Dataset directories (reference src/e2eflow/core/data.py).

The reference's ``Data`` downloads and unpacks a dataset whose directory is missing; here nothing is
ever fetched: a missing directory is a ``FileNotFoundError`` naming the layout the adapter expects.
``fast_dir``, when given, is read instead of ``data_dir`` (the reference copies the dataset there
first; here it must already be in place)."""
import os


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
