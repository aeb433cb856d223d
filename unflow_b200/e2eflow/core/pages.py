"""The pages of the reference's evaluation viewer (src/e2eflow/gui.py:8-86) as PNG files.

A page shows one evaluated example: a row per image slot, in the order the caller gives, and a column per
experiment, with the slot names in a strip on the left, the experiment's name over its column and a title
line on top.  ``eval.py --output_pages`` and ``run.py``'s ``[run] interactive_plot`` both lay out their
pages here.  Every pixel value comes from the functions the caller already ran on the device; this module
only converts them to uint8 there (``to_uint8``), copies each example to the host once (``Tiles``) and
places the tiles (``render``).  Text is drawn with OpenCV.
"""
import os
import shutil
import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

FONT_SCALE = 0.5
PAD = 6                 # space around a line of text
SEP = 2                 # separator between tiles, in the background colour
BACKGROUND = 128        # the grey of the reference's figure (gui.py:24, facecolor='grey')
PNG_COMPRESSION = 1     # zlib level 1: pages are large and written while training continues


def to_uint8(x):
    """``x`` (a device tensor of values in [0, 255]) as uint8 with the rule of ``eval.write_rgb_png``:
    clipped to [0, 255], then truncated.  Callers pass ``image * 255`` for images in [0, 1], so a
    single-channel mask of 0 / 1 becomes black / white."""
    return x.float().clamp(0, 255).to(torch.uint8)


class Tiles:
    """Host copies of the uint8 image slots of evaluated examples, in evaluation order; at most ``limit``
    examples (-1: all)."""

    def __init__(self, limit=-1):
        self.limit = limit
        self.names = None
        self.examples = []

    def wants_more(self):
        return self.limit < 0 or len(self.examples) < self.limit

    def add(self, names, tiles):
        """One example: ``tiles`` are uint8 device tensors ``[1,h,w,C]`` (``to_uint8``), C = 1 or 3,
        named by ``names``.  They are copied to the host with one device-to-host copy."""
        flat = torch.cat([t.reshape(-1) for t in tiles]).cpu().numpy()
        host, at = [], 0
        for t in tiles:
            host.append(flat[at:at + t.numel()].reshape(t.shape[1:]))
            at += t.numel()
        self.names = list(names)
        self.examples.append(host)


def _text_size(text):
    import cv2
    (w, h), baseline = cv2.getTextSize(text, cv2.FONT_HERSHEY_SIMPLEX, FONT_SCALE, 1)
    return w, h, baseline


def _line_height():
    _, h, baseline = _text_size("Ag")
    return h + baseline + 2 * PAD


def _put(page, text, x, y_baseline):
    import cv2
    cv2.putText(page, text, (int(x), int(y_baseline)), cv2.FONT_HERSHEY_SIMPLEX, FONT_SCALE, (0, 0, 0), 1,
                cv2.LINE_AA)


def _fit(text, width):
    """``text`` shortened from the end until it fits ``width`` pixels."""
    while len(text) > 1 and _text_size(text)[0] > width:
        text = text[:-1]
    return text


def layout(title, row_labels, ncols, h, w):
    """The geometry ``render`` gives a page of ``len(row_labels)`` x ``ncols`` tiles of h x w:
    ``(page height, page width, origins)``, ``origins[r][c]`` the (y, x) of tile (r, c).  A title wider
    than the grid widens the page to its right."""
    label_w = max(_text_size(t)[0] for t in row_labels) + 2 * PAD
    top = 2 * _line_height()        # title line, then the column headers
    origins = [[(top + SEP + r * (h + SEP), label_w + SEP + c * (w + SEP)) for c in range(ncols)]
               for r in range(len(row_labels))]
    width = max(label_w + SEP + ncols * (w + SEP), _text_size(title)[0] + 2 * PAD)
    return top + SEP + len(row_labels) * (h + SEP), width, origins


def render(title, row_labels, col_labels, tiles):
    """One page: ``tiles[row][col]`` uint8 arrays ``[h,w,3]`` (RGB) or ``[h,w,1]`` (gray), all of one
    size, ``row_labels`` the slot names, ``col_labels`` the experiment names.  Returns the RGB page."""
    h, w = tiles[0][0].shape[:2]
    if len(tiles) != len(row_labels) or any(len(row) != len(col_labels) for row in tiles):
        raise ValueError("pages: %d row labels and %d column labels for a %d-row grid"
                         % (len(row_labels), len(col_labels), len(tiles)))
    if any(t.shape[:2] != (h, w) or t.shape[2] not in (1, 3) for row in tiles for t in row):
        raise ValueError("pages: the tiles of a page must all be %dx%d with 1 or 3 channels" % (h, w))
    page_h, page_w, origins = layout(title, row_labels, len(col_labels), h, w)
    line = _line_height()
    page = np.full((page_h, page_w, 3), BACKGROUND, np.uint8)
    _put(page, title, PAD, line - PAD - _text_size(title)[2])
    for c, label in enumerate(col_labels):
        y, x = origins[0][c]
        _put(page, _fit(label, w), x, 2 * line - PAD - _text_size(label)[2])
    for r, label in enumerate(row_labels):
        y, _ = origins[r][0]
        _, th, _ = _text_size(label)
        _put(page, label, PAD, y + (h + th) // 2)
        for c in range(len(col_labels)):
            y, x = origins[r][c]
            page[y:y + h, x:x + w] = tiles[r][c]       # [h,w,1] broadcasts to gray
    return page


def write(path, page):
    import cv2
    if not cv2.imwrite(path, np.ascontiguousarray(page[:, :, ::-1]), [cv2.IMWRITE_PNG_COMPRESSION, PNG_COMPRESSION]):
        raise IOError("cannot write " + path)


def write_pages(out_dir, title, col_labels, columns, threads=1):
    """``out_dir/%06d.png``: page i shows example i of every ``Tiles`` in ``columns`` (one per column, the
    same slots) under ``title(i)``.  The pages are written into ``out_dir + '.partial'``, which then
    replaces ``out_dir``, so ``out_dir`` holds one complete set at any time but the moment of the swap.
    ``threads`` pages are rendered and encoded at once (OpenCV releases the GIL while it encodes)."""
    names = next((c.names for c in columns if c.names is not None), None)
    if any(c.names not in (None, names) for c in columns):
        raise ValueError("pages: the columns have different slots")
    tmp = out_dir + '.partial'
    if os.path.isdir(tmp):
        shutil.rmtree(tmp)
    os.makedirs(tmp)

    def page(i, example):
        grid = [[col[r] for col in example] for r in range(len(names))]
        write(os.path.join(tmp, '%06d.png' % i), render(title(i), names, col_labels, grid))
    examples = list(enumerate(zip(*(c.examples for c in columns))))
    if threads > 1:
        with ThreadPoolExecutor(threads) as pool:
            for done in [pool.submit(page, i, ex) for i, ex in examples]:
                done.result()
    else:
        for i, ex in examples:
            page(i, ex)
    if os.path.isdir(out_dir):
        shutil.rmtree(out_dir)
    os.rename(tmp, out_dir)


class PageWriter:
    """``write_pages`` on one background thread, one set of pages at a time.  ``start`` first waits for the
    previous set; ``join`` waits and raises, on the calling thread, the error the last write ended with."""

    def __init__(self):
        self._thread = None
        self._error = None

    def start(self, *args):
        self.join()

        def work():
            try:
                write_pages(*args)
            except BaseException as e:      # handed to the next join
                self._error = e
        self._thread = threading.Thread(target=work, name='unflow-pages')
        self._thread.start()

    def join(self):
        if self._thread is not None:
            self._thread.join()
            self._thread = None
        if self._error is not None:
            error, self._error = self._error, None
            raise error
