"""Synthetic inputs shared by the parity tests (re-exported from the package)."""
from unflow_b200.synthetic import *  # noqa: F401,F403
from unflow_b200.synthetic import KITTI_NORMALIZATION, KITTI_PARAMS, image_pair, level_inputs  # noqa: F401


# ---- tests/golden/reference_run.npz ------------------------------------------------------------------
# The generator (tests/golden/make_reference_run.py) leaves out what is cheap to redraw -- the image pairs,
# from their seeds -- and keeps the full-resolution output flows of unsupervised_loss at a fixed sample of
# positions, so that the file stays small.
RUN_IMAGES = {'fn_c': (64, 128, 121, True), 'fn_s': (64, 64, 122, True), 'fn_cs': (64, 64, 123, True),
              'fn_sfull': (64, 64, 124, True), 'ul_c': (128, 128, 131, False), 'ul_s': (128, 128, 132, False),
              'ul_cs': (128, 128, 133, False)}      # tag: (H, W, seed, scaled to [-0.4, 0.6))
RUN_SAMPLE = 4096


def run_images(tag):
    import numpy as np
    H, W, seed, scaled = RUN_IMAGES[tag]
    i1, i2, _ = image_pair(1, H, W, seed=seed)
    if scaled:
        i1, i2 = i1 / 255.0 - 0.4, i2 / 255.0 - 0.4
    return np.ascontiguousarray(i1.numpy()), np.ascontiguousarray(i2.numpy())


class ReferenceRun:
    """The golden vectors by name; ``<tag>_im1`` / ``<tag>_im2`` of RUN_IMAGES are redrawn on demand."""

    def __init__(self, path):
        import numpy as np
        self.z = np.load(path)
        self.files = list(self.z.files) + ['%s_im%d' % (t, i) for t in RUN_IMAGES for i in (1, 2)]

    def __getitem__(self, key):
        tag, _, last = key.rpartition('_')
        if tag in RUN_IMAGES and last in ('im1', 'im2'):
            return run_images(tag)[int(last[-1]) - 1]
        return self.z[key]


def sampled_close(got, G, key, rtol, atol_rel):
    """``got`` (full tensor) against the sampled reference output ``key`` of ReferenceRun ``G``: the
    tolerance of numpy's assert_allclose at the stored positions, atol relative to max |reference|."""
    import numpy as np
    got = got.detach().cpu().numpy()
    assert got.shape == tuple(int(v) for v in G[key + '_shape']), key
    atol = atol_rel * max(float(G[key + '_absmax']), 1e-12)
    np.testing.assert_allclose(got.reshape(-1)[G[key + '_idx']], G[key + '_val'], rtol=rtol, atol=atol, err_msg=key)
