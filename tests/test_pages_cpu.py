"""Evaluation pages (core/pages.py): the renderer, ``eval --output_pages --num_vis`` with a stub flow
estimator on the CPU, the slot sets per kind of ground truth, ``[run] interactive_plot`` parsing and the
background writer.  The warp of the brightness-error slot is the CPU oracle's here; the GPU tests run
the product's."""
import os

import numpy as np
import pytest
import torch

cv2 = pytest.importorskip("cv2")

from oracle.image_warp import image_warp as oracle_warp
from unflow_b200 import eval as E
from unflow_b200 import run as R
from unflow_b200.e2eflow.core import flow_io, pages

KITTI_SLOTS = ['overlay', 'brightness error', 'flow', 'flow error']
GT_SLOTS = ['overlay', 'brightness error', 'flow', 'gt']
TEST_SLOTS = ['first image', 'warp error', 'flow prediction']


def read_rgb(path):
    im = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    assert im is not None, path
    return im[:, :, ::-1]


def tile(page, row_labels, ncols, h, w, r, c):
    y, x = pages.layout('', row_labels, ncols, h, w)[2][r][c]      # the title only widens the page
    return page[y:y + h, x:x + w]


# ---- renderer ----------------------------------------------------------------------------------------
def test_render_places_tiles_under_labels_and_headers():
    rng = np.random.default_rng(1)
    rows, cols, (h, w) = ['overlay', 'a much longer slot name'], ['expA', 'expB', 'expC'], (30, 50)
    grid = [[rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for _ in cols] for _ in rows]
    grid[1][2] = np.where(rng.random((h, w, 1)) < 0.5, 0, 255).astype(np.uint8)    # a binary mask
    page = pages.render('title', rows, cols, grid)
    gh, gw, origins = pages.layout('title', rows, len(cols), h, w)
    assert page.dtype == np.uint8 and page.shape == (gh, gw, 3)
    for r in range(len(rows)):
        for c in range(len(cols)):
            want = np.broadcast_to(grid[r][c], (h, w, 3))
            assert np.array_equal(tile(page, rows, len(cols), h, w, r, c), want), (r, c)
    # the gray tile: 0 is black, 1 (255) white, on all three channels
    t = tile(page, rows, len(cols), h, w, 1, 2)
    assert set(np.unique(t).tolist()) == {0, 255} and (t == t[:, :, :1]).all()
    top, left = origins[0][0]
    # separators: the background between tiles and around them
    assert (page[top - pages.SEP:top, left:] == pages.BACKGROUND).all()
    assert (page[:, left + w:left + w + pages.SEP] == pages.BACKGROUND).all()
    assert (page[top + h:top + h + pages.SEP, left:] == pages.BACKGROUND).all()
    # label strip: text in each row's band left of the tiles, wide enough for the longest label
    for r in range(len(rows)):
        y = origins[r][0][0]
        assert (page[y:y + h, :left] != pages.BACKGROUND).any(), r
    assert left > cv2.getTextSize(rows[1], cv2.FONT_HERSHEY_SIMPLEX, pages.FONT_SCALE, 1)[0][0]
    # a header over every column, and the title line above the headers
    line = top // 2
    for c in range(len(cols)):
        x = origins[0][c][1]
        assert (page[line:top, x:x + w] != pages.BACKGROUND).any(), c
    assert (page[:line] != pages.BACKGROUND).any()
    # the header names the column: a page with other experiment names differs only in the header band
    other = pages.render('title', rows, ['expA', 'expB', 'expX'], grid)
    differ = np.argwhere((other != page).any(2))
    assert len(differ) and differ[:, 0].min() >= line and differ[:, 0].max() < top
    assert differ[:, 1].min() >= origins[0][2][1]


def test_render_sizes_per_page_and_rejects_mixed_tiles(tmp_path):
    rows, cols = ['first image', 'warp error'], ['e']
    small = pages.render('t', rows, cols, [[np.zeros((20, 36, 3), np.uint8)], [np.zeros((20, 36, 1), np.uint8)]])
    large = pages.render('t', rows, cols, [[np.ones((40, 90, 3), np.uint8)], [np.ones((40, 90, 3), np.uint8)]])
    assert small.shape[:2] == pages.layout('t', rows, 1, 20, 36)[:2]
    assert large.shape[:2] == pages.layout('t', rows, 1, 40, 90)[:2]
    with pytest.raises(ValueError):
        pages.render('t', rows, cols, [[np.zeros((20, 36, 3), np.uint8)], [np.zeros((21, 36, 3), np.uint8)]])
    with pytest.raises(ValueError):
        pages.render('t', rows, ['e', 'f'], [[np.zeros((20, 36, 3), np.uint8)]] * 2)
    # a title wider than the grid widens the page; the tiles stay where they were
    title = 'a title much wider than one small tile'
    wide = pages.render(title, rows, cols, [[np.zeros((20, 36, 3), np.uint8)], [np.zeros((20, 36, 1), np.uint8)]])
    assert wide.shape[:2] == pages.layout(title, rows, 1, 20, 36)[:2]
    assert wide.shape[0] == small.shape[0] and wide.shape[1] > small.shape[1]
    assert pages.layout(title, rows, 1, 20, 36)[2] == pages.layout('t', rows, 1, 20, 36)[2]
    # written as RGB: cv2 reads it back in BGR
    page = np.zeros((8, 8, 3), np.uint8)
    page[..., 0] = 200
    pages.write(str(tmp_path / 'p.png'), page)
    assert np.array_equal(read_rgb(str(tmp_path / 'p.png')), page)


def test_to_uint8_clips_and_truncates_like_write_rgb_png(tmp_path):
    x = torch.tensor([-3.0, 0.0, 0.999, 1.0, 127.9, 254.99, 255.0, 300.0]).view(1, 1, 8, 1)
    got = pages.to_uint8(x)
    assert got.dtype == torch.uint8 and got.view(-1).tolist() == [0, 0, 0, 1, 127, 254, 255, 255]
    E.write_rgb_png(x.numpy(), str(tmp_path / 'x.png'))
    assert read_rgb(str(tmp_path / 'x.png'))[0, :, 0].tolist() == got.view(-1).tolist()
    assert pages.to_uint8(torch.tensor([[[[True], [False]]]]) * 255).view(-1).tolist() == [255, 0]


def test_tiles_copy_each_example_once_and_keep_uint8():
    t = pages.Tiles(limit=2)
    for k in range(2):
        assert t.wants_more()
        t.add(['rgb', 'mask'], [torch.full((1, 4, 5, 3), k, dtype=torch.uint8), torch.ones(1, 4, 5, 1, dtype=torch.uint8)])
    assert not t.wants_more() and t.names == ['rgb', 'mask']
    assert [a.shape for a in t.examples[1]] == [(4, 5, 3), (4, 5, 1)]
    assert all(a.dtype == np.uint8 for ex in t.examples for a in ex) and (t.examples[1][0] == 1).all()
    assert pages.Tiles().wants_more() and not pages.Tiles(0).wants_more()


# ---- eval --output_pages ---------------------------------------------------------------------------
H, W = 20, 36


def _png(path, im):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    assert cv2.imwrite(path, im)


def _image(rng):
    return cv2.GaussianBlur(rng.integers(0, 255, (H, W, 3), dtype=np.uint8), (0, 0), 2)


@pytest.fixture
def trees(tmp_path):
    """KITTI 2012 training (5 pairs, 4-tensor ground truth), FlyingChairs validation (2 pairs, flow + mask)
    and Middlebury test (2 pairs, no ground truth), all at 20x36."""
    rng = np.random.default_rng(0)
    data = tmp_path / "data"
    j = os.path.join
    tr = j(str(data), "data_stereo_flow", "training")
    for i in range(5):
        im = _image(rng)
        _png(j(tr, "colored_0", "%06d_10.png" % i), im)
        _png(j(tr, "colored_0", "%06d_11.png" % i), np.roll(im, 2, axis=1))
        flow = np.zeros((H, W, 2), np.float32)
        flow[..., 0] = 2.0 + i
        noc = np.ones((H, W))
        noc[:, :18] = 0
        for sub, mask in (("flow_occ", np.ones((H, W))), ("flow_noc", noc)):
            os.makedirs(j(tr, sub), exist_ok=True)
            flow_io.write_kitti_flow(j(tr, sub, "%06d_10.png" % i), flow, mask)
    ch = j(str(data), "flying_chairs")
    os.makedirs(j(ch, "image"))
    for i in range(2):
        _png(j(ch, "test_image", "%05d_img1.png" % i), _image(rng))
        _png(j(ch, "test_image", "%05d_img2.png" % i), _image(rng))
        os.makedirs(j(ch, "flow"), exist_ok=True)
        flow_io.write_flo(j(ch, "flow", "%05d_flow.flo" % i), rng.normal(0, 2, (H, W, 2)).astype(np.float32))
    for k in range(3):
        _png(j(str(data), "middlebury", "eval-data", "Army", "frame%02d.png" % (10 + k)), _image(rng))
    return tmp_path


STUB_FLOWS = {'a': (2.0, 0.0), 'b': (0.0, -2.0)}      # px at file size: different colours and errors


def _config(root):
    """The config, and experiments a and b with a checkpoint each and their own config, which names them."""
    from unflow_b200.e2eflow.core import tf_checkpoint as ck
    from unflow_b200.e2eflow.core.flownet import FlowNetVariables
    ini = root / "config.ini"
    text = ("[dirs]\nlog = %s/log\ncheckpoints = %s/ckpts\ndata = %s/data\n[run]\nbatch_size = 4\n"
            "[train]\nflownet = s\nternary_weight = 1.0\n" % (root, root, root))
    ini.write_text(text)
    for seed, name in enumerate(STUB_FLOWS):
        ck.save_variables(FlowNetVariables("s", False, seed=seed), str(root / "ckpts" / name / "model.ckpt-1"))
        (root / "log" / "ex" / name).mkdir(parents=True, exist_ok=True)
        (root / "log" / "ex" / name / "config.ini").write_text(text + "stub = %s\n" % name)
    return str(ini)


def stub_flow_fn(params, normalization, variables):
    """make_flow_fn for run_eval: experiment ``params['stub']`` estimates the constant flow of STUB_FLOWS."""
    u, v = STUB_FLOWS[params['stub']]

    def fn(im1, im2):
        fw = torch.zeros(im1.shape[:3] + (2,))
        fw[..., 0], fw[..., 1] = u * im1.shape[2] / W, v * im1.shape[1] / H
        return fw, -fw
    return fn


def run(root, argv, monkeypatch):
    monkeypatch.setattr("unflow_b200.e2eflow.core.image_warp.image_warp", oracle_warp)
    args = E.arg_parser().parse_args(argv + ["--config", _config(root), "--out", str(root / "out")])
    return E.run_eval(args, torch.device("cpu"), make_flow_fn=stub_flow_fn)


def test_pages_are_the_output_visual_tiles_per_experiment(trees, monkeypatch, capsys):
    res = run(trees, ["--ex", "a,b", "--num", "5", "--num_vis", "3", "--output_pages", "--output_visual"],
              monkeypatch)
    assert set(res) == {"a", "b"}
    out = trees / "out"
    assert sorted(os.listdir(out / "pages")) == ["%06d.png" % i for i in range(3)]
    for i in range(3):
        page = read_rgb(str(out / "pages" / ("%06d.png" % i)))
        assert page.shape[:2] == pages.layout("Flow eval: kitti/train_2012 %06d" % i, KITTI_SLOTS, 2, H, W)[:2]
        for c, name in enumerate(("a", "b")):
            for r, suffix in ((0, "_img"), (2, "_flow"), (3, "_err")):
                want = read_rgb(str(out / name / ("%06d%s.png" % (i, suffix))))
                assert np.array_equal(tile(page, KITTI_SLOTS, 2, H, W, r, c), want), (i, name, suffix)
        # the columns differ where the experiments' flows do
        assert not np.array_equal(tile(page, KITTI_SLOTS, 2, H, W, 2, 0), tile(page, KITTI_SLOTS, 2, H, W, 2, 1))
    # the brightness error |im1 - warp(im2, flow)|: a's flow is the 2 px shift between the frames, b's is not
    page = read_rgb(str(out / "pages" / "000000.png"))
    assert tile(page, KITTI_SLOTS, 2, H, W, 1, 0)[:, 4:W - 4].mean() < tile(page, KITTI_SLOTS, 2, H, W, 1, 1)[:, 4:W - 4].mean()
    # column order follows --ex
    run(trees, ["--ex", "b,a", "--num", "1", "--output_pages"], monkeypatch)
    swapped = read_rgb(str(out / "pages" / "000000.png"))
    assert sorted(os.listdir(out / "pages")) == ["000000.png"]         # the earlier pages are replaced
    assert np.array_equal(tile(swapped, KITTI_SLOTS, 2, H, W, 2, 0), tile(page, KITTI_SLOTS, 2, H, W, 2, 1))


def test_num_vis_minus_one_pages_every_example(trees, monkeypatch):
    run(trees, ["--ex", "a", "--num", "4", "--num_vis", "-1", "--output_pages"], monkeypatch)
    assert sorted(os.listdir(trees / "out" / "pages")) == ["%06d.png" % i for i in range(4)]
    run(trees, ["--ex", "a", "--num", "-1", "--num_vis", "-1", "--output_pages"], monkeypatch)
    assert len(os.listdir(trees / "out" / "pages")) == 5
    run(trees, ["--ex", "a", "--num", "-1", "--output_pages"], monkeypatch)       # default 100
    assert len(os.listdir(trees / "out" / "pages")) == 5


def _outputs(root):
    out = {}
    for name in ("a", "b"):
        d = root / "out" / name
        for f in sorted(os.listdir(d)):
            out[(name, f)] = (d / f).read_bytes()
    return out


def test_without_output_pages_outputs_are_unchanged(trees, monkeypatch, capsys):
    flags = ["--ex", "a,b", "--num", "3", "--output_benchmark", "--output_visual", "--output_backward"]
    with_pages = run(trees, flags + ["--output_pages", "--num_vis", "2"], monkeypatch)
    printed_with = capsys.readouterr().out
    files_with = _outputs(trees)
    assert os.path.isdir(trees / "out" / "pages")
    import shutil
    shutil.rmtree(trees / "out")
    without = run(trees, flags + ["--num_vis", "2"], monkeypatch)
    printed_without = capsys.readouterr().out
    assert not os.path.exists(trees / "out" / "pages")
    assert without == with_pages and printed_without == printed_with
    files_without = _outputs(trees)
    assert sorted(files_without) == sorted(files_with) and len(files_with) == 2 * (1 + 3 * 5)
    assert all(files_without[k] == files_with[k] for k in files_with)


@pytest.mark.parametrize("dataset,variant,slots,n", [("kitti", "train_2012", KITTI_SLOTS, 5),
                                                     ("chairs", "test", GT_SLOTS, 2),
                                                     ("mdb", "test", TEST_SLOTS, 2)])
def test_slot_sets_follow_the_ground_truth(trees, monkeypatch, dataset, variant, slots, n):
    run(trees, ["--dataset", dataset, "--variant", variant, "--ex", "a,b", "--num", "-1", "--output_pages"],
        monkeypatch)
    files = sorted(os.listdir(trees / "out" / "pages"))
    assert files == ["%06d.png" % i for i in range(n)]
    for f in files:
        page = read_rgb(str(trees / "out" / "pages" / f))
        assert page.shape[:2] == pages.layout("Flow eval: %s/%s %s" % (dataset, variant, f[:6]), slots, 2, H, W)[:2]
    # the collector sees the names in that order
    monkeypatch.setattr("unflow_b200.e2eflow.core.image_warp.image_warp", oracle_warp)
    data_input, input_fn = E.dataset_input(dataset, variant, str(trees / "data"))
    got = pages.Tiles(1)
    E.evaluate_examples("a", input_fn(), data_input.dims, lambda a, b: (torch.ones(a.shape[:3] + (2,)),) * 2,
                        torch.device("cpu"), num=-1, pages=got, log=open(os.devnull, "w"))
    assert got.names == slots and len(got.examples) == 1
    assert [t.shape for t in got.examples[0]] == [(H, W, 3)] * len(slots)


def test_output_pages_refuses_an_experiment_named_pages(trees, monkeypatch):
    with pytest.raises(SystemExit):
        run(trees, ["--ex", "pages", "--output_pages", "--output_benchmark"], monkeypatch)


def test_help_states_the_host_memory_and_num_vis():
    text = ' '.join(E.arg_parser().format_help().split())
    assert "--output_pages" in text and "num_vis x slots" in text and "No effect without --output_pages" in text


# ---- [run] interactive_plot and the background writer -----------------------------------------------
@pytest.mark.parametrize("line,want", [("", False), ("interactive_plot = True\n", True),
                                       ("interactive_plot = False\n", False)])
def test_interactive_plot_key(tmp_path, line, want):
    ini = tmp_path / "config.ini"
    ini.write_text("[run]\nbatch_size = 4\n" + line)
    assert R.interactive_plot(R.config_dict(str(ini))["run"]) is want


def _one_page_tiles(n):
    t = pages.Tiles()
    for k in range(n):
        t.add(['flow', 'occ'], [torch.full((1, 6, 8, 3), 40 * k, dtype=torch.uint8),
                                torch.zeros(1, 6, 8, 1, dtype=torch.uint8)])
    return t


def test_page_writer_replaces_the_previous_pages_and_raises_at_the_next_join(tmp_path):
    out = str(tmp_path / "ex" / "eval_pages")
    w = pages.PageWriter()
    w.start(out, lambda i: "ex (i=2)", ["ex"], [_one_page_tiles(3)])
    w.join()
    assert sorted(os.listdir(out)) == ["000000.png", "000001.png", "000002.png"]
    w.start(out, lambda i: "ex (i=4)", ["ex"], [_one_page_tiles(2)])
    w.join()
    assert sorted(os.listdir(out)) == ["000000.png", "000001.png"]
    assert not os.path.exists(out + ".partial")
    page = read_rgb(os.path.join(out, "000001.png"))
    want = pages.render("ex (i=4)", ['flow', 'occ'], ["ex"], [[t] for t in _one_page_tiles(2).examples[1]])
    assert np.array_equal(page, want)
    # a write that fails (the page directory's parent is a file) is raised on the joining thread, once
    blocker = tmp_path / "file"
    blocker.write_text("x")
    w.start(str(blocker / "eval_pages"), lambda i: "t", ["ex"], [_one_page_tiles(1)])
    with pytest.raises(OSError):
        w.join()
    w.join()
    # ... also when the next evaluation's start is what joins
    w.start(str(blocker / "eval_pages"), lambda i: "t", ["ex"], [_one_page_tiles(1)])
    with pytest.raises(OSError):
        w.start(out, lambda i: "t", ["ex"], [_one_page_tiles(1)])
    w.join()
