"""FAST candidates of the block kernel (one CTA per 2 x 2 cells) against the CPU oracle's per-cell cv::FAST, level by level and frame
by frame of a batch, on geometries with partial blocks, clipped cells and a cell that falls back to minThFAST inside a block."""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu

INI_TH, MIN_TH = 20, 7


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def synth():
    from orb_slam3_modified_b200 import synth as s
    return s


def _check_batch(orb, images, frames, nlevels=8, scale=1.2):
    """Extract `images` in one batch call and compare every level's candidates of the listed frames with the oracle."""
    B, h, w = images.shape
    ex = orb.ORBextractor(1000, scale, nlevels, INI_TH, MIN_TH, w, h, B)
    oe = O.OracleExtractor(1000, scale, nlevels, INI_TH, MIN_TH)
    ex.extract_batch(images, (0, 1000))
    out = {}
    for f in frames:
        oe(images[f], (0, 1000))
        for l in range(nlevels):
            c = ex.candidates(l, f)
            oc = oe.candidates(l)
            ocx = np.stack([oc['x'], oc['y'], oc['response']], 1).astype(np.int32)
            assert c.shape == ocx.shape, ((w, h), 'frame', f, 'level', l, c.shape, ocx.shape)
            assert np.array_equal(c, ocx), ((w, h), 'frame', f, 'level', l, 'candidates differ')
            out[f, l] = ocx
    return out


def _level0_cells(w, h):
    """wCell, hCell of level 0 (reference src/ORBextractor.cc:789-803)."""
    width, height = w - 2 * 16, h - 2 * 16
    return int(np.ceil(width / int(width / 35))), int(np.ceil(height / int(height / 35)))


@pytest.mark.parametrize('w,h', [(640, 480), (1280, 720), (500, 375)])
def test_synthetic_batch1(orb, synth, w, h):
    _check_batch(orb, synth.frame(4, w, h)[None], [0])


def test_batch240_640x480(orb, synth):
    images = np.stack([synth.frame(t, 640, 480, seed=t % 3) for t in range(240)])
    _check_batch(orb, images, [0, 1, 117, 239])


def test_batch_720p_and_odd_sizes(orb, synth):
    _check_batch(orb, synth.frames(3, 1280, 720, t0=11), [0, 2])
    _check_batch(orb, synth.frames(3, 500, 375, t0=5), [0, 1, 2], nlevels=5, scale=1.5)


def test_flat_image(orb):
    c = _check_batch(orb, np.full((2, 480, 640), 77, np.uint8), [0, 1])
    assert all(len(v) == 0 for v in c.values())


def test_nms_stays_inside_cells_of_a_block(orb):
    """Dense corners: the oracle keeps pairs of adjacent corners on either side of a cell border inside a block.  They survive only
    if the neighbour across the border counts as 0 in NMS, so a kernel whose NMS leaks across the border loses one of each pair."""
    rng = np.random.default_rng(11)
    images = rng.integers(0, 256, (2, 480, 640)).astype(np.uint8)
    c = _check_batch(orb, images, [0, 1])
    wc, hc = _level0_cells(640, 480)
    pts = c[0, 0]
    keys = set(map(tuple, pts[:, :2].tolist()))
    # cand x = interior column + 3 + j * wCell: the border between block columns 0 and 1 lies between x = wCell + 2 and wCell + 3
    across_x = sum((wc + 2, y) in keys and (wc + 3, yy) in keys for (x, y) in keys if x == wc + 2 for yy in (y - 1, y, y + 1))
    across_y = sum((x, hc + 2) in keys and (xx, hc + 3) in keys for (x, y) in keys if y == hc + 2 for xx in (x - 1, x, x + 1))
    assert across_x > 0 and across_y > 0, (across_x, across_y)


def test_one_cell_of_a_block_falls_back_to_min_threshold(orb):
    """Isolated dots of contrast 15 (FAST score 14: minThFAST corners only) in the first cell of level 0, high contrast in the other
    three cells of its 2 x 2 block: the first cell falls back to minThFAST while its block neighbours keep iniThFAST corners only."""
    rng = np.random.default_rng(5)
    img = np.full((480, 640), 128, np.uint8)
    img[25:50:10, 25:50:10] = 143
    wc, hc = _level0_cells(640, 480)
    # level-0 pixel X belongs to the cell interior column X - 16 - 3; the first cell's ring reaches 3 px past its interior
    x1, y1 = 16 + 3 + wc + 3, 16 + 3 + hc + 3
    hi = rng.integers(0, 256, (480, 640)).astype(np.uint8)
    mask = np.zeros((480, 640), bool)
    mask[16:16 + 2 * hc + 6, x1:16 + 2 * wc + 6] = True
    mask[y1:16 + 2 * hc + 6, 16:16 + 2 * wc + 6] = True
    img[mask] = hi[mask]
    c = _check_batch(orb, img[None], [0])[0, 0]
    first = c[(c[:, 0] < wc + 3) & (c[:, 1] < hc + 3)]
    right = c[(c[:, 0] >= wc + 3) & (c[:, 0] < 2 * wc + 3) & (c[:, 1] < hc + 3)]
    below = c[(c[:, 0] < wc + 3) & (c[:, 1] >= hc + 3) & (c[:, 1] < 2 * hc + 3)]
    assert len(first) > 0 and first[:, 2].max() < INI_TH, first
    assert len(right) > 0 and right[:, 2].min() >= INI_TH
    assert len(below) > 0 and below[:, 2].min() >= INI_TH
