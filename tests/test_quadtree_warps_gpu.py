"""GPU parity of the quadtree distribution (one warp per (level, frame), candidates in shared memory when they fit, in global memory
otherwise) and of the orientation computed next to BRIEF: keypoints, octaves, angles, descriptors and counts of whole batches against
the CPU oracle, frame by frame, on the list shapes the distribution can take:

- a frame without a single FAST candidate (every level empty) next to textured frames in the same launch;
- a level with fewer candidates than nDesired, whose splitting stalls (no node splits, m == prevSize);
- periodic texture: equal responses and equal node sizes, so the careful phase's sort decides ties;
- levels with so few features wanted that the first split of the roots yields as many nodes as selCap;
- 1280x720 (two root nodes), and dense noise whose level-0 candidates do not fit in the warp's shared memory;
- batch sizes 1, 5 and 7, and one handle reused for a smaller image and then the larger one again."""
import numpy as np
import pytest

import oracle_lib as O
from orb_slam3_modified_b200 import synth
from test_extractor_paths_gpu import LAP, _check_all, _check_device, _frames

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def torch():
    import torch as t
    return t


def _flat(w, h):
    return np.full((h, w), 128, np.uint8)


def _sparse(w, h, k=12, seed=0):
    """A flat image with k bright 6x6 squares: a few dozen corners, fewer than any level asks for."""
    rng = np.random.default_rng(seed)
    img = _flat(w, h)
    for x, y in zip(rng.integers(40, w - 46, k), rng.integers(40, h - 46, k)):
        img[y:y + 6, x:x + 6] = 230
    return img


def _periodic(w, h, seed=0):
    rng = np.random.default_rng(seed)
    return np.tile(rng.integers(0, 256, (12, 12)).astype(np.uint8), (h // 12 + 1, w // 12 + 1))[:h, :w].copy()


def _noise(w, h, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (h, w)).astype(np.uint8)


def _per_level(oe, frame, nlevels):
    _, kps, _ = oe(frame, LAP)
    return np.bincount(kps['octave'], minlength=nlevels)


def _run(ex, oe, frames, tag):
    _check_all(ex, oe, frames, list(zip(*ex.extract_batch(frames, LAP))), LAP, tag)


def test_empty_sparse_and_tied_levels(orb, torch):
    w, h = 640, 480
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, w, h, 5)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    want = ex.features_per_level()
    frames = np.stack([_flat(w, h), _sparse(w, h), _periodic(w, h), synth.frame(3), _sparse(w, h, k=40, seed=1)])
    assert _per_level(oe, frames[0], 8).sum() == 0
    sparse = _per_level(oe, frames[1], 8)
    assert ((sparse > 0) & (sparse < want)).any(), (sparse, want)
    assert _per_level(oe, frames[2], 8).sum() > 500
    _run(ex, oe, frames, 'mixed B=5')
    _check_device(orb, torch, ex, oe, frames[::-1].copy(), 'packed', tag='mixed reversed')


def test_roots_fill_sel_cap(orb):
    """nfeatures = 12 at 1280x720: levels that want one or two keypoints stop after splitting their two roots, with up to 4 * nIni = 8
    nodes, which is selCap there."""
    w, h = 1280, 720
    ex = orb.ORBextractor(12, 1.2, 8, 20, 7, w, h, 3)
    oe = O.OracleExtractor(12, 1.2, 8, 20, 7)
    frames = _frames(3, w, h, t0=5)
    want = ex.features_per_level()
    counts = _per_level(oe, frames[0], 8)
    assert any(counts[l] == 8 and want[l] + 3 < 8 for l in range(8)), (counts, want)
    _run(ex, oe, frames, 'nfeatures 12')


@pytest.mark.parametrize('B', [1, 5, 7])
def test_batches_1280x720(orb, torch, B):
    w, h = 1280, 720
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, w, h, B)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    frames = _frames(B, w, h, t0=2 + B)
    if B > 1:
        frames[1] = _noise(w, h, seed=B)
    _run(ex, oe, frames, '1280x720 B=%d' % B)
    _check_device(orb, torch, ex, oe, frames, 'packed', tag='1280x720 B=%d' % B)


def test_handle_reused_after_larger_image(orb, torch):
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 1280, 720, 5)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    big = _frames(3, 1280, 720, t0=11)
    big[2] = _noise(1280, 720, seed=4)
    _run(ex, oe, big, 'first 1280x720')
    small = np.stack([_sparse(640, 480, seed=2), synth.frame(9), _noise(640, 480, seed=5), _periodic(640, 480, seed=3), _flat(640, 480)])
    _run(ex, oe, small, 'then 640x480')
    _check_device(orb, torch, ex, oe, small, 'padded', tag='then 640x480')
    _run(ex, oe, big[:2], '1280x720 again')
