"""GPU parity tests of the extractor: CUDA path (through the C-ABI) vs the CPU oracle, bit-exact."""
import numpy as np
import pytest

import oracle_lib as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def synth():
    from orb_slam3_modified_b200 import synth as s
    return s


def _compare(ex, oe, img, lap, tag=''):
    return _check_frame(ex, 0, ex(img, lap), oe, oe(img, lap), tag)


def _check_frame(ex, f, result, oe, oresult, tag=''):
    """Frame `f` of `ex`'s last call, whose (mono, kps, desc) is `result`, against the oracle's last call on the same image."""
    mono, kps, desc = result
    omono, okps, odesc = oresult
    # stage taps first: they localise a failure
    for l in range(ex.nlevels):
        lv, olv = ex.level(l, f), oe.level(l)
        assert lv.shape == olv.shape, (tag, 'level shape', l)
        assert np.array_equal(lv, olv), (tag, 'pyramid level differs', l, int((lv != olv).sum()))
        bl, obl = ex.level(l, f, blurred=True), O.blur7(olv)
        assert np.array_equal(bl, obl), (tag, 'blurred level differs', l, int((bl != obl).sum()))
    for l in range(ex.nlevels):
        c = ex.candidates(l, f)
        oc = oe.candidates(l)
        ocx = np.stack([oc['x'], oc['y'], oc['response']], 1).astype(np.int32)
        assert c.shape == ocx.shape, (tag, 'candidate count', l, c.shape, ocx.shape)
        assert np.array_equal(c, ocx), (tag, 'candidates differ', l)
    assert len(kps) == len(okps), (tag, len(kps), len(okps))
    assert mono == omono, (tag, mono, omono)
    for name in ('octave', 'x', 'y', 'response', 'size', 'angle', 'class_id'):
        assert np.array_equal(kps[name], okps[name]), (tag, 'keypoint field differs', name,
                                                        int((kps[name] != okps[name]).sum()))
    assert kps.tobytes() == okps.tobytes()
    bad = np.nonzero((desc != odesc).any(1))[0]
    assert len(bad) == 0, (tag, 'descriptor rows differ', len(bad), bad[:8])
    return len(kps)


def test_single_frame_config1(orb, synth):
    """BASELINE config 1: one 640x480 frame, nFeatures=1000, 8 levels, 1.2; mono lapping area {0,1000}."""
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 1)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    n = _compare(ex, oe, synth.frame(0), (0, 1000), 'cfg1')
    assert n >= 1000


@pytest.mark.parametrize('t', [3, 17, 40])
def test_more_frames(orb, synth, t):
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 1)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    _compare(ex, oe, synth.frame(t, seed=t % 3), (0, 1000), 'frame%d' % t)


def test_720p_lapping_split(orb, synth):
    """1280x720: keypoints with x > 1000 go to the front (monoIndex > 0), the rest fill from the back."""
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 1280, 720, 1)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    img = synth.frame(5, 1280, 720)
    _compare(ex, oe, img, (0, 1000), '720p')
    mono, _, _ = ex(img, (0, 1000))
    assert mono > 0
    _compare(ex, oe, img, (0, 0), '720p-nolap')


def test_noise_and_flat_images(orb):
    """Dense-corner (uniform noise) and corner-free (flat / gradient) inputs; the latter exercises the
    minThFAST fallback and empty levels."""
    rng = np.random.default_rng(7)
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 1)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    _compare(ex, oe, rng.integers(0, 256, (480, 640)).astype(np.uint8), (0, 1000), 'noise')
    flat = np.full((480, 640), 77, np.uint8)
    mono, kps, desc = ex(flat, (0, 1000))
    assert len(kps) == 0 and mono == 0
    grad = (np.add.outer(np.arange(480), np.arange(640)) // 5).astype(np.uint8)
    _compare(ex, oe, grad, (0, 1000), 'gradient')
    lowc = (128 + rng.integers(-6, 7, (480, 640))).astype(np.uint8)   # only minTh corners
    _compare(ex, oe, lowc, (0, 1000), 'lowcontrast')


def test_other_configs(orb, synth):
    """Init extractor (5x features), portrait phone rig 600x800 (nIni=1), odd sizes, strided input."""
    for (nf, sf, nl, w, h) in [(5000, 1.2, 8, 640, 480), (1500, 1.2, 8, 600, 800), (800, 1.5, 5, 517, 389), (1200, 2.0, 3, 640, 480),
                               (2000, 1.2, 8, 1241, 376)]:
        ex = orb.ORBextractor(nf, sf, nl, 20, 7, w, h, 1)
        oe = O.OracleExtractor(nf, sf, nl, 20, 7)
        _compare(ex, oe, synth.frame(2, w, h), (0, 1000), 'cfg %s' % ((nf, sf, nl, w, h),))
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 1)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    big = synth.frame(9, 700, 500)
    view = big[10:490, 30:670]   # non-contiguous rows: step != cols
    mono, kps, desc = ex(view, (0, 1000))
    omono, okps, odesc = oe(np.ascontiguousarray(view), (0, 1000))
    assert kps.tobytes() == okps.tobytes() and np.array_equal(desc, odesc) and mono == omono


def test_empty_and_errors(orb):
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 1)
    mono, kps, desc = ex(np.zeros((0, 0), np.uint8))
    assert mono == -1 and len(kps) == 0     # reference returns -1 on an empty image (ORBextractor.cc:1090)
    with pytest.raises(orb.OrbError):
        ex(np.zeros((481, 640), np.uint8))  # larger than configured
    with pytest.raises(orb.OrbError):
        orb.ORBextractor(1000, 1.2, 8, 20, 7, 200, 800, 1)   # aspect < 0.5 -> reference divides by zero


def test_batch_matches_single(orb, synth):
    """Batched call == per-frame calls (frames are independent units)."""
    B = 6
    imgs = synth.frames(B, t0=20)
    exb = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, B)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    monos, kps, descs = exb.extract_batch(imgs, (0, 1000))
    for b in range(B):
        omono, okps, odesc = oe(imgs[b], (0, 1000))
        assert monos[b] == omono and kps[b].tobytes() == okps.tobytes() and np.array_equal(descs[b], odesc), b


def test_determinism(orb, synth):
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 1)
    img = synth.frame(11)
    a = ex(img, (0, 1000))
    for _ in range(5):
        b = ex(img, (0, 1000))
        assert a[0] == b[0] and a[1].tobytes() == b[1].tobytes() and np.array_equal(a[2], b[2])


def test_tables(orb):
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 1)
    t = O.OracleExtractor(1000, 1.2, 8, 20, 7).tables()
    assert np.array_equal(ex.GetScaleFactors(), t['scale'])
    assert np.array_equal(ex.GetInverseScaleFactors(), t['inv_scale'])
    assert np.array_equal(ex.GetScaleSigmaSquares(), t['sigma2'])
    assert np.array_equal(ex.GetInverseScaleSigmaSquares(), t['inv_sigma2'])
    assert list(ex.features_per_level()) == [217, 181, 151, 126, 105, 87, 73, 60]
    assert ex.GetLevels() == 8
