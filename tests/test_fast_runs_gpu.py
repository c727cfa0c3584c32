"""Geometries at the edges of the quick test's row runs and of the pyramid's destination tiles, against the CPU oracle: every level's
FAST candidates and pyramid plane, bit for bit.

The quick test walks runs of up to 6 interior rows of one 4-pixel column, and the pyramid writes tiles of 128 x 64 pixels, so:
  * 1304 x 978: the clipped bottom cell row of level 0 leaves a block interior 4 rows tall, shorter than one run; every level has
    blocks whose last quad is partial, and every level but 3 has blocks whose interiors end in a partial run.
  * 466 x 353: partial runs on every level, partial last quads on levels 0-2 and 4-6.
No level height of either size is a multiple of 64, so every pyramid level ends in a partial tile row.  A cell is at least 35 rows
tall unless the image border clips it, so a block interior shorter than a run only occurs in a clipped bottom cell row."""
import numpy as np
import pytest

import oracle_lib as O
from test_fast_blocks_gpu import INI_TH, MIN_TH, _check_batch

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


@pytest.mark.parametrize('w,h', [(1304, 978), (466, 353)])
def test_partial_runs_and_quads(orb, synth, w, h):
    _check_batch(orb, synth.frames(2, w, h, t0=7), [0, 1])


@pytest.mark.parametrize('w,h', [(1304, 978), (466, 353)])
def test_pyramid_partial_tile_rows(orb, synth, w, h):
    images = synth.frames(2, w, h, t0=3)
    ex = orb.ORBextractor(1000, 1.2, 8, INI_TH, MIN_TH, w, h, 2)
    oe = O.OracleExtractor(1000, 1.2, 8, INI_TH, MIN_TH)
    ex.extract_batch(images, (0, 1000))
    for f in range(2):
        oe(images[f], (0, 1000))
        for l in range(1, 8):
            lv, olv = ex.level(l, f), oe.level(l)
            assert lv.shape == olv.shape and lv.shape[0] % 64, ((w, h), l, lv.shape, olv.shape)
            assert np.array_equal(lv, olv), ((w, h), 'frame', f, 'level', l, 'pyramid plane differs')
