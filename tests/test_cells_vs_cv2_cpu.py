"""Independent check of ComputePyramid + the per-cell FAST loop of ComputeKeyPointsOctTree (SURVEY 8a rows a2, a3;
src/ORBextractor.cc:1170-1195, 781-873): the reference's loops transcribed with the real `cv2.resize` / `cv2.FAST` calls, against the
oracle's pyramid planes and its candidate lists (position, response, order) before the quadtree."""
import math

import numpy as np
import pytest

import oracle_lib as O
from orb_slam3_modified_b200 import synth

cv2 = pytest.importorskip('cv2')
EDGE_THRESHOLD = 19


@pytest.mark.parametrize('t,ini,mn', [(4, 20, 7), (8, 20, 7), (8, 60, 12), (4, 12, 5), (4, 40, 7), (4, 20, 20), (4, 3, 1)])
def test_pyramid_and_cell_candidates(t, ini, mn):
    _pyramid_and_cell_candidates(t, ini, mn, 640, 480, 1.2, 8)


# the geometries tests/test_extractor_paths_gpu.py runs (level 1 of the first four takes the bilinear resize, then 4095 px wide, one
# level, 720p), plus a 1.9 scale factor whose levels are neither 2x decimations nor small steps
@pytest.mark.parametrize('w,h,scaleFactor,nlevels', [(517, 389, 2.0, 3), (1241, 376, 2.0, 3), (640, 480, 2.5, 3), (640, 480, 3.0, 2),
                                                     (4095, 300, 1.2, 8), (640, 480, 1.2, 1), (640, 480, 1.9, 4), (1280, 720, 1.2, 8)])
def test_pyramid_and_cell_candidates_geometry(w, h, scaleFactor, nlevels):
    _pyramid_and_cell_candidates(4, 20, 7, w, h, scaleFactor, nlevels)


def _pyramid_and_cell_candidates(t, ini, mn, w, h, scaleFactor, nlevels):
    img = synth.frame(t, w, h)
    ex = O.OracleExtractor(1000, scaleFactor, nlevels, ini, mn)
    ex(img, (0, 1000))
    inv = np.asarray(ex.tables()['inv_scale'], np.float32)
    prev = img
    for level in range(nlevels):
        if level:
            # ComputePyramid :1175-1183: Size(cvRound(cols * scale), cvRound(rows * scale)) with scale = mvInvScaleFactor[level]
            sz = (int(np.rint(np.float32(img.shape[1]) * inv[level])), int(np.rint(np.float32(img.shape[0]) * inv[level])))
            prev = cv2.resize(prev, sz, interpolation=cv2.INTER_LINEAR)
        plane = ex.level(level)
        assert plane.shape == prev.shape and np.array_equal(plane, prev), level
        # ComputeKeyPointsOctTree :788-873
        minBX = minBY = EDGE_THRESHOLD - 3
        maxBX, maxBY = plane.shape[1] - EDGE_THRESHOLD + 3, plane.shape[0] - EDGE_THRESHOLD + 3
        width, height = np.float32(maxBX - minBX), np.float32(maxBY - minBY)
        nCols, nRows = int(width / np.float32(35)), int(height / np.float32(35))
        wCell, hCell = int(math.ceil(width / nCols)), int(math.ceil(height / nRows))
        exp = []
        for i in range(nRows):
            iniY = minBY + i * hCell
            maxY = iniY + hCell + 6
            if iniY >= maxBY - 3:
                continue
            maxY = min(maxY, maxBY)
            for j in range(nCols):
                iniX = minBX + j * wCell
                maxX = iniX + wCell + 6
                if iniX >= maxBX - 6:
                    continue
                maxX = min(maxX, maxBX)
                roi = np.ascontiguousarray(plane[iniY:maxY, iniX:maxX])
                k = cv2.FastFeatureDetector_create(ini, True).detect(roi)
                if not k:
                    k = cv2.FastFeatureDetector_create(mn, True).detect(roi)
                exp += [(p.pt[0] + j * wCell, p.pt[1] + i * hCell, p.response) for p in k]
        got = ex.candidates(level)
        assert len(got) == len(exp), (level, len(got), len(exp))
        if exp:
            e = np.array(exp, np.float32)
            assert np.array_equal(got['x'], e[:, 0]) and np.array_equal(got['y'], e[:, 1]) and np.array_equal(got['response'], e[:, 2]), level
