"""CPU tests of the matcher oracle: golden vectors (cv2 BFMatcher), Hamming properties, grid queries, sanity of the
projection matchers on seeded scenes."""
import os

import numpy as np
import pytest

import oracle_lib as O
import matcher_scenes as S

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def test_bf_knn2_golden():
    g = np.load(os.path.join(G, 'primitives.npz'))
    idx, dist = O.bf_knn2(g['bf_q'], g['bf_t'])
    assert np.array_equal(idx, g['bf_idx']) and np.array_equal(dist, g['bf_dist'])


def test_bf_knn2_vs_cv2_live_with_ties():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(11)
    q = rng.integers(0, 256, (300, 32)).astype(np.uint8)
    t = rng.integers(0, 256, (400, 32)).astype(np.uint8)
    t[100:200] = t[:100]          # exact duplicates -> distance ties
    q[:50] = t[:50]
    m = cv2.BFMatcher(cv2.NORM_HAMMING).knnMatch(q, t, k=2)
    idx, dist = O.bf_knn2(q, t)
    assert np.array_equal(idx, np.array([[a.trainIdx, b.trainIdx] for a, b in m]))
    assert np.array_equal(dist, np.array([[int(a.distance), int(b.distance)] for a, b in m]))


def test_descriptor_distance_properties():
    rng = np.random.default_rng(2)
    a = rng.integers(0, 256, (64, 32)).astype(np.uint8)
    b = rng.integers(0, 256, (64, 32)).astype(np.uint8)
    for i in range(64):
        d = O.descriptor_distance(a[i], b[i])
        assert d == int(np.unpackbits(a[i] ^ b[i]).sum()) == O.descriptor_distance(b[i], a[i])
        assert O.descriptor_distance(a[i], a[i]) == 0
    assert O.descriptor_distance(np.zeros(32, np.uint8), np.full(32, 255, np.uint8)) == 256


def test_features_in_area_bruteforce():
    """Frame::GetFeaturesInArea: the set equals a brute-force window test, and the ORDER equals the (cell x, cell y, index) order of
    matcher_scenes.Cands -- the order breaks ties between equal Hamming distances in every search.  Frames: a seeded one, the
    keypoints placed on cell ties, and the ones placed just outside undistortion-like bounds."""
    frames = [(S.extract(3)[0], (0.0, 0.0, 640.0, 480.0), 200)] + [(S.special_scene(n, 0)['kps'], S.special_scene(n, 0)['bounds'], 1000) for n in ('ties', 'edges')]
    rng = np.random.default_rng(4)
    for kps, b, nq in frames:
        C = S.Cands(kps, b)
        inside = 0
        for _ in range(nq):
            x, y, r = rng.uniform(b[0] - 20, b[2] + 20), rng.uniform(b[1] - 20, b[3] + 20), rng.uniform(1, 60)
            lo, hi = int(rng.integers(-1, 6)), int(rng.integers(-1, 8))
            got = O.features_in_area(kps, b, x, y, r, lo, hi)
            x32, y32, r32 = np.float32(x), np.float32(y), np.float32(r)
            ok = (np.abs(kps['x'] - x32) < r32) & (np.abs(kps['y'] - y32) < r32) & C.ingrid
            if lo > 0 or hi >= 0:
                ok &= kps['octave'] >= lo
                if hi >= 0:
                    ok &= kps['octave'] <= hi
            assert sorted(got.tolist()) == np.nonzero(ok)[0].tolist()
            assert got.tolist() == C.query(x, y, r, lo, hi), (x, y, r, lo, hi)
            inside += int((~C.ingrid[got]).sum() == 0 and ((kps['x'][got] < b[0]) | (kps['y'][got] < b[1])).any())
        assert b[0] == 0 or inside > 0        # keypoints left of / above the bounds that still fall into cell 0 are returned


def test_last_frame_scene_matches_well():
    s = S.last_frame_scene(5)
    K = len(s['kps'])
    match = np.full(K, -1, np.int32)
    claimed = np.zeros(K, np.uint8)
    n = O.search_last_frame(s['kps'], s['desc'], s['bounds'], s['sf'], s['Tcw'], s['cam'], s['last'], 15.0, True, match, claimed)
    assert n >= int((match >= 0).sum()) > 300      # nmatches also counts overwrites of keypoints held by points without observations
    m = np.nonzero(match >= 0)[0]
    d = [O.descriptor_distance(s['desc'][i], s['last']['descriptors'][match[i]]) for i in m]
    assert max(d) <= 100
    assert all(s['last']['valid'][match[i]] for i in m)


def test_local_map_scene_matches():
    s = S.local_map_scene(6)
    K = len(s['kps'])
    match = np.full(K, -1, np.int32)
    claimed = np.zeros(K, np.uint8)
    n = O.search_local_map(s['kps'], s['desc'], s['bounds'], s['sf'], s['pts'], 1.0, 0.8, False, 50.0, match, claimed)
    assert n >= int((match >= 0).sum()) > 200     # nmatches also counts overwrites of unclaimed keypoints
    assert all(s['pts']['inView'][match[i]] and not s['pts']['bad'][match[i]] for i in np.nonzero(match >= 0)[0])


def test_search_for_initialization_oracle():
    """ORBmatcher::SearchForInitialization (src/ORBmatcher.cc:648-763), oracle only for now: two consecutive synthetic frames match
    well, and the result equals a set-based restatement of the same rules (brute force over all F2 keypoints, no grid lists)."""
    import matcher_scenes
    k1, d1 = matcher_scenes.extract(3)
    k2, d2 = matcher_scenes.extract(4)
    sf = (1.2 ** np.arange(8)).astype(np.float32)
    bounds = (0.0, 0.0, 640.0, 480.0)
    prev = np.stack([k1['x'], k1['y']], 1).astype(np.float32)
    n, m12, pm = O.search_for_initialization(k1, d1, k2, d2, bounds, sf, prev, 100, 0.9, True)
    lvl0 = int((k1['octave'] == 0).sum())
    assert n == int((m12 >= 0).sum()) and n > 0.4 * lvl0
    good = m12 >= 0
    assert np.all(k1['octave'][good] == 0) and np.all(k2['octave'][m12[good]] == 0)
    assert len(set(m12[good].tolist())) == n                                  # one F1 keypoint per matched F2 keypoint
    assert np.array_equal(pm[good], np.stack([k2['x'][m12[good]], k2['y'][m12[good]]], 1)) and np.array_equal(pm[~good], prev[~good])
    # restatement without the grid: candidates = F2 keypoints of level 0 whose grid cell lies in the query's cell range and that are
    # inside the window, enumerated in (cell x, cell y, index) order -- the order GetFeaturesInArea produces
    W = np.float32(64 / 640.0); Hh = np.float32(48 / 480.0)
    cx2 = np.round((k2['x'] - np.float32(0)) * W).astype(int); cy2 = np.round((k2['y'] - np.float32(0)) * Hh).astype(int)
    order2 = np.lexsort((np.arange(len(k2)), cy2, cx2))
    md = np.full(len(k2), 2 ** 31 - 1, np.int64); m21 = np.full(len(k2), -1); exp = np.full(len(k1), -1); cnt = 0
    hist = [[] for _ in range(30)]
    for i1 in range(len(k1)):
        if k1['octave'][i1] > 0:
            continue
        x, y, r = prev[i1, 0], prev[i1, 1], np.float32(100)
        x0 = max(0, int(np.floor((x - r) * W))); x1 = min(63, int(np.ceil((x + r) * W)))
        y0 = max(0, int(np.floor((y - r) * Hh))); y1 = min(47, int(np.ceil((y + r) * Hh)))
        best = best2 = 2 ** 31 - 1; bi = -1
        for i2 in order2:
            if k2['octave'][i2] != 0 or not (x0 <= cx2[i2] <= x1 and y0 <= cy2[i2] <= y1):
                continue
            if not (abs(k2['x'][i2] - x) < r and abs(k2['y'][i2] - y) < r):
                continue
            dist = int(np.unpackbits(d1[i1] ^ d2[i2]).sum())
            if md[i2] <= dist:
                continue
            if dist < best:
                best2, best, bi = best, dist, i2
            elif dist < best2:
                best2 = dist
        if best <= 50 and best < np.float32(best2) * np.float32(0.9):
            if m21[bi] >= 0:
                exp[m21[bi]] = -1; cnt -= 1
            exp[i1] = bi; m21[bi] = i1; md[bi] = best; cnt += 1
            rot = k1['angle'][i1] - k2['angle'][bi]
            if rot < 0:
                rot += np.float32(360)
            b = int(np.floor(np.float32(rot * np.float32(1.0 / 30)) + 0.5))
            hist[0 if b == 30 else b].append(i1)
    sizes = [len(h) for h in hist]
    top = sorted(range(30), key=lambda i: (-sizes[i], i))[:3]
    keep = [top[0]] + [t for t in top[1:] if sizes[t] >= 0.1 * sizes[top[0]]]
    for i in range(30):
        if i not in keep:
            for idx in hist[i]:
                if exp[idx] >= 0:
                    exp[idx] = -1; cnt -= 1
    assert cnt == n and np.array_equal(exp, m12)
