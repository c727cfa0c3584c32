"""A second, structurally different restatement of the two per-frame projection searches (SURVEY 8a rows a10, a11): no grid lists --
for every query the candidates are found by testing ALL keypoints (cell of the keypoint by `round`, cell range of the query by
floor/ceil, level filter, window test) and ordered by (cell x, cell y, keypoint index), which is the order Frame::GetFeaturesInArea
produces (src/Frame.cc:657-723); the matching rules are then applied literally (src/ORBmatcher.cc:43-213, 1676-1887).  The C++ oracle
(grid-list transcription) must give exactly the same assignments."""
import numpy as np

import matcher_scenes as S
import oracle_lib as O

TH_HIGH, HISTO = 100, 30


def _ham(a, b):
    return int(np.unpackbits(a ^ b).sum())


def _three_maxima(sizes):
    m = [0, 0, 0]; ind = [-1, -1, -1]
    for i, s in enumerate(sizes):
        if s > m[0]:
            m = [s, m[0], m[1]]; ind = [i, ind[0], ind[1]]
        elif s > m[1]:
            m = [m[0], s, m[1]]; ind = [ind[0], i, ind[1]]
        elif s > m[2]:
            m[2] = s; ind[2] = i
    if m[1] < np.float32(0.1) * np.float32(m[0]):
        ind[1] = ind[2] = -1
    elif m[2] < np.float32(0.1) * np.float32(m[0]):
        ind[2] = -1
    return ind


def _local_map(s, th, nnratio=0.8):
    kps, desc, sf, p = s['kps'], s['desc'], s['sf'], s['pts']
    C = S.Cands(kps, s['bounds'])
    nnratio = np.float32(nnratio)
    match = np.full(len(kps), -1, np.int32); claimed = np.zeros(len(kps), np.uint8); n = 0
    for i in range(len(p['projX'])):
        if not p['inView'][i] or p['bad'][i]:
            continue
        lvl = int(p['level'][i])
        r = np.float32(2.5 if p['viewCos'][i] > 0.998 else 4.0)
        if th != 1.0:
            r = r * np.float32(th)
        best, best2, bl, bl2, bi = 256, 256, -1, -1, -1
        for idx in C.query(p['projX'][i], p['projY'][i], r * sf[lvl], lvl - 1, lvl):
            if match[idx] >= 0 and claimed[idx]:
                continue
            d = _ham(p['descriptors'][i], desc[idx])
            if d < best:
                best2, best, bl2, bl, bi = best, d, bl, int(kps['octave'][idx]), idx
            elif d < best2:
                bl2, best2 = int(kps['octave'][idx]), d
        if best <= TH_HIGH:
            if bl == bl2 and best > nnratio * np.float32(best2):
                continue
            match[bi] = i; claimed[bi] = p['hasObs'][i]; n += 1
    return n, match, claimed


def _last_frame(s, th, ori=True):
    kps, desc, sf, L = s['kps'], s['desc'], s['sf'], s['last']
    C = S.Cands(kps, s['bounds'])
    qw, qx, qy, qz, tx, ty, tz = (np.float32(v) for v in s['Tcw'])
    fx, fy, cx, cy = (np.float32(v) for v in s['cam'])
    th = np.float32(th)
    match = np.full(len(kps), -1, np.int32); claimed = np.zeros(len(kps), np.uint8); n = 0
    hist = [[] for _ in range(HISTO)]
    for i in range(len(L['valid'])):
        if not L['valid'][i]:
            continue
        px, py, pz = (np.float32(v) for v in L['xyz'][i])
        ux, uy, uz = qy * pz - qz * py, qz * px - qx * pz, qx * py - qy * px
        ux, uy, uz = ux + ux, uy + uy, uz + uz
        xc = (px + qw * ux) + (qy * uz - qz * uy) + tx
        yc = (py + qw * uy) + (qz * ux - qx * uz) + ty
        zc = (pz + qw * uz) + (qx * uy - qy * ux) + tz
        if np.float32(1.0 / np.float64(zc)) < 0:
            continue
        u, v = fx * xc / zc + cx, fy * yc / zc + cy
        if u < C.minX or u > np.float32(s['bounds'][2]) or v < C.minY or v > np.float32(s['bounds'][3]):
            continue
        oc = int(L['octave'][i])
        best, bi = 256, -1
        for idx in C.query(u, v, th * sf[oc], oc - 1, oc + 1):
            if match[idx] >= 0 and claimed[idx]:
                continue
            d = _ham(L['descriptors'][i], desc[idx])
            if d < best:
                best, bi = d, idx
        if best <= TH_HIGH:
            match[bi] = i; claimed[bi] = L['hasObs'][i]; n += 1
            rot = np.float32(L['angle'][i]) - np.float32(kps['angle'][bi])
            if rot < 0:
                rot = rot + np.float32(360)
            b = int(np.floor(np.float64(rot * np.float32(1.0 / HISTO)) + 0.5))      # round(): half away from zero, rot >= 0
            hist[0 if b == HISTO else b].append(bi)
    if ori:
        keep = _three_maxima([len(h) for h in hist])
        for b in range(HISTO):
            if b not in keep:
                for idx in hist[b]:
                    match[idx] = -1; claimed[idx] = 0; n -= 1
    return n, match, claimed


def test_local_map_search_set_based():
    """Every scene of matcher_scenes: the seeded ones, the other geometries and bounds, and the placed ones."""
    cases = [(S.local_map_scene(t), 3.0) for t in (6, 9)] + [(S.special_scene(name, 0), 1.0) for name in S.SPECIAL]
    for k, (s, th) in enumerate(cases):
        n, match, claimed = _local_map(s, th)
        m2 = np.full(len(s['kps']), -1, np.int32); c2 = np.zeros(len(s['kps']), np.uint8)
        n2 = O.search_local_map(s['kps'], s['desc'], s['bounds'], s['sf'], s['pts'], th, 0.8, False, 50.0, m2, c2)
        assert n == n2 and np.array_equal(match, m2) and np.array_equal(claimed, c2), k


def test_last_frame_search_set_based():
    cases = [S.last_frame_scene(t) for t in (5, 8)] + [S.special_scene(name, 1) for name in S.SPECIAL]
    for k, s in enumerate(cases):
        # the restatement projects with the oracle's float evaluation order of Tcw * x, which is part of its contract
        n, match, claimed = _last_frame(s, 15.0)
        m2 = np.full(len(s['kps']), -1, np.int32); c2 = np.zeros(len(s['kps']), np.uint8)
        n2 = O.search_last_frame(s['kps'], s['desc'], s['bounds'], s['sf'], s['Tcw'], s['cam'], s['last'], 15.0, True, m2, c2)
        assert n == n2 and np.array_equal(match, m2) and np.array_equal(claimed, c2), k
