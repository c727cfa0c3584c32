"""Scenes and oracle bindings for LocalMapping::CreateNewMapPoints (test infrastructure)."""
import ctypes as C

import numpy as np

import oracle_lib as O
import matcher_scenes as S
from orb_slam3_modified_b200 import synth, NEW_POINT_DTYPE, OrbmTriFrame, OrbmNewPointsIn, KP_DTYPE

# reason codes of oracle/mapping_oracle.cpp
NO_MATCH, LOW_PARALLAX, SVD_W0, DEPTH1, DEPTH2, REPROJ1, REPROJ2, ZERO_DIST, FAR, SCALE, CREATED, TAKEN = range(12)
REASONS = ('no match', 'low parallax', 'SVD w = 0', 'depth 1', 'depth 2', 'reprojection 1', 'reprojection 2', 'zero distance', 'far', 'scale',
           'created', 'taken')


def pose34(t):
    """Tcw of frame t as the float 3x4 of GetPose().matrix3x4(), and GetCameraCenter() (float64 maths, rounded to float32)."""
    T = synth.pose(t)
    w, x, y, z = T[:4]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                  [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    return np.concatenate([R, T[4:, None]], 1).astype(np.float32), (-R.T @ T[4:]).astype(np.float32)


def scene(t, dts, seed=0, p_mp1=0.3, p_mp2=0.4):
    """Keyframe t and its neighbours t + dt (in list order), with random hasMapPoint flags and everything CreateNewMapPoints reads."""
    rng = np.random.default_rng(seed + 101 * t + len(dts))
    voc = O.synthetic_vocabulary(10, 4, seed=14)
    tab = O.OracleExtractor().tables()
    k1, d1 = S.extract(t)
    kf1 = dict(kps=k1, desc=d1, has_mp=(rng.random(len(k1)) < p_mp1).astype(np.uint8), fv=O.bow_transform(voc, d1, 2)[2:])
    kf2, ep, F12, Tcw, Ow = [], [], [], [pose34(t)[0]], [pose34(t)[1]]
    for dt in dts:
        k2, d2 = S.extract(t + dt)
        kf2.append(dict(kps=k2, desc=d2, has_mp=(rng.random(len(k2)) < p_mp2).astype(np.uint8), fv=O.bow_transform(voc, d2, 2)[2:]))
        e, F = O.triangulation_geometry(dict(T1w=synth.pose(t).astype(np.float32), T2w=synth.pose(t + dt).astype(np.float32), cam=synth.camera()))
        ep.append(e); F12.append(F)
        T, o = pose34(t + dt)
        Tcw.append(T); Ow.append(o)
    n = len(dts)
    return dict(kf1=kf1, kf2=kf2, sf=tab['scale'], sigma2=tab['sigma2'], ep=np.array(ep, np.float32).reshape(n, 2), F12=np.array(F12, np.float32).reshape(n, 9),
                Tcw=np.array(Tcw, np.float32).reshape(n + 1, 3, 4), Ow=np.array(Ow, np.float32).reshape(n + 1, 3),
                cam=np.tile(synth.camera(), (n + 1, 1)).astype(np.float32), scale_factor=np.float32(1.2))


class _In:
    """OrbmNewPointsIn over a scene, keeping every array alive."""

    def __init__(self, sc, coarse=False, inertial=False, th_far=0.0):
        self.keep = []

        def mk(kf):
            a = [np.ascontiguousarray(kf['kps'], KP_DTYPE), np.ascontiguousarray(kf['desc'], np.uint8), np.ascontiguousarray(kf['has_mp'], np.uint8),
                 np.ascontiguousarray(kf['fv'][0], np.int32), np.ascontiguousarray(kf['fv'][1], np.int32)]
            self.keep.append(a)
            return OrbmTriFrame(len(a[0]), a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data, len(a[3]), a[3].ctypes.data, a[4].ctypes.data)
        self.f1 = mk(sc['kf1'])
        n = len(sc['kf2'])
        self.f2 = (OrbmTriFrame * max(n, 1))(*[mk(k) for k in sc['kf2']])
        arr = [np.ascontiguousarray(sc[k], np.float32) for k in ('ep', 'F12', 'sf', 'sigma2', 'Tcw', 'Ow', 'cam')]
        self.keep.append(arr)
        self.s = OrbmNewPointsIn(C.pointer(self.f1), n, C.cast(self.f2, C.POINTER(OrbmTriFrame)), arr[0].ctypes.data, arr[1].ctypes.data, arr[2].ctypes.data,
                                 arr[3].ctypes.data, len(arr[2]), arr[4].ctypes.data, arr[5].ctypes.data, arr[6].ctypes.data, float(sc['scale_factor']),
                                 int(coarse), int(inertial), float(th_far))
        self.N1, self.n = len(sc['kf1']['kps']), n


def create(sc, coarse=False, inertial=False, th_far=0.0):
    """The oracle's one-shot orbo_create_new_map_points: (records, nmatches, ncreated, reason [n, N1])."""
    L = O.lib()
    i = _In(sc, coarse, inertial, th_far)
    out = np.zeros(max(i.N1, 1), NEW_POINT_DTYPE)
    nm, nc = np.zeros(i.n, np.int32), np.zeros(i.n, np.int32)
    why = np.zeros((i.n, i.N1), np.uint8)
    n = C.c_int(0)
    L.orbo_create_new_map_points.argtypes = [C.c_void_p] * 6
    L.orbo_create_new_map_points(C.byref(i.s), out.ctypes.data, C.byref(n), nm.ctypes.data, nc.ctypes.data, why.ctypes.data)
    return out[:n.value].copy(), nm, nc, why


def match(sc, k, idx1, idx2, inertial=False, th_far=0.0, _in=None):
    """orbo_new_point_for_match: (reason, record)."""
    L = O.lib()
    i = _in or _In(sc, False, inertial, th_far)
    rec = np.zeros(1, NEW_POINT_DTYPE)
    L.orbo_new_point_for_match.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p]
    return L.orbo_new_point_for_match(C.byref(i.s), k, idx1, idx2, rec.ctypes.data), rec[0]


def triangulate(x1, y1, x2, y2, T1, T2):
    """orbo_triangulate: (ok, x3D, V [4, 4] after sorting)."""
    L = O.lib()
    T1 = np.ascontiguousarray(T1, np.float32); T2 = np.ascontiguousarray(T2, np.float32)
    x = np.zeros(3, np.float32); V = np.zeros((4, 4), np.float32)
    L.orbo_triangulate.argtypes = [C.c_float] * 4 + [C.c_void_p] * 4
    ok = L.orbo_triangulate(x1, y1, x2, y2, T1.ctypes.data, T2.ctypes.data, x.ctypes.data, V.ctypes.data)
    return ok, x, V


def sequential(sc, search, coarse=False, inertial=False, th_far=0.0):
    """The reference's loop literally: for each neighbour in order, search with KF1's CURRENT hasMapPoint (search(k, has_mp1) -> matches12),
    check every match in idx1 order, and mark KF1's features that received a point.  Returns (records, nmatches, ncreated)."""
    has = sc['kf1']['has_mp'].copy()
    recs, nm, nc = [], np.zeros(len(sc['kf2']), np.int32), np.zeros(len(sc['kf2']), np.int32)
    i = _In(sc, coarse, inertial, th_far)
    for k in range(len(sc['kf2'])):
        m12 = search(k, has.copy())
        for idx1 in np.nonzero(m12 >= 0)[0]:
            nm[k] += 1
            why, rec = match(sc, k, int(idx1), int(m12[idx1]), _in=i)
            if why == CREATED:
                recs.append(rec); nc[k] += 1
                has[idx1] = 1
    return np.array(recs, NEW_POINT_DTYPE), nm, nc


def oracle_search(sc, coarse=False):
    """search(k, has_mp1) of the oracle: ORBmatcher(0.6f, false).SearchForTriangulation."""
    def run(k, has):
        kf1, kf2 = sc['kf1'], sc['kf2'][k]
        s2 = dict(k1=kf1['kps'], d1=kf1['desc'], mp1=has, fv1=kf1['fv'], k2=kf2['kps'], d2=kf2['desc'], mp2=kf2['has_mp'], fv2=kf2['fv'], sf=sc['sf'],
                  sigma2=sc['sigma2'])
        return O.search_for_triangulation(s2, sc['ep'][k], sc['F12'][k], coarse, False)[1]
    return run
