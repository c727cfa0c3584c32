"""ctypes loader for the CPU oracle (test infrastructure; never imported by the product)."""
import ctypes as C
import os
import subprocess
import numpy as np

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SO = os.path.join(_ROOT, 'oracle', 'liborb_oracle.so')

KP_DTYPE = np.dtype([('x', 'f4'), ('y', 'f4'), ('size', 'f4'), ('angle', 'f4'), ('response', 'f4'), ('octave', 'i4'), ('class_id', 'i4')])
assert KP_DTYPE.itemsize == 28

_lib = None


def lib():
    global _lib
    if _lib is None:
        srcs = [os.path.join(_ROOT, 'oracle', f) for f in os.listdir(os.path.join(_ROOT, 'oracle')) if f.endswith(('.cpp', '.h'))]
        if not os.path.exists(_SO) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs):
            subprocess.check_call(['make', '-s', '-C', os.path.join(_ROOT, 'oracle')])
        _lib = C.CDLL(_SO)
        _lib.orbo_create.restype = C.c_void_p
        _lib.orbo_create.argtypes = [C.c_int, C.c_float, C.c_int, C.c_int, C.c_int]
        _lib.orbo_destroy.argtypes = [C.c_void_p]
        _lib.orbo_fast_atan2.restype = C.c_float
        _lib.orbo_fast_atan2.argtypes = [C.c_float, C.c_float]
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class OracleExtractor:
    """Mirror of ORBextractor (reference include/ORBextractor.h:43-109) over the oracle."""

    def __init__(self, nfeatures=1000, scale=1.2, nlevels=8, ini_th=20, min_th=7):
        self.L = lib()
        self.nlevels = nlevels
        self.nfeatures = nfeatures
        self.h = C.c_void_p(self.L.orbo_create(nfeatures, scale, nlevels, ini_th, min_th))

    def __del__(self):
        if getattr(self, 'h', None):
            self.L.orbo_destroy(self.h)
            self.h = None

    def __call__(self, img, lap=(0, 0)):
        img = np.ascontiguousarray(img, np.uint8)
        cap = self.nfeatures + 64 * self.nlevels + 4096
        kps = np.zeros(cap, KP_DTYPE)
        desc = np.zeros((cap, 32), np.uint8)
        n = C.c_int(0)
        mono = self.L.orbo_extract(self.h, _p(img), img.shape[0], img.shape[1], img.strides[0], lap[0], lap[1], _p(kps), _p(desc), cap, C.byref(n))
        return mono, kps[:n.value].copy(), desc[:n.value].copy()

    def tables(self):
        nl = self.nlevels
        s, i, g, ig = (np.zeros(nl, np.float32) for _ in range(4))
        f = np.zeros(nl, np.int32)
        u = np.zeros(16, np.int32)
        self.L.orbo_tables(self.h, _p(s), _p(i), _p(g), _p(ig), _p(f), _p(u))
        return dict(scale=s, inv_scale=i, sigma2=g, inv_sigma2=ig, features_per_level=f, umax=u)

    def level(self, l):
        w, h = C.c_int(), C.c_int()
        self.L.orbo_level_size(self.h, l, C.byref(w), C.byref(h))
        out = np.zeros((h.value, w.value), np.uint8)
        self.L.orbo_level_copy(self.h, l, _p(out))
        return out

    def candidates(self, l, cap=200000):
        out = np.zeros(cap, KP_DTYPE)
        n = self.L.orbo_level_candidates(self.h, l, _p(out), cap)
        return out[:n].copy()

    def keypoints(self, l, cap=20000):
        out = np.zeros(cap, KP_DTYPE)
        n = self.L.orbo_level_keypoints(self.h, l, _p(out), cap)
        return out[:n].copy()

    def distribute(self, cands, minX, maxX, minY, maxY, N):
        cands = np.ascontiguousarray(cands, KP_DTYPE)
        out = np.zeros(len(cands) + 8, KP_DTYPE)
        n = self.L.orbo_distribute(self.h, _p(cands), len(cands), minX, maxX, minY, maxY, N, _p(out), len(out))
        return out[:n].copy()


def resize_linear(src, dw, dh):
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.zeros((dh, dw), np.uint8)
    lib().orbo_resize_linear(_p(src), src.shape[1], src.shape[0], src.strides[0], _p(dst), dw, dh, dw)
    return dst


def blur7(src):
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.zeros_like(src)
    lib().orbo_blur7(_p(src), src.shape[1], src.shape[0], src.strides[0], _p(dst), src.shape[1])
    return dst


def fast(roi, T):
    roi = np.ascontiguousarray(roi, np.uint8)
    cap = roi.size
    out = np.zeros((cap, 3), np.int32)
    n = lib().orbo_fast(_p(roi), roi.shape[1], roi.shape[0], roi.strides[0], T, _p(out), cap)
    return out[:n].copy()


def fast_atan2(y, x):
    y = np.ascontiguousarray(y, np.float32)
    x = np.ascontiguousarray(x, np.float32)
    out = np.zeros_like(y)
    lib().orbo_fast_atan2_n(_p(y), _p(x), _p(out), len(y))
    return out


def sincosf(a):
    a = np.ascontiguousarray(a, np.float32)
    s = np.zeros_like(a)
    c = np.zeros_like(a)
    lib().orbo_sincosf_n(_p(a), _p(s), _p(c), len(a))
    return s, c


# ---------------------------------------------------------------------------------------------
# matchers
# ---------------------------------------------------------------------------------------------
def _c(a, dt):
    return np.ascontiguousarray(a, dt)


def descriptor_distance(a, b):
    a = _c(a, np.uint8)
    b = _c(b, np.uint8)
    return lib().orbo_descriptor_distance(_p(a), _p(b))


def search_local_map(kps, desc, bounds, scale_factors, pts, th, nnratio, b_far, th_far, match, claimed):
    kps = _c(kps, KP_DTYPE); desc = _c(desc, np.uint8); b = _c(bounds, np.float32); sf = _c(scale_factors, np.float32)
    a = {k: _c(pts[k], dt) for k, dt in (('inView', np.uint8), ('bad', np.uint8), ('depth', np.float32), ('projX', np.float32),
                                          ('projY', np.float32), ('level', np.int32), ('viewCos', np.float32), ('hasObs', np.uint8),
                                          ('descriptors', np.uint8))}
    L = lib()
    L.orbo_search_local_map.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 9 + [C.c_float, C.c_float, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    return L.orbo_search_local_map(len(kps), _p(kps), _p(desc), _p(b), _p(sf), len(a['projX']), _p(a['inView']), _p(a['bad']), _p(a['depth']),
                                   _p(a['projX']), _p(a['projY']), _p(a['level']), _p(a['viewCos']), _p(a['hasObs']), _p(a['descriptors']),
                                   th, nnratio, int(b_far), th_far, _p(match), _p(claimed))


def search_for_initialization(kps1, desc1, kps2, desc2, bounds, scale_factors, prev_matched, window=100, nnratio=0.9, check_ori=True):
    kps1 = _c(kps1, KP_DTYPE); kps2 = _c(kps2, KP_DTYPE); d1 = _c(desc1, np.uint8); d2 = _c(desc2, np.uint8)
    b = _c(bounds, np.float32); sf = _c(scale_factors, np.float32)
    pm = _c(prev_matched, np.float32).copy()
    m12 = np.full(len(kps1), -1, np.int32)
    L = lib()
    L.orbo_search_for_initialization.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_int, C.c_float, C.c_int, C.c_void_p]
    n = L.orbo_search_for_initialization(len(kps1), _p(kps1), _p(d1), len(kps2), _p(kps2), _p(d2), _p(b), _p(sf), _p(pm), int(window), nnratio,
                                         int(check_ori), _p(m12))
    return n, m12, pm


def is_in_frustum(pts, Rcw, tcw, Ow, cam, bounds, log_scale_factor, n_levels, viewing_cos_limit=0.5, mbf=0.0):
    a = {k: _c(pts[k], np.float32) for k in ('worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance')}
    M = len(a['minDistInv'])
    R = _c(np.asarray(Rcw, np.float32).reshape(9), np.float32); t = _c(tcw, np.float32); o = _c(Ow, np.float32)
    cm = _c(cam, np.float32); b = _c(bounds, np.float32)
    out = dict(inView=np.zeros(M, np.uint8), projX=np.zeros(M, np.float32), projY=np.zeros(M, np.float32), projXR=np.zeros(M, np.float32),
               depth=np.zeros(M, np.float32), level=np.zeros(M, np.int32), viewCos=np.zeros(M, np.float32))
    L = lib()
    L.orbo_is_in_frustum.restype = None
    L.orbo_is_in_frustum.argtypes = [C.c_int] + [C.c_void_p] * 10 + [C.c_float, C.c_float, C.c_int, C.c_float] + [C.c_void_p] * 7
    L.orbo_is_in_frustum(M, _p(a['worldPos']), _p(a['normal']), _p(a['minDistInv']), _p(a['maxDistInv']), _p(a['maxDistance']), _p(R), _p(t), _p(o),
                         _p(cm), _p(b), float(mbf), float(np.float32(log_scale_factor)), int(n_levels), float(viewing_cos_limit),
                         *[_p(out[k]) for k in ('inView', 'projX', 'projY', 'projXR', 'depth', 'level', 'viewCos')])
    return out


def search_last_frame(kps, desc, bounds, scale_factors, Tcw, cam, last, th, check_ori, match, claimed):
    kps = _c(kps, KP_DTYPE); desc = _c(desc, np.uint8); b = _c(bounds, np.float32); sf = _c(scale_factors, np.float32)
    T = _c(Tcw, np.float32); cm = _c(cam, np.float32)
    a = {k: _c(last[k], dt) for k, dt in (('valid', np.uint8), ('xyz', np.float32), ('octave', np.int32), ('angle', np.float32),
                                           ('hasObs', np.uint8), ('descriptors', np.uint8))}
    L = lib()
    L.orbo_search_last_frame.argtypes = [C.c_int] + [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 6 + [C.c_float, C.c_int, C.c_void_p, C.c_void_p]
    return L.orbo_search_last_frame(len(kps), _p(kps), _p(desc), _p(b), _p(sf), _p(T), _p(cm), len(a['valid']), _p(a['valid']), _p(a['xyz']),
                                    _p(a['octave']), _p(a['angle']), _p(a['hasObs']), _p(a['descriptors']), th, int(check_ori), _p(match), _p(claimed))


def bf_knn2(q, t):
    q = _c(q, np.uint8).reshape(-1, 32); t = _c(t, np.uint8).reshape(-1, 32)
    idx = np.zeros((len(q), 2), np.int32); dist = np.zeros((len(q), 2), np.int32)
    lib().orbo_bf_knn2(_p(q), len(q), _p(t), len(t), _p(idx), _p(dist))
    return idx, dist


def features_in_area(kps, bounds, x, y, r, min_level, max_level):
    kps = _c(kps, KP_DTYPE); b = _c(bounds, np.float32)
    out = np.zeros(len(kps) + 1, np.int32)
    L = lib()
    L.orbo_features_in_area.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_int, C.c_int, C.c_void_p, C.c_int]
    n = L.orbo_features_in_area(len(kps), _p(kps), _p(b), x, y, r, min_level, max_level, _p(out), len(out))
    return out[:n].copy()


# ---------------------------------------------------------------------------------------------
# local bundle adjustment
# ---------------------------------------------------------------------------------------------
def lba_solve(prob, iterations=10, user_lambda_init=0.0, stop_flag=None):
    """Runs the oracle LBA on a synth.lba_problem dict; returns dict(poses, points, chi2, depth_pos, iters, stats)."""
    poses = _c(prob['poses'], np.float64).copy(); points = _c(prob['points'], np.float64).copy()
    fixed = _c(prob['fixed'], np.uint8); cam = _c(prob['cam'], np.float32)
    ep = _c(prob['edge_point'], np.int32); ek = _c(prob['edge_pose'], np.int32)
    obs = _c(prob['obs'], np.float64); isg = _c(prob['inv_sigma2'], np.float32)
    nE = len(ep)
    chi2 = np.zeros(nE, np.float64); dpos = np.zeros(nE, np.uint8); stats = np.zeros(8, np.float64)
    L = lib()
    L.orbo_lba_solve.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_double, C.c_int, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    sf = _p(stop_flag) if stop_flag is not None else None
    it = L.orbo_lba_solve(len(poses), _p(poses), _p(fixed), _p(cam), len(points), _p(points), nE, _p(ep), _p(ek), _p(obs), _p(isg),
                          float(prob['huber_delta']), iterations, user_lambda_init, sf, _p(chi2), _p(dpos), _p(stats))
    return dict(poses=poses, points=points, chi2=chi2, depth_pos=dpos, iters=it, stats=stats)


def lba_residuals(prob, poses, points):
    poses = _c(poses, np.float64); points = _c(points, np.float64); cam = _c(prob['cam'], np.float32)
    ep = _c(prob['edge_point'], np.int32); ek = _c(prob['edge_pose'], np.int32); obs = _c(prob['obs'], np.float64)
    res = np.zeros((len(ep), 2), np.float64)
    lib().orbo_lba_residuals(len(poses), _p(poses), _p(cam), len(points), _p(points), len(ep), _p(ep), _p(ek), _p(obs), _p(res))
    return res


def pose_optimization(frame):
    pose = _c(frame['pose'], np.float64).copy(); cam = _c(frame['cam'], np.float32)
    Xw = _c(frame['Xw'], np.float64); obs = _c(frame['obs'], np.float64); isg = _c(frame['inv_sigma2'], np.float32)
    N = len(obs)
    outl = np.zeros(max(N, 1), np.uint8); stats = np.zeros(8)
    L = lib()
    L.orbo_pose_optimization.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_void_p, C.c_void_p]
    n = L.orbo_pose_optimization(_p(pose), _p(cam), N, _p(Xw), _p(obs), _p(isg), float(np.float32(np.sqrt(5.991))), _p(outl), _p(stats))
    return dict(pose=pose, outlier=outl[:N].copy(), inliers=n, trials=int(stats[0]), exhausted=int(stats[1]), rho_zero=int(stats[2]), rounds=int(stats[3]))


# ---------------------------------------------------------------------------------------------
# inertial edges (SURVEY.md 8f rank 1)
# ---------------------------------------------------------------------------------------------
IMU_P_SIZE = 292


def imu_preintegrate(acc, gyr, dts, bias6, noise4):
    acc = _c(acc, np.float32); gyr = _c(gyr, np.float32); dts = _c(dts, np.float32); b = _c(bias6, np.float32); nz = _c(noise4, np.float32)
    P = np.zeros(IMU_P_SIZE, np.float32)
    lib().orbo_imu_preintegrate(len(dts), _p(acc), _p(gyr), _p(dts), _p(b), _p(nz), _p(P))
    return P


def imu_information(P):
    P = _c(P, np.float32)
    info = np.zeros((9, 9)); ig = np.zeros((3, 3)); ia = np.zeros((3, 3))
    lib().orbo_imu_information(_p(P), _p(info), _p(ig), _p(ia))
    return info, ig, ia


def imu_delta(P, bg, ba):
    P = _c(P, np.float32); bg = _c(bg, np.float64); ba = _c(ba, np.float64)
    dR = np.zeros((3, 3)); dV = np.zeros(3); dP = np.zeros(3)
    lib().orbo_imu_delta(_p(P), _p(bg), _p(ba), _p(dR), _p(dV), _p(dP))
    return dR, dV, dP


def imu_edge_inertial(P, s, jac=True):
    """s: dict Rwb1 [3,3], twb1, v1, bg, ba, Rwb2, twb2, v2 (float64).  Returns (err [9], J [9,24] or None)."""
    P = _c(P, np.float32)
    a = {k: _c(s[k], np.float64) for k in ('Rwb1', 'twb1', 'v1', 'bg', 'ba', 'Rwb2', 'twb2', 'v2')}
    err = np.zeros(9); J = np.zeros((9, 24)) if jac else None
    lib().orbo_imu_edge_inertial(_p(P), _p(a['Rwb1']), _p(a['twb1']), _p(a['v1']), _p(a['bg']), _p(a['ba']), _p(a['Rwb2']), _p(a['twb2']), _p(a['v2']),
                                 _p(err), _p(J) if jac else None)
    return err, J


def imu_edge_mono(Rwb, twb, Rcb, tcb, Rbc, tbc, cam4, Xw, obs, jac=True):
    a = [_c(v, np.float64) for v in (Rwb, twb, Rcb, tcb, Rbc, tbc)]
    cam = _c(cam4, np.float32); X = _c(Xw, np.float64); o = _c(obs, np.float64)
    err = np.zeros(2); Jp = np.zeros((2, 3)); Jx = np.zeros((2, 6)); dp = C.c_int(0)
    lib().orbo_imu_edge_mono(*[_p(v) for v in a], _p(cam), _p(X), _p(o), _p(err), _p(Jp) if jac else None, _p(Jx) if jac else None, C.byref(dp))
    return err, Jp, Jx, bool(dp.value)


def imu_pose_update(Rwb, twb, pu):
    R = _c(Rwb, np.float64).copy(); t = _c(twb, np.float64).copy(); u = _c(pu, np.float64)
    lib().orbo_imu_pose_update(_p(R), _p(t), _p(u))
    return R, t


def so3(what, v):
    v = _c(v, np.float64)
    out = np.zeros(3 if what == 'log' else (3, 3))
    lib().orbo_so3({'exp': 0, 'log': 1, 'Jr': 2, 'invJr': 3, 'normalize': 4}[what], _p(v), _p(out))
    return out


# ---------------------------------------------------------------------------------------------
# stereo (Frame::ComputeStereoMatches, the consumer of ORBextractor::mvImagePyramid)
# ---------------------------------------------------------------------------------------------
def stereo_matches(planes_l, planes_r, kl, dl, kr, dr, scale, inv_scale, mb, mbf):
    """planes_*: lists of the unbordered pyramid planes of the left / right extractor (OracleExtractor.level(l))."""
    nl = len(planes_l)
    pl = [np.ascontiguousarray(p, np.uint8) for p in planes_l]; pr = [np.ascontiguousarray(p, np.uint8) for p in planes_r]
    PL = (C.c_void_p * nl)(*[p.ctypes.data for p in pl]); PR = (C.c_void_p * nl)(*[p.ctypes.data for p in pr])
    w = np.array([p.shape[1] for p in pl], np.int32); h = np.array([p.shape[0] for p in pl], np.int32)
    kl = _c(kl, KP_DTYPE); kr = _c(kr, KP_DTYPE); dl = _c(dl, np.uint8); dr = _c(dr, np.uint8)
    sf = _c(scale, np.float32); isf = _c(inv_scale, np.float32)
    ur = np.zeros(len(kl), np.float32); dep = np.zeros(len(kl), np.float32)
    L = lib()
    L.orbo_stereo_matches.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p]
    n = L.orbo_stereo_matches(nl, PL, PR, _p(w), _p(h), len(kl), _p(kl), _p(dl), len(kr), _p(kr), _p(dr), _p(sf), _p(isf), mb, mbf, _p(ur), _p(dep))
    assert n >= 0, 'a SAD window left the pyramid plane'
    return ur, dep


# ---------------------------------------------------------------------------------------------
# DBoW2 transform (Frame::ComputeBoW)
# ---------------------------------------------------------------------------------------------
def synthetic_vocabulary(k=10, L=3, seed=0, stop_frac=0.02):
    """A random vocabulary tree in the flat layout of include/orb_b200.h (OrbVocabulary): node 0 is the root, every inner node has k children whose
    descriptors are bit-flipped copies of the parent's, leaves carry idf-like weights (a few are 0 = stopped words)."""
    rng = np.random.default_rng(seed)
    parent, desc, level = [0], [np.zeros(32, np.uint8)], [0]
    frontier = [0]
    for lv in range(1, L + 1):
        nxt = []
        for p in frontier:
            for _ in range(k):
                d = desc[p].copy() if lv > 1 else rng.integers(0, 256, 32).astype(np.uint8)
                for b in rng.integers(0, 256, 60 // lv):
                    d[b >> 3] ^= np.uint8(1 << (b & 7))
                parent.append(p); desc.append(d); level.append(lv); nxt.append(len(parent) - 1)
        frontier = nxt
    n = len(parent)
    children = [[] for _ in range(n)]
    for i in range(1, n):
        children[parent[i]].append(i)
    child_start = np.zeros(n + 1, np.int32)
    for i in range(n):
        child_start[i + 1] = child_start[i] + len(children[i])
    flat_children = np.array([c for ch in children for c in ch], np.int32)
    word_id = np.full(n, -1, np.int32)
    leaves = [i for i in range(1, n) if not children[i]]
    word_id[leaves] = np.arange(len(leaves))
    weight = np.zeros(n)
    weight[leaves] = rng.uniform(0.5, 9.0, len(leaves))
    weight[rng.choice(leaves, max(1, int(stop_frac * len(leaves))), replace=False)] = 0.0
    return dict(k=k, L=L, parent=np.array(parent, np.int32), desc=np.stack(desc), weight=weight, child_start=child_start, children=flat_children,
                word_id=word_id, n_words=len(leaves))


def bow_transform(voc, feats, levelsup=4, weighting=0, norm=1):
    feats = _c(feats, np.uint8).reshape(-1, 32)
    N = len(feats)
    ow = np.zeros(max(N, 1), np.int32); ov = np.zeros(max(N, 1)); fn = np.zeros(max(N, 1), np.int32); ff = np.zeros(max(N, 1), np.int32); nf = C.c_int(0)
    L = lib()
    L.orbo_bow_transform.argtypes = [C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    n = L.orbo_bow_transform(voc['L'], weighting, norm, _p(voc['child_start']), _p(voc['children']), _p(_c(voc['desc'], np.uint8)), _p(_c(voc['weight'], np.float64)),
                             _p(voc['word_id']), N, _p(feats), levelsup, _p(ow), _p(ov), len(ow), _p(fn), _p(ff), C.byref(nf))
    return ow[:n].copy(), ov[:n].copy(), fn[:nf.value].copy(), ff[:nf.value].copy()


def bow_score_l1(a, b):
    i1, v1 = _c(a[0], np.int32), _c(a[1], np.float64); i2, v2 = _c(b[0], np.int32), _c(b[1], np.float64)
    L = lib()
    L.orbo_bow_score_l1.restype = C.c_double
    L.orbo_bow_score_l1.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    return L.orbo_bow_score_l1(len(i1), _p(i1), _p(v1), len(i2), _p(i2), _p(v2))


def search_by_bow(kps_kf, desc_kf, kf_point, fv_kf, kps_f, desc_f, fv_f, nnratio=0.7, check_ori=True, _lib=None, _name='orbo_search_by_bow'):
    """fv_*: (node ids, feature indices) parallel arrays in DBoW2::FeatureVector order.  Returns (nmatches, match [nF] = KF feature index or -1)."""
    kk = _c(kps_kf, KP_DTYPE); dk = _c(desc_kf, np.uint8); kp = _c(kf_point, np.uint8); kf_ = _c(kps_f, KP_DTYPE); df = _c(desc_f, np.uint8)
    nk, fk = _c(fv_kf[0], np.int32), _c(fv_kf[1], np.int32); nf, ff = _c(fv_f[0], np.int32), _c(fv_f[1], np.int32)
    match = np.full(len(kf_), -1, np.int32)
    L = _lib or lib()
    fn = getattr(L, _name)
    fn.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                   C.c_float, C.c_int, C.c_void_p]
    n = fn(len(kk), _p(kk), _p(dk), _p(kp), len(nk), _p(nk), _p(fk), len(kf_), _p(kf_), _p(df), len(nf), _p(nf), _p(ff), nnratio, int(check_ori), _p(match))
    return n, match


def distinctive_descriptor(desc, _lib=None, _name='orbo_distinctive_descriptor'):
    d = _c(desc, np.uint8).reshape(-1, 32)
    L = _lib or lib()
    return getattr(L, _name)(len(d), _p(d))


def fuse_scene(t, seed=0, M=3000):
    """A keyframe (frame t) and map points seen from neighbouring frames, for ORBmatcher::Fuse."""
    import matcher_scenes
    from orb_slam3_modified_b200 import synth
    rng = np.random.default_rng(seed + 13 * t)
    kps, desc = matcher_scenes.extract(t)
    T = synth.pose(t)
    w, x, y, z = T[:4]
    Rm = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                   [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    Ow = -Rm.T @ T[4:]
    P, D, Oc = [], [], []
    for dt in (-2, -1, 1, 2):
        k, d = matcher_scenes.extract(t + dt)
        P.append(synth.backproject(np.stack([k['x'], k['y']], 1), t + dt) + rng.normal(0, 0.004, (len(k), 3))); D.append(d); Oc.append(k['octave'])
    P, D, Oc = np.concatenate(P), np.concatenate(D), np.concatenate(Oc)
    sel = rng.permutation(len(P))[:M]
    P, D, Oc = P[sel], D[sel], Oc[sel]
    PO = P - Ow
    dist = np.linalg.norm(PO, axis=1)
    n = PO / dist[:, None] + rng.normal(0, 0.25, P.shape)
    n /= np.linalg.norm(n, axis=1)[:, None]
    dmax = (dist * 1.2 ** Oc * rng.uniform(0.8, 1.3, len(P))).astype(np.float32)
    dmin = (dmax / np.float32(1.2 ** 7)).astype(np.float32)
    state = rng.choice([0, 1, 1, 1, 1, 1, 1, 2, 3], len(P)).astype(np.uint8)
    kf_point = np.where(rng.random(len(kps)) < 0.5, rng.integers(0, 6, len(kps)), -1).astype(np.int32)
    sf = OracleExtractor().tables()
    return dict(kps=kps, desc=desc, bounds=(0.0, 0.0, 640.0, 480.0), sf=sf['scale'], isg=sf['inv_sigma2'], log_sf=np.float32(np.log(np.float32(1.2))),
                Tcw=T.astype(np.float32), Ow=Ow.astype(np.float32), cam=synth.camera(), kf_point=kf_point, kf_point_bad=np.zeros(len(kps), np.uint8),
                state=state, xyz=P.astype(np.float32), normal=n.astype(np.float32), min_d=dmin, max_d=dmax, mp_desc=D,
                mp_obs=rng.integers(1, 6, len(P)).astype(np.int32))


def fuse_search(sc, th=3.0):
    M = len(sc['state'])
    bi = np.zeros(M, np.int32); bd = np.zeros(M, np.int32)
    L = lib()
    L.orbo_fuse_search.restype = None
    L.orbo_fuse_search.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_float] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 6 + [C.c_float, C.c_void_p, C.c_void_p]
    a = [_c(sc['kps'], KP_DTYPE), _c(sc['desc'], np.uint8), _c(sc['bounds'], np.float32), _c(sc['sf'], np.float32), _c(sc['isg'], np.float32)]
    b = [_c(sc['Tcw'], np.float32), _c(sc['Ow'], np.float32), _c(sc['cam'], np.float32)]
    c = [_c(sc['state'], np.uint8), _c(sc['xyz'], np.float32), _c(sc['normal'], np.float32), _c(sc['min_d'], np.float32), _c(sc['max_d'], np.float32), _c(sc['mp_desc'], np.uint8)]
    L.orbo_fuse_search(len(a[0]), *[_p(v) for v in a], len(a[3]), float(sc['log_sf']), *[_p(v) for v in b], M, *[_p(v) for v in c], th, _p(bi), _p(bd))
    return bi, bd


def triangulation_scene(t, dt=3, k=10, L=4, levelsup=2, seed=0):
    """Two keyframes (frames t and t + dt of the synthetic stream) for ORBmatcher::SearchForTriangulation: keypoints, descriptors,
    which features hold a map point, DBoW2 feature vectors, poses, camera, level tables."""
    import matcher_scenes
    from orb_slam3_modified_b200 import synth
    rng = np.random.default_rng(seed + 31 * t + dt)
    voc = synthetic_vocabulary(k, L, seed=k + L)
    k1, d1 = matcher_scenes.extract(t); k2, d2 = matcher_scenes.extract(t + dt)
    tab = OracleExtractor().tables()
    return dict(k1=k1, d1=d1, k2=k2, d2=d2, mp1=(rng.random(len(k1)) < 0.4).astype(np.uint8), mp2=(rng.random(len(k2)) < 0.4).astype(np.uint8),
                fv1=bow_transform(voc, d1, levelsup)[2:], fv2=bow_transform(voc, d2, levelsup)[2:], sf=tab['scale'], sigma2=tab['sigma2'],
                T1w=synth.pose(t).astype(np.float32), T2w=synth.pose(t + dt).astype(np.float32), cam=synth.camera())


def search_for_triangulation(sc, ep, F12, coarse=False, check_ori=True):
    a = [_c(sc['k1'], KP_DTYPE), _c(sc['d1'], np.uint8), _c(sc['mp1'], np.uint8), _c(sc['fv1'][0], np.int32), _c(sc['fv1'][1], np.int32)]
    b = [_c(sc['k2'], KP_DTYPE), _c(sc['d2'], np.uint8), _c(sc['mp2'], np.uint8), _c(sc['fv2'][0], np.int32), _c(sc['fv2'][1], np.int32)]
    c = [_c(sc['sf'], np.float32), _c(sc['sigma2'], np.float32), _c(ep, np.float32), _c(F12, np.float32)]
    m12 = np.full(len(a[0]), -1, np.int32)
    L = lib()
    L.orbo_search_for_triangulation.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p] * 2 + [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_void_p]
    n = L.orbo_search_for_triangulation(len(a[0]), _p(a[0]), _p(a[1]), _p(a[2]), len(a[3]), _p(a[3]), _p(a[4]),
                                        len(b[0]), _p(b[0]), _p(b[1]), _p(b[2]), len(b[3]), _p(b[3]), _p(b[4]), *[_p(v) for v in c], int(coarse), int(check_ori), _p(m12))
    return n, m12


def triangulation_geometry(sc):
    """Epipole of KF1's centre in KF2 and the fundamental matrix F12 = K1^-T [t12]x R12 K2^-1 (src/ORBmatcher.cc:913-929, Pinhole.cpp:109-112) in numpy
    float64, rounded to float32: inputs of the search (the reference evaluates them with Eigen / Sophus)."""
    def Rt(T):
        w, x, y, z = [float(v) for v in T[:4]]
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        return R, np.asarray(T[4:], np.float64)
    R1, t1 = Rt(sc['T1w']); R2, t2 = Rt(sc['T2w'])
    fx, fy, cx, cy = [float(v) for v in sc['cam']]
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])
    Cw = -R1.T @ t1
    C2 = R2 @ Cw + t2
    ep = np.array([fx * C2[0] / C2[2] + cx, fy * C2[1] / C2[2] + cy])
    R12 = R1 @ R2.T
    t12 = t1 - R12 @ t2
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
    F12 = np.linalg.inv(K.T) @ tx @ R12 @ np.linalg.inv(K)
    return ep.astype(np.float32), F12.astype(np.float32).reshape(9)


def search_by_bow_kf(k1, d1, point1, fv1, k2, d2, point2, fv2, nnratio=0.8, check_ori=True, _lib=None, _name='orbo_search_by_bow_kf'):
    """ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*, vpMatches12): (nmatches, match12 [N1] = KF2 feature index or -1)."""
    a = [_c(k1, KP_DTYPE), _c(d1, np.uint8), _c(point1, np.uint8), _c(fv1[0], np.int32), _c(fv1[1], np.int32)]
    b = [_c(k2, KP_DTYPE), _c(d2, np.uint8), _c(point2, np.uint8), _c(fv2[0], np.int32), _c(fv2[1], np.int32)]
    m12 = np.full(len(a[0]), -1, np.int32)
    fn = getattr(_lib or lib(), _name)
    fn.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p] * 2 + [C.c_float, C.c_int, C.c_void_p]
    n = fn(len(a[0]), _p(a[0]), _p(a[1]), _p(a[2]), len(a[3]), _p(a[3]), _p(a[4]), len(b[0]), _p(b[0]), _p(b[1]), _p(b[2]), len(b[3]), _p(b[3]), _p(b[4]),
           nnratio, int(check_ori), _p(m12))
    return n, m12


def fuse_search_sim3(sc, Tcw, Ow, th=3.0):
    """The search of ORBmatcher::Fuse(pKF, Scw, vpPoints, th, vpReplacePoint): (bestIdx, bestDist); Tcw / Ow = the decomposition of Scw."""
    M = len(sc['state'])
    bi = np.zeros(M, np.int32); bd = np.zeros(M, np.int32)
    L = lib()
    L.orbo_fuse_search_sim3.restype = None
    L.orbo_fuse_search_sim3.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_float] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 6 + [C.c_float, C.c_void_p, C.c_void_p]
    a = [_c(sc['kps'], KP_DTYPE), _c(sc['desc'], np.uint8), _c(sc['bounds'], np.float32), _c(sc['sf'], np.float32)]
    b = [_c(Tcw, np.float32), _c(Ow, np.float32), _c(sc['cam'], np.float32)]
    c = [_c(sc['state'], np.uint8), _c(sc['xyz'], np.float32), _c(sc['normal'], np.float32), _c(sc['min_d'], np.float32), _c(sc['max_d'], np.float32), _c(sc['mp_desc'], np.uint8)]
    L.orbo_fuse_search_sim3(len(a[0]), *[_p(v) for v in a], len(a[3]), float(sc['log_sf']), *[_p(v) for v in b], M, *[_p(v) for v in c], th, _p(bi), _p(bd))
    return bi, bd


def sim3_scene(t, dt=2, seed=0):
    """Two keyframes with a map point at (most of) their features and a similarity S12 close to the true relative pose, for ORBmatcher::SearchBySim3."""
    import matcher_scenes
    from orb_slam3_modified_b200 import synth
    rng = np.random.default_rng(seed + 7 * t + dt)
    tab = OracleExtractor().tables()
    out = dict(sf=tab['scale'], log_sf=np.float32(np.log(np.float32(1.2))), bounds=(0.0, 0.0, 640.0, 480.0), cam=synth.camera())
    for k, tt in ((1, t), (2, t + dt)):
        kp, de = matcher_scenes.extract(tt)
        P = synth.backproject(np.stack([kp['x'], kp['y']], 1), tt) + rng.normal(0, 0.003, (len(kp), 3))
        T = synth.pose(tt)
        w, x, y, z = T[:4]
        Rm = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                       [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        dist = np.linalg.norm(P - (-Rm.T @ T[4:]), axis=1)
        dmax = (dist * 1.2 ** kp['octave'] * rng.uniform(0.9, 1.2, len(kp))).astype(np.float32)
        out.update({'k%d' % k: kp, 'd%d' % k: de, 'T%dw' % k: T.astype(np.float32), 'R%d' % k: Rm, 't%d' % k: T[4:], 'state%d' % k: rng.choice([0, 1, 1, 1, 1, 1, 2], len(kp)).astype(np.uint8),
                    'xyz%d' % k: P.astype(np.float32), 'max%d' % k: dmax, 'min%d' % k: (dmax / np.float32(1.2 ** 7)).astype(np.float32),
                    'mpd%d' % k: de.copy()})
    # S12: camera 2 -> camera 1 (scale 1 + a little), R12 = R1 R2^T, t12 = t1 - R12 t2
    R12 = out['R1'] @ out['R2'].T
    t12 = out['t1'] - R12 @ out['t2']
    tr = np.trace(R12)
    qw = np.sqrt(max(tr + 1, 1e-12)) / 2
    q = np.array([qw, (R12[2, 1] - R12[1, 2]) / (4 * qw), (R12[0, 2] - R12[2, 0]) / (4 * qw), (R12[1, 0] - R12[0, 1]) / (4 * qw)])
    out['S12'] = np.concatenate([[1.0 + 0.01 * rng.normal()], q / np.linalg.norm(q), t12 + rng.normal(0, 0.002, 3)]).astype(np.float32)
    pre = np.full(len(out['k1']), -1, np.int32)
    cand = np.flatnonzero(out['state1'] == 1)[:40]
    good2 = np.flatnonzero(out['state2'] == 1)
    pre[cand[::4]] = rng.choice(good2, len(cand[::4]), replace=False)
    out['pre12'] = pre
    return out


def search_by_sim3(sc, pc2of1, pc1of2, th=7.5):
    L = lib()
    m12 = np.zeros(len(sc['k1']), np.int32)
    L.orbo_search_by_sim3.argtypes = [C.c_int, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p] + [C.c_int] + [C.c_void_p] * 7 + [C.c_int] + [C.c_void_p] * 7 + [C.c_float, C.c_void_p, C.c_void_p]
    g = [_c(sc['sf'], np.float32), _c(sc['bounds'], np.float32), _c(sc['cam'], np.float32)]
    a = [_c(sc['k1'], KP_DTYPE), _c(sc['d1'], np.uint8), _c(sc['state1'], np.uint8), _c(pc2of1, np.float32), _c(sc['min1'], np.float32), _c(sc['max1'], np.float32), _c(sc['mpd1'], np.uint8)]
    b = [_c(sc['k2'], KP_DTYPE), _c(sc['d2'], np.uint8), _c(sc['state2'], np.uint8), _c(pc1of2, np.float32), _c(sc['min2'], np.float32), _c(sc['max2'], np.float32), _c(sc['mpd2'], np.uint8)]
    pre = _c(sc['pre12'], np.int32)
    n = L.orbo_search_by_sim3(len(g[0]), _p(g[0]), float(sc['log_sf']), _p(g[1]), _p(g[2]), len(a[0]), *[_p(v) for v in a], len(b[0]), *[_p(v) for v in b], th, _p(pre), _p(m12))
    return n, m12


def sim3_camera_points(sc):
    """The map points of each keyframe in the other keyframe's camera frame (S21 * (T1w * p), S12 * (T2w * p); src/ORBmatcher.cc:1507-1508, :1586-1587)
    in numpy float64, rounded to float32: inputs of the search (the reference evaluates them with Sophus)."""
    s, q, t = float(sc['S12'][0]), sc['S12'][1:5].astype(np.float64), sc['S12'][5:].astype(np.float64)
    w, x, y, z = q
    R12 = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                    [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
    c1 = sc['xyz1'].astype(np.float64) @ sc['R1'].T + sc['t1']
    c2 = sc['xyz2'].astype(np.float64) @ sc['R2'].T + sc['t2']
    p21 = ((c1 - t) @ R12) / s              # S21 = S12^-1
    p12 = s * (c2 @ R12.T) + t
    return p21.astype(np.float32), p12.astype(np.float32)


def pose_inertial_opt_last_kf(pr, preint, rec_init=False, rounds=4, iters=10):
    """Optimizer::PoseInertialOptimizationLastKeyFrame: returns dict(state [21], outlier [N], H [15,15], ret)."""
    L = lib()
    N = len(pr['Xw'])
    st = _c(pr['state'], np.float64).copy(); out = np.zeros(N, np.uint8); H = np.zeros((15, 15))
    L.orbo_pose_inertial_opt_last_kf_n.argtypes = [C.c_int] + [C.c_void_p] * 9 + [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    a = [_c(pr['Xw'], np.float32), _c(pr['obs'], np.float32), _c(pr['inv_sigma2'], np.float32), _c(pr['track_depth'], np.float32), _c(pr['cam'], np.float32),
         _c(pr['extr'], np.float64), _c(preint, np.float32), _c(pr['kf_state'], np.float64)]
    ret = L.orbo_pose_inertial_opt_last_kf_n(N, *[_p(v) for v in a], _p(st), int(rec_init), _p(out), _p(H), rounds, iters)
    return dict(state=st, outlier=out, H=H, ret=ret)


def pose_inertial_opt_one_step(pr, preint):
    return pose_inertial_opt_last_kf(pr, preint, rounds=1, iters=1)['state']


def pose_inertial_opt_last_frame(pr, P_frame, P_kf, rec_init=False, rounds=4, iters=10):
    """Optimizer::PoseInertialOptimizationLastFrame: dict(state [21], prev_state [21], outlier [N], H [15,15], ret)."""
    L = lib()
    N = len(pr['Xw'])
    st = _c(pr['state'], np.float64).copy(); pv = _c(pr['prev_state'], np.float64).copy(); out = np.zeros(N, np.uint8); H = np.zeros((15, 15))
    L.orbo_pose_inertial_opt_last_frame_n.argtypes = [C.c_int] + [C.c_void_p] * 12 + [C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    a = [_c(pr['Xw'], np.float32), _c(pr['obs'], np.float32), _c(pr['inv_sigma2'], np.float32), _c(pr['track_depth'], np.float32), _c(pr['cam'], np.float32),
         _c(pr['extr'], np.float64), _c(P_frame, np.float32), _c(P_kf, np.float32), _c(pr['prior_state'], np.float64), _c(pr['prior_H'], np.float64)]
    ret = L.orbo_pose_inertial_opt_last_frame_n(N, *[_p(v) for v in a], _p(pv), _p(st), int(rec_init), _p(out), _p(H), rounds, iters)
    return dict(state=st, prev_state=pv, outlier=out, H=H, ret=ret)


def constraint_pose_imu_information(H):
    H = _c(H, np.float64); out = np.zeros((15, 15))
    lib().orbo_constraint_pose_imu_information(_p(H), _p(out))
    return out


def liba_preints(pr):
    """The IMU::Preintegrated of every inertial edge of a synth.local_inertial_ba_problem: [nI, 292] float32."""
    from orb_slam3_modified_b200 import synth
    return np.stack([imu_preintegrate(a, g, d, pr['bias6'], synth.IMU_NOISE) for a, g, d in pr['imu']])


def local_inertial_ba(pr, preint, iterations=None, lambda_init=None):
    """Optimizer::LocalInertialBA numeric core: dict(state [nKF,21], tcw [nKF,12], points [nL,3], erase [nE], chi2 [nE], iters, err, err_end, failed, lam, trials)."""
    L = lib()
    st = _c(pr['state'], np.float64).copy(); tc = _c(pr['tcw'], np.float64).copy(); pts = _c(pr['points'], np.float64).copy()
    nE = len(pr['e_pt']); nI = len(pr['ie_kf1'])
    erase = np.zeros(nE, np.uint8); chi2 = np.zeros(nE); stats = np.zeros(8)
    a = dict(cam=_c(pr['cam'], np.float32), extr=_c(pr['extr'], np.float64), k1=_c(pr['ie_kf1'], np.int32), k2=_c(pr['ie_kf2'], np.int32), P=_c(preint, np.float32),
             rob=_c(pr['ie_robust'], np.uint8), sc=_c(pr['ie_info_scale'], np.float64), td=_c(pr['track_depth'], np.float32), ep=_c(pr['e_pt'], np.int32),
             ek=_c(pr['e_kf'], np.int32), obs=_c(pr['obs'], np.float64), isg=_c(pr['inv_sigma2'], np.float32))
    L.orbo_local_inertial_ba.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 4 + \
        [C.c_int, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    it = L.orbo_local_inertial_ba(pr['n_kf'], pr['n_opt'], _p(st), _p(tc), _p(a['cam']), _p(a['extr']), nI, _p(a['k1']), _p(a['k2']), _p(a['P']), _p(a['rob']), _p(a['sc']),
                                  len(pts), _p(pts), _p(a['td']), nE, _p(a['ep']), _p(a['ek']), _p(a['obs']), _p(a['isg']),
                                  pr['iterations'] if iterations is None else iterations, pr['lambda_init'] if lambda_init is None else lambda_init, int(pr['large']),
                                  _p(erase), _p(chi2), _p(stats))
    return dict(state=st, tcw=tc, points=pts, erase=erase, chi2=chi2, iters=it, err=stats[0], err_end=stats[1], failed=bool(stats[2]), lam=stats[3], trials=int(stats[4]))


def local_inertial_ba_residuals(pr, tcw, points):
    res = np.zeros((len(pr['e_pt']), 2))
    tc = _c(tcw, np.float64); pts = _c(points, np.float64); ep = _c(pr['e_pt'], np.int32); ek = _c(pr['e_kf'], np.int32); cam = _c(pr['cam'], np.float32); obs = _c(pr['obs'], np.float64)
    lib().orbo_local_inertial_ba_residuals(len(ep), _p(ep), _p(ek), _p(tc), _p(cam), _p(pts), _p(obs), _p(res))
    return res
