"""Optimizer::LocalInertialBA as a whole (reference src/Optimizer.cc:2383-2958, monocular observations) over a small map model built on
liba_scenes.graph: keyframes with mPrevKF, bImu, mpImuPreintegrated, the IMU state, the camera pose and slots; map points with
observations {keyframe id: keypoint index}, nObs, mpRefKF, mTrackDepth and the bad flag.  Keyframe-id order is the stand-in for KeyFrame*
order (the order of every std::map); the graph's keyframes are relabelled at random, so that order is not the window's.
- flatten: the LocalInertialBAMap dict of one map and its keyframe pKF (local_inertial_ba_map_batch, the CPU oracle);
- restate: an independent restatement of the walk (rules 1-8 of the window, the local points, lFixedKeyFrames and the edges) and of the
  finish (the erase test, the cascade and the float write-back, numpy float32 with one rounding per operation), given the solver's results;
- oracle: the CPU oracle over a flattened map, with the problem it builds;
- planted: named maps, each with the branch it plants."""
import ctypes as C

import numpy as np

import liba_scenes
import local_ba_lib as LB
import oracle_lib as O
import orb_slam3_modified_b200 as orb
from track_inertial_lib import se3_from_matrix
from track_lib import pose_matrices

F32 = np.float32
BAD, OTHER, IMU, PREINT = orb.KF_BAD, orb.KF_OTHER_MAP, orb.KF_IMU, orb.KF_PREINT
SF = LB.SF
ISG = (1.0 / 1.44 ** np.arange(8)).astype(F32)       # liba_scenes.graph's invSigma2 per octave
TH = 5.991


# ---- map model ----
class KeyFrame(LB.KeyFrame):
    def __init__(self, kid, state21, tcw12, cam, pts, octave):
        pose7 = np.array(se3_from_matrix(np.asarray(tcw12[:9], F32), np.asarray(tcw12[9:], F32)), F32)
        super().__init__(kid, kid, pose7, cam, pts, octave)
        self.state21, self.tcw12 = np.asarray(state21, F32), np.asarray(tcw12, F32)
        self.prev, self.imu, self.preint = -1, True, None
        self.velocity, self.bias6 = self.state21[12:15].copy(), np.concatenate([self.state21[18:21], self.state21[15:18]])


class MapPoint(LB.MapPoint):
    def __init__(self, pid, pos, track_depth):
        super().__init__(pid, pid, pos)
        self.track_depth = F32(track_depth)


class Map(LB.Map):
    def __init__(self, extr):
        super().__init__(inertial=True)
        self.extr = np.asarray(extr, np.float64)


def from_graph(pr, seed, slots_extra=3):
    """The map model of a liba_scenes.graph problem: keyframe k of the graph (0 = pKF, window newest first) gets a random id; k links to
    k + 1 through mPrevKF along the graph's chain, with the graph's preintegration.  Returns (M, ids) with ids[k] the id of graph keyframe k."""
    rng = np.random.default_rng(seed)
    nkf = pr['n_kf']
    ids = [int(i) for i in rng.permutation(nkf) * 2 + 3]
    M = Map(pr['extr'])
    per_kf = [[] for _ in range(nkf)]
    for e, (j, k) in enumerate(zip(pr['e_pt'], pr['e_kf'])):
        per_kf[k].append((int(j), e))
    octave = np.rint(np.log(1.0 / pr['inv_sigma2'].astype(np.float64)) / np.log(1.44)).astype(np.int32)
    assert np.array_equal(ISG[octave], pr['inv_sigma2'])
    for k in range(nkf):
        rows = per_kf[k] + [(-1, -1)] * slots_extra
        rows = [rows[i] for i in rng.permutation(len(rows))]
        pts = [pr['obs'][e] if e >= 0 else (0.0, 0.0) for _, e in rows]
        octs = [octave[e] if e >= 0 else 0 for _, e in rows]
        f = KeyFrame(ids[k], pr['state'][k], pr['tcw'][k], pr['cam'][k], pts, octs)
        for i, (j, _) in enumerate(rows):
            f.mp[i] = j
        M.kfs[ids[k]] = f
    for a, b in zip(pr['ie_kf1'], pr['ie_kf2']):      # the inertial link a -> b: b's mPrevKF is a, b's preintegration the link's
        M.kfs[ids[b]].prev = ids[a]
    for i, b in enumerate(pr['ie_kf2']):
        M.kfs[ids[b]].preint = pr['preint'][i].copy()
    for j in range(len(pr['points'])):
        M.pts[j] = MapPoint(j, pr['points'][j].astype(F32), pr['track_depth'][j])
    for kid, f in M.kfs.items():
        for i, j in enumerate(f.mp):
            if j >= 0:
                M.pts[int(j)].obs[kid] = i
                M.pts[int(j)].nObs += 1
    for q in M.pts.values():
        q.ref = sorted(q.obs)[len(q.obs) // 2] if q.obs else -1
    return M, ids


# ---- flatten ----
def nd(kf_in_map, large):
    return min(kf_in_map - 2, 25 if large else 10)


def flatten(M, pkf, kf_in_map, large=False, rec_init=False):
    """The LocalInertialBAMap dict of map M for keyframe pkf, plus 'kf_ids' / 'pt_ids' (table entry -> model id)."""
    chain = [pkf]
    while len(chain) <= nd(kf_in_map, large) and M.kfs[chain[-1]].prev >= 0 and M.kfs[chain[-1]].prev not in chain:
        chain.append(M.kfs[chain[-1]].prev)
    cands = chain[:max(1, nd(kf_in_map, large))]
    pt_ids, seen = [], set()
    for k in cands:
        for p in M.kfs[k].mp:
            if p >= 0 and p not in seen:
                seen.add(int(p)); pt_ids.append(int(p))
    rest = sorted({k for p in pt_ids for k in M.pts[p].obs} - set(chain))
    kf_ids = chain + rest
    kix = {k: i for i, k in enumerate(kf_ids)}
    pix = {p: i for i, p in enumerate(pt_ids)}
    kfs, pts = [M.kfs[k] for k in kf_ids], [M.pts[p] for p in pt_ids]
    slots = [M.kfs[k].mp if k in cands else [] for k in kf_ids]
    obs = [sorted(q.obs.items()) for q in pts]
    preint = np.zeros((len(kfs), orb.IMU_PREINT_FLOATS), F32)
    for i, f in enumerate(kfs):
        if f.preint is not None:
            preint[i] = f.preint
    return dict(kfFlags=np.array([BAD * f.bad | OTHER * f.other | IMU * f.imu | PREINT * (f.preint is not None) for f in kfs], np.uint8),
                prevKF=np.array([kix.get(f.prev, -1) for f in kfs], np.int32), state21=np.stack([f.state21 for f in kfs]),
                tcw12=np.stack([f.tcw12 for f in kfs]), cameraCenter=np.stack([f.Ow for f in kfs]), cam4=np.stack([f.cam for f in kfs]),
                preint=preint, extrinsics24=M.extr, slotStart=np.cumsum([0] + [len(s) for s in slots]).astype(np.int32),
                slotPoint=np.array([pix[int(p)] if p >= 0 else -1 for s in slots for p in s], np.int32),
                pointFlags=np.array([BAD * q.bad for q in pts], np.uint8),
                worldPos=np.stack([q.pos for q in pts]) if pts else np.zeros((0, 3), F32), trackDepth=np.array([q.track_depth for q in pts], F32),
                refKF=np.array([kix.get(q.ref, -1) for q in pts], np.int32), obsStart=np.cumsum([0] + [len(o) for o in obs]).astype(np.int32),
                obsKF=np.array([kix[k] for o in obs for k, _ in o], np.int32), obsIdx=np.array([i for o in obs for _, i in o], np.int32),
                obsPt=np.array([M.kfs[k].pt[i] for o in obs for k, i in o], F32).reshape(-1, 2),
                obsOctave=np.array([M.kfs[k].octave[i] for o in obs for k, i in o], np.int32), invLevelSigma2=ISG, scaleFactors=SF,
                keyFramesInMap=kf_in_map, bLarge=int(large), bRecInit=int(rec_init), kf_ids=kf_ids, pt_ids=pt_ids)


# ---- CPU oracle ----
class _Built(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('kfState21', 'kfTcw12', 'cam4', 'ieKf1', 'ieKf2', 'preint', 'ieRobust', 'ieInfoScale', 'points3', 'trackDepth',
                                          'edgePoint', 'edgeKf', 'obs2', 'invSigma2', 'sizes', 'lambdaInit')]


def oracle(m, given=None):
    """The oracle's LocalInertialBA on flattened map m: (result dict as Optimizer.local_inertial_ba_map_batch returns it with debug, the
    built problem as a liba_scenes / synth.local_inertial_ba_problem dict).  given: the solver's results (LIBA_MAP_DEBUG + stats8) to finish
    from instead of solving."""
    s, out, keep = orb.liba_map_struct(m, debug=True, given=given)
    nK, nP = len(m['kfFlags']), len(m['pointFlags'])
    nO = int(m['obsStart'][-1]) if nP else 0
    b = dict(kfState21=np.zeros((nK, 21)), kfTcw12=np.zeros((nK, 12)), cam4=np.zeros((nK, 4), F32), ieKf1=np.zeros(nK, np.int32),
             ieKf2=np.zeros(nK, np.int32), preint=np.zeros((nK, orb.IMU_PREINT_FLOATS), F32), ieRobust=np.zeros(nK, np.uint8),
             ieInfoScale=np.zeros(nK), points3=np.zeros((nP, 3)), trackDepth=np.zeros(nP, F32), edgePoint=np.zeros(nO, np.int32),
             edgeKf=np.zeros(nO, np.int32), obs2=np.zeros((nO, 2)), invSigma2=np.zeros(nO, F32), sizes=np.zeros(6, np.int32), lambdaInit=np.zeros(1))
    bs = _Built(*[b[n].ctypes.data for n, _ in _Built._fields_])
    L = O.lib()
    L.orbo_local_inertial_ba_map.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.orbo_local_inertial_ba_map(C.byref(s), int(given is not None), C.byref(bs))
    nKp, nOpt, nI, nL, nE, it = (int(v) for v in b['sizes'])
    pr = dict(n_kf=nKp, n_opt=nOpt, state=b['kfState21'][:nKp], tcw=b['kfTcw12'][:nKp], cam=b['cam4'][:nKp], extr=np.asarray(m['extrinsics24'], np.float64),
              ie_kf1=b['ieKf1'][:nI], ie_kf2=b['ieKf2'][:nI], preint=b['preint'][:nI], ie_robust=b['ieRobust'][:nI], ie_info_scale=b['ieInfoScale'][:nI],
              points=b['points3'][:nL], track_depth=b['trackDepth'][:nL], e_pt=b['edgePoint'][:nE], e_kf=b['edgeKf'][:nE], obs=b['obs2'][:nE],
              inv_sigma2=b['invSigma2'][:nE], iterations=it, lambda_init=float(b['lambdaInit'][0]), large=bool(m['bLarge']))
    return orb.liba_map_result(out), pr


def given_of(r):
    """The solver's results of a debug record, as oracle(given=...) reads them (full-length arrays)."""
    return {n: r[n] for n in ('optState21', 'optTcw12', 'optPoint', 'edgeChi2', 'stats8')}


def padded(r, m):
    """A debug record's solver doubles padded back to the table's lengths (liba_map_result cuts them to the lists)."""
    nK, nP = len(m['kfFlags']), len(m['pointFlags'])
    g = dict(edgeChi2=r['edgeChi2'], stats8=r['stats8'])
    for n, rows, w in (('optState21', nK, 21), ('optTcw12', nK, 12), ('optPoint', nP, 3)):
        a = np.zeros((rows, w)); a[:len(r[n])] = r[n]; g[n] = a
    return g


# ---- independent restatement ----
def restate(M, pkf, kf_in_map, large, rec_init, lm=None):
    """The whole function on model M (changed in place when lm is given and the map does not FAIL).  lm = dict(state {kf id: double [21]},
    tcw {kf id: double [12]}, point {pt id: double [3]}, chi2 {(pt id, kf id): value}, failed).  Returns the record in model ids."""
    K, P = M.kfs, M.pts
    Nd = nd(kf_in_map, large)
    win = [pkf]
    for _ in range(1, Nd):
        if K[win[-1]].prev < 0:
            break
        win.append(K[win[-1]].prev)
    local, fixed_mark = set(win), set()
    pts, seen = [], set()
    for k in win:
        for p in K[k].mp:
            if p >= 0 and not P[p].bad and p not in seen:
                seen.add(int(p)); pts.append(int(p))
    if K[win[-1]].prev >= 0:
        fixed = [K[win[-1]].prev]
    else:
        fixed = [win.pop()]
        local.discard(fixed[0])
    fixed_mark.add(fixed[0])
    for p in pts:
        for k in sorted(P[p].obs):
            if k not in local and k not in fixed_mark:
                fixed_mark.add(k)
                if not K[k].bad:
                    fixed.append(k)
                    break
        if len(fixed) >= 200:
            break
    N = len(win)
    linked = [K[k].prev >= 0 and K[k].imu and K[K[k].prev].imu and K[k].preint is not None for k in win]
    marked = local | fixed_mark
    edges = [(p, k) for p in pts for k in sorted(P[p].obs) if k in marked and not K[k].bad and not K[k].other]
    rec = dict(window=win, fixed=fixed, points=pts, linked=linked, edges=edges, erase=[],
               ie=[(fixed[0] if i == N - 1 else win[i + 1], win[i], i == N - 1 or bool(rec_init), 1e-2 if i == N - 1 else 1.0)
                   for i in range(N) if linked[i]])
    if lm is None:
        return rec
    rec['status'] = orb.LIBA_LOCAL_FAILED if lm['failed'] else orb.LIBA_LOCAL_RAN
    if lm['failed']:
        return rec
    vk = win + fixed
    for p, k in edges:
        T, X = lm['tcw'][k], lm['point'][p]
        depth_pos = T[6] * X[0] + T[7] * X[1] + T[8] * X[2] + T[11] > 0.0
        c2, close = lm['chi2'][(p, k)], P[p].track_depth < F32(10)
        if (c2 > F32(TH) and not close) or (c2 > F32(1.5) * F32(TH) and close) or not depth_pos:
            rec['erase'].append((p, k))
    assert set(vk) >= {k for _, k in edges}
    for p, k in rec['erase']:
        M.erase_match(k, p)
        M.erase_observation(p, k)
    for k in win:
        T = lm['tcw'][k]
        K[k].Tcw = np.array(se3_from_matrix(T[:9].astype(F32), T[9:].astype(F32)), F32)
        K[k].Ow = pose_matrices(K[k].Tcw)[2]
        s = lm['state'][k]
        K[k].velocity, K[k].bias6 = s[12:15].astype(F32), np.concatenate([s[18:21], s[15:18]]).astype(F32)
    for p in pts:
        P[p].pos = np.asarray(lm['point'][p], np.float64).astype(F32)
        LB.update_normal_and_depth(M, P[p])
    return rec


def lm_of(m, r):
    """The solver's results of a flattened map's debug record r in model ids, for restate."""
    kid, pid = m['kf_ids'], m['pt_ids']
    vk = list(r['optKF']) + list(r['fixedKF'])
    lm = dict(state={kid[k]: r['optState21'][v] for v, k in enumerate(vk)}, tcw={kid[k]: r['optTcw12'][v] for v, k in enumerate(vk)},
              point={pid[p]: r['optPoint'][i] for i, p in enumerate(r['localPoint'])}, chi2={}, failed=bool(r['stats8'][2]))
    for p in range(len(pid)):
        for o in range(m['obsStart'][p], m['obsStart'][p + 1]):
            lm['chi2'][(pid[p], kid[m['obsKF'][o]])] = r['edgeChi2'][o]
    return lm


def record_in_ids(m, r):
    """A call's record in model ids, comparable with restate's."""
    kid, pid = m['kf_ids'], m['pt_ids']
    obs = lambda flags: [(pid[p], kid[m['obsKF'][o]]) for p in r['localPoint'] for o in range(m['obsStart'][p], m['obsStart'][p + 1]) if r['obsFlag'][o] in flags]
    return dict(status=r['status'], window=[kid[k] for k in r['optKF']], fixed=[kid[k] for k in r['fixedKF']], points=[pid[p] for p in r['localPoint']],
                linked=[bool(x) for x in r['ieLinked']], edges=obs((orb.LBA_OBS_KEPT, orb.LBA_OBS_ERASED)), erase=obs((orb.LBA_OBS_ERASED,)))


def check_model(M, m, r):
    """The model after restate equals the record's write-back."""
    kid, pid = m['kf_ids'], m['pt_ids']
    for i, k in enumerate(r['optKF']):
        f = M.kfs[kid[k]]
        assert f.Tcw.tobytes() == r['kfPose7'][i].tobytes() and f.Ow.tobytes() == r['kfCenter'][i].tobytes()
        assert f.velocity.tobytes() == r['kfVelocity'][i].tobytes() and f.bias6.tobytes() == r['kfBias6'][i].tobytes()
    for i, p in enumerate(r['localPoint']):
        q = M.pts[pid[p]]
        assert q.pos.tobytes() == r['pointPos'][i].tobytes() and q.bad == bool(r['pointBad'][i])
        assert q.ref == (kid[r['pointRefKF'][i]] if r['pointRefKF'][i] >= 0 else -1)
        if not q.bad:
            assert q.normal.tobytes() == r['normal'][i].tobytes() and F32(q.min_d) == r['minDistance'][i] and F32(q.max_d) == r['maxDistance'][i]


# ---- scenes ----
def scene(seed, n_opt=6, n_cov=3, pred=True, n_pts=120, obs_per_pt=4, **kw):
    """A map on liba_scenes.graph: the window (n_opt keyframes), its predecessor when pred, n_cov older keyframes seen only through points.
    Returns (M, pKF id, ids)."""
    pr = liba_scenes.graph(n_opt, n_cov=n_cov, pred=pred, n_pts=n_pts, obs_per_pt=obs_per_pt, seed=seed, **kw)
    M, ids = from_graph(pr, seed + 500)
    return M, ids[0], ids


def plant_outliers(M, pid, kids, px=60.0):
    for i, k in enumerate(kids):
        M.kfs[k].pt[M.pts[pid].obs[k]] += np.array([0, px if i % 2 else -px], F32)


def planted():
    """Named maps: (M, pKF, KeyFramesInMap, bLarge, bRecInit), each with the branch it plants."""
    out = {}
    M, k, ids = scene(1, n_opt=6, n_cov=3)
    out['normal'] = (M, k, 40, False, False)
    M, k, ids = scene(2, n_opt=5, n_cov=2, pred=False)
    out['popped_predecessor'] = (M, k, 40, False, False)         # the chain breaks before Nd: its last keyframe is popped into the fixed list
    M, k, ids = scene(3, n_opt=8, n_cov=2)
    out['kf_in_map_limits_nd'] = (M, k, 6, False, False)          # Nd = 4: the window stops inside the chain
    M, k, ids = scene(4, n_opt=10, n_cov=4, n_pts=200)
    M.kfs[ids[3]].preint = None                                   # a window keyframe without a preintegration: no inertial edge
    M.kfs[ids[10]].imu = False                                    # the predecessor without bImu: no edge to it either
    out['no_preint'] = (M, k, 40, False, True)                    # bRecInit: every inertial edge robust
    M, k, ids = scene(5, n_opt=6, n_cov=5, n_pts=150)
    M.kfs[ids[7]].bad = True                                      # bad observers: marked, not added, no edges
    M.kfs[ids[9]].bad = True
    M.kfs[ids[8]].other = True                                    # an other-map fixed keyframe: a vertex without edges
    out['bad_other'] = (M, k, 40, False, False)
    M, k, ids = scene(6, n_opt=12, n_cov=3, n_pts=260)
    out['large'] = (M, k, 60, True, False)
    pr = liba_scenes.fixed_200(n_opt=4, n_cov=300, seed=7)         # more than maxFixKF candidates: the cap, and the rule-6 break leaves later observers
    M, ids = from_graph(pr, 507)
    out['cap_200'] = (M, ids[0], 100, False, False)
    pr = liba_scenes.observers(n_opt=6, seed=8)                   # points seen once, fixed-only points, negative depths, trackDepth on 10.0f
    M, ids = from_graph(pr, 508)
    out['observers'] = (M, ids[0], 40, False, False)
    M, k, ids = scene(9, n_opt=6, n_cov=3, n_pts=160, outlier_frac=0.0)
    hub = [j for j, q in M.pts.items() if len(q.obs) >= 4 and not any(M.kfs[kk].bad for kk in q.obs)]
    p0 = hub[0]                                                   # an erase that moves mpRefKF
    plant_outliers(M, p0, [M.pts[p0].ref])
    p1 = hub[1]                                                   # nObs down to 2: the point turns bad, and a later erase finds nothing
    ks = sorted(M.pts[p1].obs)
    M.pts[p1].ref = ks[0]
    plant_outliers(M, p1, ks[1:], px=150.0)
    out['cascade'] = (M, k, 40, False, False)
    M, k, ids = scene(10, n_opt=5, n_cov=2)
    j = next(p for p in M.kfs[k].mp if p >= 0)
    M.kfs[k].pt[M.pts[int(j)].obs[k]] = np.float32([np.nan, 100.0])   # err is NaN: the FAIL test fires
    out['fail'] = (M, k, 40, False, False)
    return out


def seeded(seed):
    """A seeded map of random shape."""
    rng = np.random.default_rng(seed)
    n_opt = int(rng.integers(2, 12))
    M, k, ids = scene(100 + seed, n_opt=n_opt, n_cov=int(rng.integers(0, 5)), pred=bool(rng.random() < 0.8), n_pts=int(rng.integers(40, 200)),
                      obs_per_pt=int(rng.integers(2, 5)))
    for kid in rng.choice(list(M.kfs), 2, replace=False):
        if kid != k and rng.random() < 0.5:
            M.kfs[int(kid)].bad = True
    return M, k, int(rng.integers(3, 30)), bool(rng.random() < 0.3), bool(rng.random() < 0.3)
