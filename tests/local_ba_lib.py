"""Optimizer::LocalBundleAdjustment as a whole (reference src/Optimizer.cc:1116-1498, monocular) over a small map model: keyframes with
mvpMapPoints, keypoints and a float pose; map points with observations {keyframe id: keypoint index}, nObs, mpRefKF and the bad flag.
Keyframe-id order is the stand-in for KeyFrame* order (the order of every std::map); mnIds are separate, so g2o's vertex order differs.
- flatten: the LbaLocalMap dict of one map and its keyframe pKF (lba_local_bundle_adjustment_batch, the CPU oracle);
- restate: an independent restatement of the walk, the EraseObservation cascade and the float write-back (numpy float32, one rounding per
  operation, as track_lib does) on the model, given the optimiser's results;
- replay: the reference's own calls (EraseMapPointMatch / EraseObservation in the returned order, SetPose, SetWorldPos with the record's
  normal and distances) applied to the model from a record;
- oracle: the CPU oracle over a flattened map; scene / planted: seeded maps whose geometry comes from lba_scenes, with real projections,
  noise and gross outliers, so that erasures happen."""
import copy
import ctypes as C

import numpy as np

import lba_scenes
import oracle_lib as O
import orb_slam3_modified_b200 as orb
from track_lib import pose_matrices, set_pose

F32 = np.float32
BAD, INIT, OTHER = orb.KF_BAD, orb.KF_INIT, orb.KF_OTHER_MAP
TH = 5.991
SF = (F32(1.2) ** np.arange(8, dtype=F32)).astype(F32)
ISG = (F32(1) / (SF * SF)).astype(F32)


# ---- map model ----
class KeyFrame:
    def __init__(self, kid, mnId, Tcw, cam, pts, octave):
        self.id, self.mnId, self.Tcw, self.cam = kid, mnId, np.asarray(Tcw, F32), np.asarray(cam, F32)
        self.Ow = pose_matrices(self.Tcw)[2]
        self.pt, self.octave = np.asarray(pts, F32), np.asarray(octave, np.int32)
        self.mp = np.full(len(pts), -1, np.int64)
        self.bad = self.other = self.init = False


class MapPoint:
    def __init__(self, pid, mnId, pos):
        self.id, self.mnId, self.pos = pid, mnId, np.asarray(pos, F32)
        self.obs, self.nObs, self.ref = {}, 0, -1
        self.bad = self.other = False
        self.normal, self.min_d, self.max_d = np.zeros(3, F32), F32(0), F32(0)


class Map:
    def __init__(self, inertial=False):
        self.kfs, self.pts, self.cov, self.inertial, self.stop = {}, {}, {}, inertial, False

    def state(self):
        kf = {k: (f.Tcw.tobytes(), f.Ow.tobytes(), f.mp.tobytes()) for k, f in self.kfs.items()}
        pt = {p: (q.pos.tobytes(), sorted(q.obs.items()), q.nObs, q.ref, q.bad, q.normal.tobytes(), q.min_d.tobytes(), q.max_d.tobytes())
              for p, q in self.pts.items()}
        return kf, pt

    # KeyFrame::EraseMapPointMatch(pMP), MapPoint::EraseObservation(pKF) and SetBadFlag (src/KeyFrame.cc, src/MapPoint.cc)
    def erase_match(self, kid, pid):
        idx = self.pts[pid].obs.get(kid, -1)
        if idx >= 0:
            self.kfs[kid].mp[idx] = -1

    def erase_observation(self, pid, kid):
        p = self.pts[pid]
        if kid not in p.obs:
            return
        p.nObs -= 1
        del p.obs[kid]
        if p.ref == kid:
            p.ref = min(p.obs) if p.obs else -1
        if p.nObs <= 2:
            p.bad = True
            for k, i in p.obs.items():
                self.kfs[k].mp[i] = -1
            p.obs = {}


# ---- flatten ----
def flatten(M, pkf):
    """The LbaLocalMap dict of map M for keyframe pkf, plus 'kf_ids' / 'pt_ids' (table entry -> model id)."""
    cov = M.cov[pkf]
    cands = [pkf] + list(cov)
    pt_ids, seen = [], set()
    for k in cands:
        for p in M.kfs[k].mp:
            if p >= 0 and p not in seen:
                seen.add(int(p)); pt_ids.append(int(p))
    rest = sorted({k for p in pt_ids for k in M.pts[p].obs} - set(cands))
    kf_ids = cands + rest
    kix = {k: i for i, k in enumerate(kf_ids)}
    pix = {p: i for i, p in enumerate(pt_ids)}
    kfs, pts = [M.kfs[k] for k in kf_ids], [M.pts[p] for p in pt_ids]
    slots = [M.kfs[k].mp for k in cands]
    obs = [sorted(q.obs.items()) for q in pts]
    m = dict(mnId=np.array([f.mnId for f in kfs], np.uint64),
             kfFlags=np.array([BAD * f.bad | OTHER * f.other | INIT * f.init for f in kfs], np.uint8),
             pose7=np.stack([f.Tcw for f in kfs]), cameraCenter=np.stack([f.Ow for f in kfs]), cam4=np.stack([f.cam for f in kfs]),
             cov=np.array([kix[k] for k in cov], np.int32), slotStart=np.cumsum([0] + [len(s) for s in slots]).astype(np.int32),
             slotPoint=np.array([pix[int(p)] if p >= 0 else -1 for s in slots for p in s], np.int32),
             pointId=np.array([q.mnId for q in pts], np.uint64), pointFlags=np.array([BAD * q.bad | OTHER * q.other for q in pts], np.uint8),
             worldPos=np.stack([q.pos for q in pts]) if pts else np.zeros((0, 3), F32),
             refKF=np.array([kix.get(q.ref, -1) for q in pts], np.int32),
             obsStart=np.cumsum([0] + [len(o) for o in obs]).astype(np.int32),
             obsKF=np.array([kix[k] for o in obs for k, _ in o], np.int32), obsIdx=np.array([i for o in obs for _, i in o], np.int32),
             obsPt=np.array([M.kfs[k].pt[i] for o in obs for k, i in o], F32).reshape(-1, 2),
             obsOctave=np.array([M.kfs[k].octave[i] for o in obs for k, i in o], np.int32),
             invLevelSigma2=ISG, scaleFactors=SF, inertial=int(M.inertial), kf_ids=kf_ids, pt_ids=pt_ids)
    if M.stop:
        m['stop'] = np.ones(1, np.uint8)
    return m


# ---- CPU oracle ----
class _Built(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('poses', 'fixed', 'cam', 'points', 'edgePoint', 'edgePose', 'obs', 'invSigma2', 'vertKF', 'vertPoint',
                                          'sizes')]


def oracle(m, given=None):
    """The oracle's LocalBundleAdjustment on flattened map m: (result dict as Optimizer.local_bundle_adjustment_batch returns it with debug,
    built problem dict in synth.lba_problem's layout + vert_kf / vert_point).  given: the optimiser's results to finish instead of solving."""
    s, out, keep = orb.local_ba_struct(m, debug=True, given=given)
    nK, nP = len(m['kfFlags']), len(m['pointFlags'])
    nO = int(m['obsStart'][-1]) if nP else 0
    b = dict(poses=np.zeros((nK, 7)), fixed=np.zeros(nK, np.uint8), cam=np.zeros((nK, 4), F32), points=np.zeros((nP, 3)),
             edge_point=np.zeros(nO, np.int32), edge_pose=np.zeros(nO, np.int32), obs=np.zeros((nO, 2)), inv_sigma2=np.zeros(nO, F32),
             vert_kf=np.zeros(nK, np.int32), vert_point=np.zeros(nP, np.int32), sizes=np.zeros(3, np.int32))
    bs = _Built(*[b[n].ctypes.data for n in ('poses', 'fixed', 'cam', 'points', 'edge_point', 'edge_pose', 'obs', 'inv_sigma2', 'vert_kf',
                                             'vert_point', 'sizes')])
    L = O.lib()
    L.orbo_local_ba.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.orbo_local_ba(C.byref(s), int(given is not None), C.byref(bs))
    nPo, nL, nE = (int(v) for v in b['sizes'])
    built = dict(poses=b['poses'][:nPo], fixed=b['fixed'][:nPo], cam=b['cam'][:nPo], points=b['points'][:nL], edge_point=b['edge_point'][:nE],
                 edge_pose=b['edge_pose'][:nE], obs=b['obs'][:nE], inv_sigma2=b['inv_sigma2'][:nE], vert_kf=b['vert_kf'][:nPo],
                 vert_point=b['vert_point'][:nL], huber_delta=float(F32(np.sqrt(5.991))))
    return orb.local_ba_result(out), built


# ---- independent restatement ----
def _norm(v):
    return np.sqrt(F32(F32(F32(v[0] * v[0]) + F32(v[1] * v[1])) + F32(v[2] * v[2])))


def update_normal_and_depth(M, p):
    if p.bad or not p.obs:
        return
    n = np.zeros(3, F32)
    for k in sorted(p.obs):
        v = (p.pos - M.kfs[k].Ow).astype(F32)
        n = (n + (v / _norm(v)).astype(F32)).astype(F32)
    r = M.kfs[p.ref]
    p.normal = (n / F32(len(p.obs))).astype(F32)
    p.max_d = F32(_norm((p.pos - r.Ow).astype(F32)) * SF[r.octave[p.obs[p.ref]]])
    p.min_d = F32(p.max_d / SF[-1])


def restate(M, pkf, lm):
    """The whole function on model M (changed in place) with the optimiser's results lm = dict(pose {kf id: double [7]}, point {pt id: double
    [3]}, chi2 / dpos {(pt id, kf id): value}).  Returns the record in model ids: status, counts, the three lists, vToErase."""
    K, P = M.kfs, M.pts
    good = lambda k: not K[k].bad and not K[k].other
    marked = {pkf} | set(M.cov[pkf])
    local = [pkf] + [k for k in M.cov[pkf] if good(k)]
    pts, seen = [], set()
    for k in local:
        for p in K[k].mp:
            if p >= 0 and not P[p].bad and not P[p].other and p not in seen:
                seen.add(int(p)); pts.append(int(p))
    fixed, fseen = [], set()
    for p in pts:
        for k in sorted(P[p].obs):
            if k not in marked and k not in fseen:
                fseen.add(k)
                if good(k):
                    fixed.append(k)
    num_fixed = len(fixed) + int(any(K[k].init for k in local))
    rec = dict(local=local, fixed=fixed, points=pts, erase=[])
    if num_fixed == 0:
        return dict(rec, status=orb.LBA_LOCAL_NO_FIXED, counts=[0, 0, 0, 0])
    edges = [(p, k) for p in pts for k in sorted(P[p].obs) if good(k)]
    rec['counts'] = [num_fixed, len(local), len(pts), len(edges)]
    # the graph g2o sees: vertices by mnId, edges in insertion order with the observation and mvInvLevelSigma2[octave]
    verts = sorted(local + fixed, key=lambda k: K[k].mnId)
    rec['built'] = dict(vert_kf=verts, vert_point=sorted(pts, key=lambda p: P[p].mnId), edges=edges,
                        fixed=[k not in local or K[k].init for k in verts], poses=[K[k].Tcw.astype(np.float64) for k in verts],
                        points=[P[p].pos.astype(np.float64) for p in sorted(pts, key=lambda p: P[p].mnId)],
                        obs=[K[k].pt[P[p].obs[k]].astype(np.float64) for p, k in edges], inv_sigma2=[ISG[K[k].octave[P[p].obs[k]]] for p, k in edges],
                        cam=[K[k].cam for k in verts])
    if M.stop:
        return dict(rec, status=orb.LBA_LOCAL_STOPPED)
    rec['erase'] = [(p, k) for p, k in edges if lm['chi2'][(p, k)] > TH or not lm['dpos'][(p, k)]]
    for p, k in rec['erase']:
        M.erase_match(k, p)
        M.erase_observation(p, k)
    for k in local:
        K[k].Tcw = set_pose(lm['pose'][k])
        K[k].Ow = pose_matrices(K[k].Tcw)[2]
    for p in pts:
        P[p].pos = np.asarray(lm['point'][p], np.float64).astype(F32)
        update_normal_and_depth(M, P[p])
    return dict(rec, status=orb.LBA_LOCAL_RAN)


def lm_of(m, r):
    """The optimiser's results of a flattened map's record r (debug outputs) in model ids, for restate."""
    kid, pid = m['kf_ids'], m['pt_ids']
    lm = dict(pose={kid[k]: r['optPose'][i] for i, k in enumerate(r['localKF'])}, point={pid[p]: r['optPoint'][i] for i, p in enumerate(r['localPoint'])},
              chi2={}, dpos={})
    for p in range(len(pid)):
        for o in range(m['obsStart'][p], m['obsStart'][p + 1]):
            lm['chi2'][(pid[p], kid[m['obsKF'][o]])] = r['edgeChi2'][o]
            lm['dpos'][(pid[p], kid[m['obsKF'][o]])] = r['edgeDepthPositive'][o]
    return lm


def record_in_ids(m, r):
    """A call's record in model ids, comparable with restate's."""
    kid, pid = m['kf_ids'], m['pt_ids']
    erase = [(pid[p], kid[m['obsKF'][o]]) for p in r['localPoint'] for o in range(m['obsStart'][p], m['obsStart'][p + 1])
             if r['obsFlag'][o] == orb.LBA_OBS_ERASED]
    out = dict(status=r['status'], local=[kid[k] for k in r['localKF']], fixed=[kid[k] for k in r['fixedKF']], points=[pid[p] for p in r['localPoint']],
               erase=erase if r['status'] == orb.LBA_LOCAL_RAN else [])
    out['counts'] = [r['num_fixedKF'], r['num_OptKF'], r['num_MPs'], r['num_edges']]
    return out


def replay(M, m, r):
    """The shim's replay of a record onto model M: EraseMapPointMatch / EraseObservation in the returned order, SetPose, SetWorldPos and the
    point's normal and distances from the record."""
    if r['status'] != orb.LBA_LOCAL_RAN:
        return
    kid, pid = m['kf_ids'], m['pt_ids']
    for p, k in record_in_ids(m, r)['erase']:
        M.erase_match(k, p)
        M.erase_observation(p, k)
    for i, k in enumerate(r['localKF']):
        M.kfs[kid[k]].Tcw, M.kfs[kid[k]].Ow = r['kfPose7'][i].copy(), r['kfCenter'][i].copy()
    for i, p in enumerate(r['localPoint']):
        q = M.pts[pid[p]]
        q.pos = r['pointPos'][i].copy()
        assert q.bad == bool(r['pointBad'][i]) and q.ref == (kid[r['pointRefKF'][i]] if r['pointRefKF'][i] >= 0 else -1)
        if not q.bad:
            q.normal, q.min_d, q.max_d = r['normal'][i].copy(), F32(r['minDistance'][i]), F32(r['maxDistance'][i])


# ---- scenes ----
def scene(seed, n_kf=8, n_pts=300, obs_per_pt=4, n_cov=None, outlier_frac=0.05, inertial=False, slots_extra=5):
    """A map of n_kf keyframes on lba_scenes' arc; the last one is pKF, its covisibles the n_cov keyframes before it (newest first), the
    others are reached as observers.  Point j is seen by a window of obs_per_pt consecutive keyframes (real projections with noise and
    gross outliers, lba_scenes.make).  mnIds are a random permutation, not the id order."""
    rng = np.random.default_rng(seed)
    gt, cam = lba_scenes.keyframes(n_kf), lba_scenes.cameras(n_kf, seed + 1000)
    windows = lba_scenes._windows(n_kf, n_pts, obs_per_pt)
    p = lba_scenes.make(gt, cam, np.zeros(n_kf, np.uint8), windows, seed=seed, outlier_frac=outlier_frac)
    octave = np.searchsorted(-ISG, -p['inv_sigma2'])
    assert np.array_equal(ISG[octave], p['inv_sigma2'])
    M = Map(inertial)
    per_kf = [[] for _ in range(n_kf)]
    for e, (j, k) in enumerate(zip(p['edge_point'], p['edge_pose'])):
        per_kf[k].append((j, e))
    kf_mn = rng.permutation(n_kf) * 3 + 5
    for k in range(n_kf):
        rows = per_kf[k] + [(-1, -1)] * slots_extra
        order = rng.permutation(len(rows))
        rows = [rows[i] for i in order]
        pts = [p['obs'][e] if e >= 0 else (0.0, 0.0) for _, e in rows]
        octs = [octave[e] if e >= 0 else 0 for _, e in rows]
        M.kfs[k] = KeyFrame(k, int(kf_mn[k]), p['poses'][k], cam[k], pts, octs)
        for i, (j, e) in enumerate(rows):
            if j >= 0:
                M.kfs[k].mp[i] = j
    pt_mn = rng.permutation(n_pts) * 7 + 11
    for j in range(n_pts):
        M.pts[j] = MapPoint(j, int(pt_mn[j]), p['points'][j])
    for k in range(n_kf):
        for i, j in enumerate(M.kfs[k].mp):
            if j >= 0:
                M.pts[j].obs[k] = i
                M.pts[j].nObs += 1
    for j, q in M.pts.items():
        q.ref = sorted(q.obs)[len(q.obs) // 2]
    pkf = n_kf - 1
    n_cov = n_kf // 2 if n_cov is None else n_cov
    M.cov[pkf] = list(range(pkf - 1, pkf - 1 - n_cov, -1))
    return M, pkf


def plant_outliers(M, pid, kids, px=40.0):
    """Gross outliers: move the keypoints of point pid in keyframes kids by px pixels."""
    for i, k in enumerate(kids):                    # alternate up and down: no point position explains them
        M.kfs[k].pt[M.pts[pid].obs[k]] += np.array([0, px if i % 2 else -px], F32)


def planted():
    """Named maps, each with the branch it plants."""
    out = {}
    M, k = scene(1, n_kf=10, n_pts=200, obs_per_pt=4, n_cov=5)
    cov = M.cov[k]
    M.kfs[cov[4]].bad = True                        # a bad covisible
    M.kfs[cov[3]].other = True                      # an other-map covisible
    slot_pts = [int(p) for p in M.kfs[k].mp if p >= 0]
    M.pts[slot_pts[0]].bad = True                   # bad and other-map points in local slots
    M.pts[slot_pts[1]].other = True
    M.kfs[2].bad = True                             # bad and other-map observers (fixed-camera candidates the walk reaches)
    M.kfs[1].other = True
    hub = [q for q in slot_pts[2:] if len(M.pts[q].obs) >= 4 and all(not M.kfs[kk].bad and not M.kfs[kk].other for kk in M.pts[q].obs)][:3]
    p0 = hub[0]                                     # an erase that moves mpRefKF
    plant_outliers(M, p0, [M.pts[p0].ref])
    p1 = hub[1]                                     # nObs to 2, then a later erase of the same point
    ks = sorted(M.pts[p1].obs)
    M.pts[p1].ref = ks[0]
    plant_outliers(M, p1, ks[1:], px=120.0)
    out['mixed'] = (M, k)
    M, k = scene(2, n_kf=8, n_pts=150, obs_per_pt=3, n_cov=7)
    M.kfs[3].init = True                            # the init keyframe among the local ones, and it is the only fixed one
    out['init_only'] = (M, k)
    M, k = scene(3, n_kf=6, n_pts=60, obs_per_pt=2, n_cov=5)
    out['no_fixed'] = (M, k)                        # every observer is local and none is the init keyframe
    M, k = scene(4, n_kf=8, n_pts=120, obs_per_pt=4, n_cov=3)
    M.stop = True
    out['stopped'] = (M, k)
    M, k = scene(5, n_kf=8, n_pts=200, obs_per_pt=4, n_cov=3, inertial=True)
    out['inertial'] = (M, k)
    M, k = scene(6, n_kf=12, n_pts=200, obs_per_pt=3, n_cov=2)
    far = 0                                         # a fixed camera reached by many points
    for j, q in M.pts.items():
        if far not in q.obs and len(q.obs) and j % 3 == 0:
            i = len(M.kfs[far].mp)
            M.kfs[far].mp = np.append(M.kfs[far].mp, j)
            M.kfs[far].pt = np.vstack([M.kfs[far].pt, M.kfs[far].pt[:1]])
            M.kfs[far].octave = np.append(M.kfs[far].octave, 0)
            q.obs[far] = i
            q.nObs += 1
    out['hub_fixed'] = (M, k)
    return out


def check_margin(r, margin=1e-3):
    """No chi2 of an edge lies within margin of 5.991, so that the outlier test cannot flip between two solvers that agree to rounding."""
    chi2 = r['edgeChi2'][r['obsFlag'] != orb.LBA_OBS_NO_EDGE]
    assert not (np.abs(chi2 - TH) < margin).any(), 'a chi2 lies within %g of 5.991' % margin


def copy_map(M):
    return copy.deepcopy(M)
