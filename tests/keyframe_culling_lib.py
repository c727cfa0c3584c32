"""LocalMapping::KeyFrameCulling() (src/LocalMapping.cc; monocular and mono-inertial) over a small map model (test infrastructure):
- the map model: search_in_neighbors_lib's KeyFrame (mvpMapPoints as point ids, keypoint octaves) and MapPoint (observations
  {keyframe id: keypoint index}, nObs, bad), plus the keyframe fields the loop reads (mnId, init, mbNotErase, prev / next, timestamp,
  IMU position) and the map's scalars;
- `flatten`: the OrbmCullingMap arrays of a model (keyframe table = the model's keyframes, points = its points);
- `oracle`: orbo_keyframe_culling (oracle/keyframe_culling_oracle.cpp) on the flattened map, with its final state;
- `restate`: an independent Python restatement of the loop on a copy of the model; static=True evaluates every keyframe against the
  call-start state (not the reference: it shows that the sequential rule matters);
- `replay`: the host side of the GPU call, applying the statuses in order to a copy of the model (MergePrevious logged, relink,
  SetBadFlag);
- `corridor`: the seeded scene generator, a corridor of keyframes whose points are each seen by a window of consecutive keyframes."""
import copy
import ctypes as C

import numpy as np

import oracle_lib as O
from search_in_neighbors_lib import KeyFrame, MapPoint
import orb_slam3_modified_b200 as orb
from orb_slam3_modified_b200 import KP_DTYPE, KF_BAD, KF_INIT, KF_NOT_ERASE

ND = 21
F32 = np.float32
TO_BE_ERASED = 8
NOT_VISITED, SKIPPED, KEPT, KEPT_FEW_KFS, KEPT_RECENT, KEPT_NO_LINK, KEPT_IMU, CULLED, CULLED_TIME, CULLED_STILL, NOT_ERASE = range(11)
ERASING = (CULLED, CULLED_TIME, CULLED_STILL, NOT_ERASE)        # statuses whose keyframe got SetBadFlag
CONTINUES = (SKIPPED, KEPT_FEW_KFS, KEPT_RECENT)                # statuses whose path skips the break test


# ---- map model ----
def new_keyframe(kid, octaves, mnId=None):
    kps = np.zeros(len(octaves), KP_DTYPE)
    kps['octave'] = octaves
    kf = KeyFrame(kid, kps, np.zeros((len(octaves), 32), np.uint8), np.zeros(7, F32), np.zeros(3, F32))
    kf.mnId = kid if mnId is None else mnId
    kf.init = kf.not_erase = kf.to_be_erased = False
    kf.prev = kf.next = None                          # keyframe ids
    kf.ts, kf.pos = 0.0, np.zeros(3, F32)
    return kf


class CullingMap:
    """A map: keyframes (id = index), points (id = index), the local keyframes in GetVectorCovisibleKeyFrames() order and the scalars."""
    def __init__(self, inertial=False):
        self.kfs, self.pts, self.local = [], [], []
        self.inertial, self.imu_init, self.ba2, self.abort = inertial, False, False, False
        self.kf_in_map, self.current_id, self.last_id = 0, 0, 0
        self.merges = []                              # (next, culled): mNextKF->mpImuPreintegrated->MergePrevious(culled's)

    def add_point(self, obs, bad=False):
        p = MapPoint(len(self.pts), np.zeros(3, F32), np.zeros(32, np.uint8))
        for kid, idx in obs:
            p.AddObservation(self.kfs[kid], idx)
            self.kfs[kid].mp[idx] = p.id
        p.bad = bad
        self.pts.append(p)
        return p

    def octave(self, kid, idx):
        return int(self.kfs[kid].kps['octave'][idx])

    # MapPoint::SetBadFlag / EraseObservation, KeyFrame::SetBadFlag
    def point_set_bad(self, p):
        p.bad = True
        obs, p.obs = p.obs, {}
        for kid, idx in obs.items():
            self.kfs[kid].mp[idx] = -1

    def erase_observation(self, p, kf):
        if kf.id in p.obs:
            p.nObs -= 1
            del p.obs[kf.id]
            if p.nObs <= 2:
                self.point_set_bad(p)

    def kf_set_bad(self, kf):
        if kf.init:
            return
        if kf.not_erase:
            kf.to_be_erased = True
            return
        for pid in kf.mp:
            if pid >= 0:
                self.erase_observation(self.pts[pid], kf)
        kf.bad = True
        self.kf_in_map -= 1

    def unlink(self, kf):
        """The inertial cull's MergePrevious (logged) and relink."""
        nxt, prv = self.kfs[kf.next], self.kfs[kf.prev]
        self.merges.append((nxt.id, kf.id))
        nxt.prev, prv.next = prv.id, nxt.id
        kf.prev = kf.next = None

    def state(self):
        """The final state in the oracle's terms: kfFlags (with TO_BE_ERASED), prev, next, pointBad, nObs, KeyFramesInMap."""
        flags = np.array([(KF_BAD if k.bad else 0) | (KF_INIT if k.init else 0) | (KF_NOT_ERASE if k.not_erase else 0) |
                          (TO_BE_ERASED if k.to_be_erased else 0) for k in self.kfs], np.uint8)
        link = lambda v: -1 if v is None else v                     # noqa: E731
        prev = np.array([link(k.prev) for k in self.kfs], np.int32) if self.inertial else None
        nxt = np.array([link(k.next) for k in self.kfs], np.int32) if self.inertial else None
        return dict(kfFlags=flags, prev=prev, next=nxt, pointBad=np.array([p.bad for p in self.pts], np.uint8),
                    nObs=np.array([p.nObs for p in self.pts], np.int32), kfInMap=self.kf_in_map)


def flatten(cm):
    """The OrbmCullingMap arrays and scalars of a model (ORBmatcher.keyframe_culling_batch's map dict)."""
    slot_start, slot_point, slot_oct = [0], [], []
    for kid in cm.local:
        kf = cm.kfs[kid]
        for i in np.nonzero(kf.mp >= 0)[0]:
            slot_point.append(int(kf.mp[i])); slot_oct.append(int(kf.kps['octave'][i]))
        slot_start.append(len(slot_point))
    obs_start, obs_kf, obs_oct = [0], [], []
    for p in cm.pts:
        for kid, idx in sorted(p.obs.items()):
            obs_kf.append(kid); obs_oct.append(cm.octave(kid, idx))
        obs_start.append(len(obs_kf))
    link = lambda v: -1 if v is None else v                         # noqa: E731
    m = dict(mnId=np.array([k.mnId for k in cm.kfs], np.uint64),
             kfFlags=np.array([(KF_BAD if k.bad else 0) | (KF_INIT if k.init else 0) | (KF_NOT_ERASE if k.not_erase else 0) for k in cm.kfs], np.uint8),
             local=np.array(cm.local, np.int32), slotStart=np.array(slot_start, np.int32), slotPoint=np.array(slot_point, np.int32),
             slotOctave=np.array(slot_oct, np.int32), pointBad=np.array([p.bad for p in cm.pts], np.uint8), obsStart=np.array(obs_start, np.int32),
             obsKF=np.array(obs_kf, np.int32), obsOctave=np.array(obs_oct, np.int32),
             inertial=int(cm.inertial), imuInitialized=int(cm.imu_init), inertialBA2=int(cm.ba2), abortBA=int(cm.abort),
             keyFramesInMap=cm.kf_in_map, currentId=cm.current_id, lastId=cm.last_id)
    if cm.inertial:
        m.update(prevKF=np.array([link(k.prev) for k in cm.kfs], np.int32), nextKF=np.array([link(k.next) for k in cm.kfs], np.int32),
                 timeStamp=np.array([k.ts for k in cm.kfs], np.float64), imuPosition=np.array([k.pos for k in cm.kfs], np.float32).reshape(-1, 3))
    return m


# ---- the oracle ----
def oracle(m):
    """orbo_keyframe_culling on map dict `m`: (result dict(status, nMPs, nRedundant, visited), final state as CullingMap.state())."""
    L = O.lib()
    s, out, keep = orb.culling_struct(m)
    nK, nP = s.nKF, s.nPoints
    flags, prev, nxt = np.zeros(nK, np.uint8), np.zeros(nK, np.int32), np.zeros(nK, np.int32)
    bad, nobs, kin = np.zeros(nP, np.uint8), np.zeros(nP, np.int32), C.c_int(0)
    L.orbo_keyframe_culling.argtypes = [C.c_void_p] * 7
    L.orbo_keyframe_culling(C.byref(s), flags.ctypes.data, prev.ctypes.data, nxt.ctypes.data, bad.ctypes.data, nobs.ctypes.data, C.byref(kin))
    res = dict(out, visited=int(out['visited'][0]))
    inertial = bool(m['inertial'])
    return res, dict(kfFlags=flags, prev=prev if inertial else None, next=nxt if inertial else None, pointBad=bad, nObs=nobs, kfInMap=kin.value)


# ---- the Python restatement ----
def _decide(cm, kf, mps, red):
    """The decision after the counts, on the live model: (status, erase?, falls through to the break test?)."""
    if not np.float32(red) > np.float32(0.9) * np.float32(mps):
        return KEPT, False, True
    if not cm.inertial:
        return CULLED, True, True
    if cm.kf_in_map <= ND:
        return KEPT_FEW_KFS, False, False
    if kf.mnId > (cm.current_id - 2) % 2 ** 64:
        return KEPT_RECENT, False, False
    if kf.prev is None or kf.next is None:
        return KEPT_NO_LINK, False, True
    t = np.float32(np.float64(cm.kfs[kf.next].ts) - np.float64(cm.kfs[kf.prev].ts))
    if (cm.imu_init and kf.mnId < cm.last_id and t < 3) or t < 0.5:
        return CULLED_TIME, True, True
    d = (np.asarray(kf.pos, F32) - np.asarray(cm.kfs[kf.prev].pos, F32)).astype(F32)
    sq = np.float32(np.float32(np.float32(d[0] * d[0]) + np.float32(d[1] * d[1])) + np.float32(d[2] * d[2]))
    if not cm.ba2 and np.float64(np.sqrt(sq)) < 0.02 and t < 3:
        return CULLED_STILL, True, True
    return KEPT_IMU, False, True


def _counts(cm, kf, view):
    """nMPs and nRedundantObservations of keyframe kf; `view` gives (bad, nObs, observations) of a point."""
    mps = red = 0
    for i in np.nonzero(kf.mp >= 0)[0]:
        bad, nobs, obs = view(cm.pts[int(kf.mp[i])])
        if bad:
            continue
        mps += 1
        if nobs > 3:
            lvl = int(kf.kps['octave'][i])
            red += sum(1 for kid, idx in obs.items() if kid != kf.id and cm.octave(kid, idx) <= lvl + 1) > 3
    return mps, red


def restate(cm, static=False):
    """The loop on a copy of the model: (result dict(status, nMPs, nRedundant, visited), final state, merges).  static=True counts every
    keyframe against the call-start state of the points (bad flags, nObs and observations) instead of the live one."""
    cm = copy.deepcopy(cm)
    start = {p.id: (p.bad, p.nObs, dict(p.obs)) for p in cm.pts}
    slots = {k.id: k.mp.copy() for k in cm.kfs}
    n = len(cm.local)
    st, nmps, nred = np.zeros(n, np.uint8), np.full(n, -1, np.int32), np.full(n, -1, np.int32)
    count = 0
    for li, kid in enumerate(cm.local):
        count += 1
        kf = cm.kfs[kid]
        if kf.init or kf.bad:
            st[li] = SKIPPED
            continue
        if static:
            live = kf.mp
            kf.mp = slots[kid]
            mps, red = _counts(cm, kf, lambda p: start[p.id])
            kf.mp = live
        else:
            mps, red = _counts(cm, kf, lambda p: (p.bad, p.nObs, p.obs))
        nmps[li], nred[li] = mps, red
        s, erase, through = _decide(cm, kf, mps, red)
        if erase:
            if cm.inertial:
                cm.unlink(kf)
            if kf.not_erase:
                s = NOT_ERASE
            cm.kf_set_bad(kf)
        st[li] = s
        if through and ((count > 20 and cm.abort) or count > 100):
            break
    return dict(status=st, nMPs=nmps, nRedundant=nred, visited=count), cm.state(), cm.merges


def replay(cm, res):
    """What a host shim does with the GPU call's result: the culls in status order on a copy of the model.  Returns (state, merges)."""
    cm = copy.deepcopy(cm)
    for li, kid in enumerate(cm.local[:res['visited']]):
        s = int(res['status'][li])
        if s in ERASING:
            kf = cm.kfs[kid]
            if cm.inertial:
                cm.unlink(kf)
            cm.kf_set_bad(kf)
    return cm.state(), cm.merges


def same_state(a, b):
    return all((a[k] is None and b[k] is None) or np.array_equal(a[k], b[k]) for k in ('kfFlags', 'prev', 'next', 'pointBad', 'nObs')) and \
        a['kfInMap'] == b['kfInMap']


def same_result(a, b):
    return all(np.array_equal(a[k], b[k]) for k in ('status', 'nMPs', 'nRedundant')) and a['visited'] == b['visited']


# ---- seeded scenes ----
def corridor(seed, n_kf=40, n_local=None, n_kp=320, new_per_kf=10, window=(6, 16), p_low=0.7, inertial=False, n_bad_kf=1, n_not_erase=1,
             p_bad_point=0.02, order='newest', id_base=0, kf_extra=0, dt=(0.05, 0.6), p_still=0.25, imu_init=True, ba2=False, abort=False):
    """A corridor of n_kf keyframes (the last is the current keyframe; keyframe 0 is the map's init keyframe).  Keyframe j creates
    new_per_kf points, each seen by keyframes j .. j + w - 1 (w drawn from `window`, clipped at the corridor's end) at a free keypoint.
    Keypoint octaves are drawn geometrically (P(0) = p_low); with the defaults about half of the keyframes are redundant.
    The local keyframes are the n_local keyframes before the current one, newest first ('newest') or shuffled.  n_bad_kf keyframes are
    bad (their observations erased as SetBadFlag would), n_not_erase have mbNotErase, a share of points is bad.  Inertial: links along
    the corridor, timestamps with steps drawn from `dt`, IMU positions with a still step (< 0.02) with probability p_still."""
    rng = np.random.default_rng(seed)
    cm = CullingMap(inertial)
    for j in range(n_kf):
        oct_ = np.minimum(rng.geometric(p_low, n_kp) - 1, 7)
        cm.kfs.append(new_keyframe(j, oct_, id_base + j))
    free = [list(rng.permutation(n_kp)) for _ in range(n_kf)]
    for j in range(n_kf):
        for _ in range(new_per_kf):
            w = int(rng.integers(window[0], window[1] + 1))
            obs = [(k, free[k].pop()) for k in range(j, min(j + w, n_kf)) if free[k]]
            if len(obs) >= 2:
                cm.add_point(obs)
    cm.kfs[0].init = True
    n_local = n_kf - 1 if n_local is None else n_local
    cand = list(range(n_kf - 2, n_kf - 2 - n_local, -1))
    cm.local = cand if order == 'newest' else [int(x) for x in rng.permutation(cand)]
    inner = [k for k in range(1, n_kf - 1)]
    for k in rng.choice(inner, n_bad_kf, replace=False) if n_bad_kf else []:
        cm.kf_set_bad(cm.kfs[int(k)])
    for k in rng.choice(inner, n_not_erase, replace=False) if n_not_erase else []:
        cm.kfs[int(k)].not_erase = True
    for p in cm.pts:
        if not p.bad and rng.random() < p_bad_point:
            p.bad, p.obs = True, {}                   # bad, but still in its keyframes' slots (isBad() is what the loop tests)
    for p in cm.pts:
        p.nObs = len(p.obs)                           # Observations() as the flattened map gives it
    cm.kf_in_map = n_kf + kf_extra
    cm.kf_in_map -= sum(k.bad for k in cm.kfs)
    cm.current_id = cm.kfs[-1].mnId
    if inertial:
        ts = 0.0
        pos = np.zeros(3)
        for j, kf in enumerate(cm.kfs):
            kf.prev = j - 1 if j else None
            kf.next = j + 1 if j + 1 < n_kf else None
            kf.ts = ts
            kf.pos = pos.astype(F32)
            ts += float(rng.uniform(*dt))
            step = rng.normal(0, 1, 3)
            pos = pos + step / np.linalg.norm(step) * (rng.uniform(0.001, 0.015) if rng.random() < p_still else rng.uniform(0.03, 0.3))
        for kf in cm.kfs:
            if kf.bad:                                # culled earlier: unlinked by its own cull
                if kf.prev is not None and kf.next is not None:
                    cm.kfs[kf.prev].next, cm.kfs[kf.next].prev = kf.next, kf.prev
                kf.prev = kf.next = None
        aux = cm.kfs[-1]
        for _ in range(ND):
            if aux.prev is None:
                break
            aux = cm.kfs[aux.prev]
        cm.last_id = aux.mnId
        cm.imu_init, cm.ba2 = imu_init, ba2
    cm.abort = abort
    return cm


def dense(n_kf, n_pts=10, inertial=False, kf_in_map=100):
    """n_kf keyframes that all see the same n_pts points at octave 0 (keyframe 0 the init keyframe, the last the current one); the local
    keyframes are all the others, newest first.  Every keyframe stays redundant while more than four observers remain.  Inertial: links
    in id order, timestamps 0.2 s apart (so t = 0.4 < 0.5 culls by time), IMU positions 1 m apart."""
    cm = CullingMap(inertial)
    for j in range(n_kf):
        cm.kfs.append(new_keyframe(j, np.zeros(n_pts, np.int32)))
    for i in range(n_pts):
        cm.add_point([(k, i) for k in range(n_kf)])
    cm.kfs[0].init = True
    cm.local = list(range(n_kf - 2, 0, -1))
    cm.kf_in_map, cm.current_id = kf_in_map, n_kf - 1
    if inertial:
        for j, kf in enumerate(cm.kfs):
            kf.prev, kf.next = (j - 1 if j else None), (j + 1 if j + 1 < n_kf else None)
            kf.ts, kf.pos = 0.2 * j, np.array([j, 0, 0], F32)
        cm.last_id = max(0, n_kf - 1 - ND)
    return cm


def cascade():
    """Local keyframes A (1) then B (2).  A: 19 redundant points and P; B: 9 redundant points and P.  P is seen by A, B and keyframe 3
    only.  At the call start B has 9 redundant of 10 (9 > 0.9f * 10 is false); culling A drops P to two observations, P becomes bad, and
    B has 9 of 9."""
    cm = CullingMap()
    for j in range(8):
        cm.kfs.append(new_keyframe(j, np.zeros(24, np.int32)))
    cm.kfs[0].init = True
    for i in range(19):
        cm.add_point([(1, i)] + [(k, i) for k in (3, 4, 5, 6, 7)] + ([(2, i)] if i < 9 else []))
    cm.add_point([(1, 20), (2, 20), (3, 20)])
    cm.local, cm.kf_in_map, cm.current_id = [1, 2], 8, 7
    return cm



def boundary(n, nr):
    """One local keyframe with n points, nr of them redundant (four other observers at octave 0), the rest seen by one other keyframe."""
    cm = CullingMap()
    for j in range(6):
        cm.kfs.append(new_keyframe(j, np.zeros(n, np.int32)))
    for i in range(n):
        cm.add_point([(1, i)] + ([(k, i) for k in (2, 3, 4, 5)] if i < nr else [(2, i)]))
    cm.local, cm.kf_in_map, cm.current_id = [1], 6, 5
    return cm



def one_inertial(dt_pair, gap=1.0, imu_init=False, ba2=False, mnid_below_last=True):
    """A dense inertial map whose only local keyframe is 5: t = ts[6] - ts[4] = dt_pair, |p5 - p4| = gap."""
    cm = dense(30, inertial=True)
    cm.local = [5]
    cm.kfs[6].ts = cm.kfs[4].ts + dt_pair
    cm.kfs[5].pos = (cm.kfs[4].pos.astype(np.float64) + np.array([gap, 0, 0])).astype(F32)
    cm.imu_init, cm.ba2 = imu_init, ba2
    cm.last_id = 10 if mnid_below_last else 3
    return cm

