"""LocalMapping::ProcessNewKeyFrame's map-point loop and the tail of SearchInNeighbors, each followed by KeyFrame::UpdateConnections
(src/LocalMapping.cc, src/KeyFrame.cc, src/MapPoint.cc; monocular observations), over a small map model (test infrastructure):
- the model: `Scene` holds a keyframe table (entry 0 the current keyframe) and points; every keyframe has a std::map key `order`, mnId,
  flags, its camera centre, keypoint octaves and descriptor rows, mConnectedKeyFrameWeights and (once known) its ordered list;
- `flatten`: the OrbmConnectionsItem arrays of a scene;
- `oracle`: orbo_update_connections (oracle/update_connections_oracle.cpp) on the flattened item, with its final map;
- `restate`: an independent Python restatement of the outputs; sum_order='mnId' sums the normals in mnId order and new_row='end' puts the
  new observation's descriptor row last (neither is the reference: they show that the key order is exercised);
- `replay`: the host side of the GPU call, applying the outputs to a copy of the scene;
- `scene`: the seeded scene generator (key orders shuffled against mnId), `from_search_in_neighbors`: a SearchInNeighbors job as a scene;
- `planted`: hand-made scenes, one per rule the tests pin."""
import copy
import ctypes as C

import numpy as np

import oracle_lib as O
import orb_slam3_modified_b200 as orb
from orb_slam3_modified_b200 import KF_BAD, KF_INIT, KF_OTHER_MAP, UC_PROCESS_NEW_KEYFRAME as PNK, UC_SEARCH_IN_NEIGHBORS as SIN

F32 = np.float32
TH = 15
NONE, ADDED, IN_KF, UPDATED = range(4)
OUT_KEYS = tuple(n for n, _ in orb.CONNECTIONS_OUTPUTS)


# ---- model ----
class KeyFrame:
    def __init__(self, t, order, mnId, Ow, octaves, desc):
        self.t, self.order, self.mnId = t, int(order), int(mnId)
        self.Ow = np.asarray(Ow, F32)
        self.oct, self.desc = np.asarray(octaves, np.int32), np.asarray(desc, np.uint8)
        self.bad = self.other = self.init = False
        self.conn = {}                       # mConnectedKeyFrameWeights: table index -> weight
        self.ordered = None                  # [(table index, weight)] once this call set it; None = the caller's list
        self.first, self.parent, self.children = False, None, []
        self.mp = np.full(len(octaves), -1, np.int64)    # the current keyframe's slots (point ids)


class MapPoint:
    def __init__(self, pid, pos, ref):
        self.id, self.pos, self.ref = pid, np.asarray(pos, F32), ref
        self.obs = {}                        # table index -> keypoint index
        self.bad = False
        self.normal, self.min_d, self.max_d, self.desc = None, None, None, None   # desc: (table index, keypoint index)


class Scene:
    def __init__(self, mode, sf):
        self.mode, self.sf, self.kfs, self.pts, self.recent = mode, np.asarray(sf, F32), [], [], []

    def add_kf(self, order, mnId, Ow, octaves, desc, bad=False, other=False):
        kf = KeyFrame(len(self.kfs), order, mnId, Ow, octaves, desc)
        kf.bad, kf.other = bad, other
        self.kfs.append(kf)
        return kf

    def add_point(self, pos, obs, ref=None, bad=False):
        p = MapPoint(len(self.pts), pos, None)
        for t, idx in obs:
            p.obs[t] = int(idx)
        p.ref = (min(p.obs, key=lambda t: self.kfs[t].order) if p.obs else 0) if ref is None else ref
        p.bad = bad
        self.pts.append(p)
        return p

    def key_sorted(self, ts, by='order'):
        return sorted(ts, key=lambda t: getattr(self.kfs[t], by))


def flatten(sc):
    """The OrbmConnectionsItem arrays and scalars of a scene (ORBmatcher.update_connections_batch's item dict)."""
    kfs, cur = sc.kfs, sc.kfs[0]
    conn_start, conn_kf, conn_w = [0], [], []
    for kf in kfs:
        for t in sc.key_sorted(kf.conn):
            conn_kf.append(t); conn_w.append(kf.conn[t])
        conn_start.append(len(conn_kf))
    obs_start, okf, oidx, ooct, odesc = [0], [], [], [], []
    for p in sc.pts:
        for t in sc.key_sorted(p.obs):
            i = p.obs[t]
            okf.append(t); oidx.append(i); ooct.append(int(kfs[t].oct[i])); odesc.append(kfs[t].desc[i])
        obs_start.append(len(okf))
    flags = [(KF_BAD if k.bad else 0) | (KF_OTHER_MAP if k.other else 0) | (KF_INIT if k.init and k.t == 0 else 0) for k in kfs]
    return dict(mode=sc.mode, firstConnection=int(cur.first),
                order=np.array([k.order for k in kfs], np.uint64), mnId=np.array([k.mnId for k in kfs], np.uint64), kfFlags=np.array(flags, np.uint8),
                cameraCenter=np.array([k.Ow for k in kfs], F32).reshape(-1, 3), connStart=np.array(conn_start, np.int32),
                connKF=np.array(conn_kf, np.int32), connWeight=np.array(conn_w, np.int32), scaleFactors=sc.sf,
                slotPoint=cur.mp.astype(np.int32), slotOctave=cur.oct, slotDesc=cur.desc.reshape(-1, 32),
                pointBad=np.array([p.bad for p in sc.pts], np.uint8), pointPos=np.array([p.pos for p in sc.pts], F32).reshape(-1, 3),
                pointRefKF=np.array([p.ref for p in sc.pts], np.int32), obsStart=np.array(obs_start, np.int32), obsKF=np.array(okf, np.int32),
                obsIdx=np.array(oidx, np.int32), obsOctave=np.array(ooct, np.int32), obsDesc=np.array(odesc, np.uint8).reshape(-1, 32))


# ---- the oracle ----
class _Final(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ('obsStart', 'obsKF', 'obsIdx', 'connStart', 'connKF', 'connWeight', 'recent', 'nRecent', 'firstConnection')]


def oracle(m):
    """orbo_update_connections on item dict `m`: (outputs as ORBmatcher.update_connections_batch returns them, final map dict)."""
    s, out, keep = orb.connections_struct(m)
    nK, nP, nS = s.nKF, s.nPoints, s.nSlots
    nO, nC = int(keep['obsStart'][-1]) if nP else 0, int(keep['connStart'][-1])
    fin = dict(obsStart=np.zeros(nP + 1, np.int32), obsKF=np.zeros(nO + nP, np.int32), obsIdx=np.zeros(nO + nP, np.int32),
               connStart=np.zeros(nK + 1, np.int32), connKF=np.zeros(nC + 2 * nK, np.int32), connWeight=np.zeros(nC + 2 * nK, np.int32),
               recent=np.zeros(max(nS, 1), np.int32), nRecent=np.zeros(1, np.int32), firstConnection=np.zeros(1, np.int32))
    f = _Final(*[fin[n].ctypes.data for n, _ in _Final._fields_])
    L = O.lib()
    L.orbo_update_connections.argtypes = [C.c_void_p, C.c_void_p]
    L.orbo_update_connections(C.byref(s), C.byref(f))
    return orb._connections_result(out), _final_dict(fin)


def _final_dict(fin):
    n, c = fin['obsStart'], fin['connStart']
    return dict(obs=[list(zip(fin['obsKF'][n[p]:n[p + 1]].tolist(), fin['obsIdx'][n[p]:n[p + 1]].tolist())) for p in range(len(n) - 1)],
                conn=[list(zip(fin['connKF'][c[k]:c[k + 1]].tolist(), fin['connWeight'][c[k]:c[k + 1]].tolist())) for k in range(len(c) - 1)],
                recent=fin['recent'][:fin['nRecent'][0]].tolist(), firstConnection=int(fin['firstConnection'][0]))


def final_state(sc):
    """The scene in the oracle's final-map terms."""
    return dict(obs=[[(t, p.obs[t]) for t in sc.key_sorted(p.obs)] for p in sc.pts],
                conn=[[(t, k.conn[t]) for t in sc.key_sorted(k.conn)] for k in sc.kfs], recent=list(sc.recent), firstConnection=int(sc.kfs[0].first))


# ---- the Python restatement ----
def _popcount_matrix(rows):
    x = rows[:, None, :] ^ rows[None, :, :]
    return np.unpackbits(x, axis=2).sum(axis=2)


def distinctive(rows):
    """Index of the first row with the least median distance (element int(0.5 (n - 1)) of its sorted distances, 0 to itself)."""
    D = _popcount_matrix(np.asarray(rows, np.uint8))
    med = np.sort(D, axis=1)[:, int(0.5 * (len(rows) - 1))]
    return int(np.argmin(med))


def _norm(v):
    return np.sqrt(F32(F32(F32(v[0] * v[0]) + F32(v[1] * v[1])) + F32(v[2] * v[2])))


def _update_point(sc, p, obs, new_t, sum_order, new_row):
    """(normal, min, max, desc) of point p with observations obs {t: idx}; new_t is the observation this call adds (or None)."""
    n = np.zeros(3, F32)
    for t in sc.key_sorted(obs, sum_order):
        v = (p.pos - sc.kfs[t].Ow).astype(F32)
        d = _norm(v)
        n = (n + (v / d).astype(F32)).astype(F32)
    normal = (n / F32(len(obs))).astype(F32)
    ref = sc.kfs[p.ref]
    dist = _norm((p.pos - ref.Ow).astype(F32))
    dmax = F32(dist * sc.sf[ref.oct[obs[p.ref]]])
    dmin = F32(dmax / sc.sf[-1])
    who = [t for t in sc.key_sorted(obs) if not sc.kfs[t].bad]
    if new_row == 'end' and new_t in who:
        who.remove(new_t); who.append(new_t)
    desc = None
    if who:
        b = who[distinctive(np.stack([sc.kfs[t].desc[obs[t]] for t in who]))]
        desc = (b, obs[b])
    return normal, dmin, dmax, desc


def _empty_outputs(sc):
    nK, nP = len(sc.kfs), len(sc.pts)
    nN = sum(len(k.conn) for k in sc.kfs) + nK
    return dict(slotStatus=np.zeros(len(sc.kfs[0].mp), np.uint8), pointUpdated=np.zeros(nP, np.uint8), normal=np.zeros((nP, 3), F32),
                minDistance=np.zeros(nP, F32), maxDistance=np.zeros(nP, F32), descKF=np.full(nP, -1, np.int32), descIdx=np.full(nP, -1, np.int32),
                counter=np.zeros(nK, np.int32), nConnected=-1, orderedKF=np.full(nK, -1, np.int32), orderedWeight=np.zeros(nK, np.int32), parent=-1,
                nbrCount=np.full(nK, -1, np.int32), nbrKF=np.full(nN, -1, np.int32), nbrWeight=np.zeros(nN, np.int32))


def restate(sc, sum_order='order', new_row='key'):
    """The outputs of the call on scene `sc`, restated in Python."""
    out = _empty_outputs(sc)
    kfs, cur = sc.kfs, sc.kfs[0]
    obs = {p.id: dict(p.obs) for p in sc.pts}
    for i, pid in enumerate(cur.mp):
        if pid < 0 or sc.pts[pid].bad:
            continue
        p = sc.pts[pid]
        new_t = None
        if sc.mode == PNK:
            if 0 in obs[pid]:
                out['slotStatus'][i] = IN_KF
                continue
            obs[pid][0] = i
            new_t = 0
            out['slotStatus'][i] = ADDED
        else:
            out['slotStatus'][i] = UPDATED
        normal, dmin, dmax, desc = _update_point(sc, p, obs[pid], new_t, sum_order, new_row)
        out['pointUpdated'][pid] = 1
        out['normal'][pid], out['minDistance'][pid], out['maxDistance'][pid] = normal, dmin, dmax
        if desc is not None:
            out['descKF'][pid], out['descIdx'][pid] = desc
    # UpdateConnections
    cnt = {}
    for pid in cur.mp:
        if pid < 0 or sc.pts[pid].bad:
            continue
        for t in obs[pid]:
            k = kfs[t]
            if k.mnId == cur.mnId or k.bad or k.other:
                continue
            cnt[t] = cnt.get(t, 0) + 1
    if not cnt:
        return out
    for t, c in cnt.items():
        out['counter'][t] = c
    keyed = sc.key_sorted(cnt)
    nmax = max(cnt.values())
    kmax = next(t for t in keyed if cnt[t] == nmax)
    pairs = [t for t in keyed if cnt[t] >= TH] or [kmax]
    nbr_off = np.cumsum([0] + [len(k.conn) + 1 for k in kfs])
    for t in pairs:
        k, w = kfs[t], cnt[t]
        if k.conn.get(0) == w:
            continue
        new = dict(k.conn)
        new[0] = w
        lst = sorted(((w2, kfs[t2].order, t2) for t2, w2 in new.items() if not kfs[t2].bad), reverse=True)
        out['nbrCount'][t] = len(lst)
        for r, (w2, _, t2) in enumerate(lst):
            out['nbrKF'][nbr_off[t] + r], out['nbrWeight'][nbr_off[t] + r] = t2, w2
    ordered = sorted(((cnt[t], kfs[t].order, t) for t in pairs), reverse=True)
    out['nConnected'] = len(ordered)
    for r, (w, _, t) in enumerate(ordered):
        out['orderedKF'][r], out['orderedWeight'][r] = t, w
    if cur.first and not cur.init:
        out['parent'] = ordered[0][2]
    return out


# ---- the host replay ----
def replay(sc, out):
    """What a host shim does with the call's outputs, on a copy of the scene."""
    sc = copy.deepcopy(sc)
    kfs, cur = sc.kfs, sc.kfs[0]
    for i, st in enumerate(out['slotStatus']):
        pid = int(cur.mp[i])
        if st == ADDED:
            sc.pts[pid].obs[0] = i                                    # AddObservation(KF, i)
        elif st == IN_KF:
            sc.recent.append(pid)                                     # mlpRecentAddedMapPoints.push_back
    for p in sc.pts:
        if out['pointUpdated'][p.id]:
            p.normal, p.min_d, p.max_d = out['normal'][p.id].copy(), out['minDistance'][p.id], out['maxDistance'][p.id]
            if out['descKF'][p.id] >= 0:
                p.desc = (int(out['descKF'][p.id]), int(out['descIdx'][p.id]))
    if out['nConnected'] >= 0:
        nbr_off = np.cumsum([0] + [len(k.conn) + 1 for k in kfs])
        for t, n in enumerate(out['nbrCount']):
            if n >= 0:
                kfs[t].conn[0] = int(out['counter'][t])
                kfs[t].ordered = list(zip(out['nbrKF'][nbr_off[t]:nbr_off[t] + n].tolist(), out['nbrWeight'][nbr_off[t]:nbr_off[t] + n].tolist()))
        cur.conn = {t: int(c) for t, c in enumerate(out['counter']) if c > 0}
        n = out['nConnected']
        cur.ordered = list(zip(out['orderedKF'][:n].tolist(), out['orderedWeight'][:n].tolist()))
        if out['parent'] >= 0:
            cur.parent, cur.first = out['parent'], False
            kfs[out['parent']].children.append(0)                    # AddChild
    return sc


def same_outputs(a, b):
    return all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in OUT_KEYS)


# ---- seeded scenes ----
def _orders(rng, n):
    """n distinct pointer-like keys in an order unrelated to the table's or the mnIds'."""
    return (0x7f3a00000000 + rng.permutation(n).astype(np.int64) * 0x2c0 + rng.integers(0, 0x100, n) * 2).tolist()


def scene(seed, mode, n_kf=150, n_slots=1000, p_filled=0.7, obs_per_point=10, p_dup=0.02, p_in_kf=0.3, p_bad_point=0.03, n_bad_kf=3,
          n_other=2, p_conn_cur=0.5, p_equal=0.3, first=None, init=False, nlevels=8):
    """A current keyframe (table entry 0) with n_slots slots, p_filled of them holding a point; each point observed by about
    obs_per_point keyframes drawn from a local window of the table (so counts fall on both sides of 15).  ProcessNewKeyFrame: p_in_kf of
    the points already observe the current keyframe, p_dup of the slots repeat an earlier slot's point.  SearchInNeighbors: every point
    observes it.  Keys shuffled against mnIds; n_bad_kf bad and n_other other-map keyframes; every observer has a connection map, with the
    current keyframe in it with probability p_conn_cur, at exactly the count this call gives it with probability p_equal."""
    rng = np.random.default_rng(seed)
    sf = (F32(1.2) ** np.arange(nlevels)).astype(F32)
    sc = Scene(mode, sf)
    orders, ids = _orders(rng, n_kf), (1000 + rng.permutation(n_kf)).tolist()
    for t in range(n_kf):
        N = n_slots if t == 0 else max(n_slots, 64)      # a keyframe observes each point at most once
        sc.add_kf(orders[t], ids[t], rng.uniform(-1, 1, 3), np.minimum(rng.geometric(0.6, N) - 1, nlevels - 1), rng.integers(0, 256, (N, 32), np.uint8))
    cur = sc.kfs[0]
    cur.first = bool(rng.random() < 0.5) if first is None else first
    cur.init = init
    for t in rng.choice(np.arange(1, n_kf), n_bad_kf + n_other, replace=False)[:n_bad_kf] if n_kf > 1 else []:
        sc.kfs[int(t)].bad = True
    others = [t for t in range(1, n_kf) if not sc.kfs[t].bad]
    for t in rng.choice(others, min(n_other, len(others)), replace=False) if others else []:
        sc.kfs[int(t)].other = True
    free = {t: list(rng.permutation(len(sc.kfs[t].oct))) for t in range(1, n_kf)}
    window = max(1, min(n_kf - 1, 3 * obs_per_point))
    for i in range(n_slots):
        if rng.random() >= p_filled:
            continue
        if mode == PNK and i and rng.random() < p_dup:
            prev = [int(q) for q in cur.mp[:i] if q >= 0 and 0 not in sc.pts[int(q)].obs]
            if prev:
                cur.mp[i] = prev[int(rng.integers(len(prev)))]
                continue
        base = rng.integers(0, 256, 32, np.uint8)
        c0 = int(rng.integers(1, max(2, n_kf - window + 1)))
        m = int(min(window, max(1, rng.poisson(obs_per_point - 1) + 1)))
        obs = []
        for t in rng.choice(np.arange(c0, min(c0 + window, n_kf)), min(m, min(c0 + window, n_kf) - c0), replace=False) if n_kf > 1 else []:
            t = int(t)
            idx = free[t].pop()
            d = base.copy()
            d[rng.integers(0, 32, 3)] ^= rng.integers(1, 256, 3).astype(np.uint8)    # a noisy view of the point's descriptor
            sc.kfs[t].desc[idx] = d
            obs.append((t, idx))
        cur.desc[i] = base
        if mode == SIN or rng.random() < p_in_kf:
            obs.append((0, i))
        if not obs:
            continue
        pos = np.array([rng.uniform(-4, 4), rng.uniform(-3, 3), rng.uniform(4, 12)])
        ts = [t for t, _ in obs]
        p = sc.add_point(pos, obs, ref=int(ts[int(rng.integers(len(ts)))]))
        if rng.random() < p_bad_point:
            p.bad, p.obs = True, {}
        cur.mp[i] = p.id
    cnt = restate(sc)['counter'] if n_kf > 1 else np.zeros(1, np.int32)
    for t in range(1, n_kf):
        k = sc.kfs[t]
        for u in rng.choice(np.arange(1, n_kf), min(8, n_kf - 1), replace=False) if n_kf > 2 else []:
            if int(u) != t:
                k.conn[int(u)] = int(rng.integers(1, 80))
        if rng.random() < p_conn_cur:
            k.conn[0] = int(cnt[t]) if cnt[t] and rng.random() < p_equal else int(rng.integers(1, 60))
    return sc


def from_search_in_neighbors(job, seed=0):
    """The new keyframe of a search_in_neighbors_lib job after SearchInNeighbors, as a SearchInNeighbors-mode scene.  That model orders
    keyframes by id, so the keys follow the ids; the mnIds are shuffled against them.  Every point's mpRefKF is its first observer."""
    mp, c = job['map'], job['cur']
    rng = np.random.default_rng(seed)
    ids = (500 + rng.permutation(len(mp.kfs))).tolist()
    table = [c] + [k for k in range(len(mp.kfs)) if k != c]
    pos = {k: t for t, k in enumerate(table)}
    sc = Scene(SIN, mp.g['sf'])
    for k in table:
        kf = mp.kfs[k]
        sc.add_kf(0x55d000000000 + 0x340 * k, ids[k], kf.Ow, kf.kps['octave'], kf.desc, bad=kf.bad)
    sc.kfs[0].first = True
    for p in mp.pts:
        q = sc.add_point(p.xyz, [(pos[k], i) for k, i in p.obs.items()], bad=p.bad)
        if p.bad:
            q.obs = {}
    sc.kfs[0].mp = np.array([int(x) for x in mp.kfs[c].mp], np.int64)
    return sc


# ---- planted scenes ----
def _small(mode, n_kf, orders, ids, n_slots=40, seed=0):
    rng = np.random.default_rng(seed)
    sc = Scene(mode, (F32(1.2) ** np.arange(8)).astype(F32))
    for t in range(n_kf):
        sc.add_kf(orders[t], ids[t], rng.uniform(-1, 1, 3), rng.integers(0, 8, n_slots), rng.integers(0, 256, (n_slots, 32), np.uint8))
    return sc


def _fill(sc, slots, observers, rng, pos=None):
    """One point per slot in `slots`, observed by `observers` (table indices) at the slot's keypoint index and, in SearchInNeighbors mode,
    by the current keyframe."""
    for i in slots:
        obs = [(t, i) for t in observers] + ([(0, i)] if sc.mode == SIN else [])
        p = sc.add_point(rng.uniform([-3, -3, 4], [3, 3, 10]) if pos is None else pos, obs)
        sc.kfs[0].mp[i] = p.id


def planted():
    """{name: scene}: one scene per rule the tests pin (see tests/test_update_connections_cpu.py)."""
    rng = np.random.default_rng(7)
    out = {}
    # weight ties decided by key: keyframes 1 and 2 both at 20, key(1) > key(2), mnId(1) < mnId(2)
    sc = _small(SIN, 3, [100, 300, 200], [9, 5, 7])
    _fill(sc, range(20), [1, 2], rng)
    out['tie_by_key'] = sc
    # no count >= 15: 1 and 2 both at 5, the tie goes to the smaller key (2)
    sc = _small(SIN, 3, [100, 300, 200], [9, 5, 7])
    _fill(sc, range(5), [1, 2], rng)
    out['fallback_tie'] = sc
    # an empty counter: the only observers are bad or of another map; mbFirstConnection stays, no parent
    sc = _small(PNK, 3, [100, 300, 200], [9, 5, 7])
    sc.kfs[1].bad, sc.kfs[2].other = True, True
    sc.kfs[0].first = True
    sc.kfs[1].conn, sc.kfs[2].conn = {0: 4}, {0: 4}
    _fill(sc, range(12), [1, 2], rng)
    out['empty_counter'] = sc
    # bad and other-map observers: 3 bad, 4 other map; not counted, 3 summed into the normal but not a descriptor row
    sc = _small(PNK, 5, [500, 100, 200, 300, 400], [1, 5, 4, 3, 2])
    sc.kfs[3].bad, sc.kfs[4].other = True, True
    _fill(sc, range(18), [1, 2, 3, 4], rng)
    out['bad_other_observers'] = sc
    # a point in two slots (ProcessNewKeyFrame): slot 0 adds it, slot 5 finds it in the keyframe; keyframe 1 counts it twice
    sc = _small(PNK, 2, [100, 300], [9, 5])
    _fill(sc, [0], [1], rng)
    sc.kfs[0].mp[5] = sc.kfs[0].mp[0]
    out['two_slots'] = sc
    # an equal-weight AddConnection: keyframe 1 already holds the current keyframe at 20 and a bad keyframe (3) in its map
    # a re-sorted list dropping bad keyframes: keyframe 2 holds the current keyframe at 3 and the bad keyframe 3 at 40
    sc = _small(SIN, 5, [250, 300, 200, 150, 350], [9, 5, 7, 4, 6], n_slots=60)
    sc.kfs[3].bad = True
    _fill(sc, range(20), [1], rng)
    _fill(sc, range(20, 36), [2], rng)
    sc.kfs[1].conn = {0: 20, 3: 50, 4: 10}
    sc.kfs[2].conn = {0: 3, 3: 40, 4: 7, 1: 16}
    out['equal_weight_and_resort'] = sc
    # the map's init keyframe gets no parent; the same scene without the flag does
    for init in (True, False):
        sc = _small(SIN, 3, [100, 300, 200], [0, 5, 7])
        sc.kfs[0].first, sc.kfs[0].init = True, init
        _fill(sc, range(16), [1], rng)
        _fill(sc, range(16, 19), [2], rng)
        out['init_no_parent' if init else 'first_connection_parent'] = sc
    # a median tie decided by where the new row goes: new row == keyframe 1's row; keys: current < 1 < 2 < 3
    sc = _small(PNK, 4, [100, 300, 400, 500], [9, 1, 2, 3])
    p = sc.add_point([0.5, 0.2, 6.0], [(1, 3), (2, 3), (3, 3)])
    sc.kfs[1].desc[3] = sc.kfs[0].desc[3]
    sc.kfs[2].desc[3] = ~sc.kfs[0].desc[3]
    sc.kfs[3].desc[3] = sc.kfs[0].desc[3] ^ np.uint8(0x0f)
    sc.kfs[0].mp[3] = p.id
    out['median_tie_insert'] = sc
    # normals whose bits depend on the summation order: many points of 4-7 observers, keys shuffled against mnIds
    out['normal_order'] = scene(11, PNK, n_kf=12, n_slots=80, obs_per_point=5)
    return out
