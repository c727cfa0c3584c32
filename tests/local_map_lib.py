"""Tracking::UpdateLocalMap's UpdateLocalKeyFrames and UpdateLocalPoints (src/Tracking.cc; monocular and mono-inertial) over a small
model (test infrastructure):
- the model: keyframes (a pointer-order `key`, isBad(), the ordered covisibles, children, parent, mPrevKF, slots of point ids or None),
  points (isBad(), observations {keyframe: slot}, the fields the local-map slabs carry) and one stream's vote source (the frame's match
  index space `src`, the frame's `match` row or the last frame voting, the sensor and mpLastKeyFrame);
- `flatten`: one stream's item dict of orbm_update_local_map_batch (keyframe table in key order), with the table and point orders;
- `oracle`: orbo_update_local_map (oracle/local_map_oracle.cpp) on a batch dict;
- `restate`: an independent Python restatement on the model;
- `replay`: what a host shim does with the call's result, in model terms (comparable with `restate`);
- `scene` and the planted scenes."""
import ctypes as C

import numpy as np

import oracle_lib as O
import orb_slam3_modified_b200 as orb

F32 = np.float32


class KF:
    def __init__(self, kid, key, bad=False):
        self.id, self.key, self.bad = kid, key, bad
        self.cov, self.children, self.parent, self.prev, self.slots = [], set(), None, None, []


class MP:
    def __init__(self, pid, rng, bad=False):
        self.id, self.bad, self.obs = pid, bad, {}
        self.worldPos = rng.normal(0, 3, 3).astype(F32)
        self.normal = rng.normal(0, 1, 3).astype(F32)
        self.maxDistance = F32(rng.uniform(1, 20))
        self.minDistInv, self.maxDistInv = F32(0.8) * self.maxDistance / F32(7.0), F32(1.2) * self.maxDistance
        self.desc = rng.integers(0, 256, 32, dtype=np.uint8)
        self.hasObs = np.uint8(rng.random() > 0.1)


class Scene:
    """One stream.  src: the frame's match index space (point ids or None); match: the current frame's row (indices into src or -1), read
    when vote_last is False; vote_last: the last frame (every src entry) votes; inertial: IMU sensor; last_kf: mpLastKeyFrame (id or None)."""
    def __init__(self, seed=0):
        self.rng = np.random.default_rng(seed)
        self.kfs, self.pts = [], []
        self.src, self.match, self.vote_last, self.inertial, self.last_kf = [], [], False, False, None

    def add_kf(self, key=None, bad=False, n_slots=0):
        k = KF(len(self.kfs), len(self.kfs) * 8 + 4096 if key is None else key, bad)
        k.slots = [None] * n_slots
        self.kfs.append(k)
        return k.id

    def add_point(self, obs=(), bad=False):
        """obs: keyframe ids; the point takes a new slot at the end of each."""
        p = MP(len(self.pts), self.rng, bad)
        for k in obs:
            p.obs[k] = len(self.kfs[k].slots)
            self.kfs[k].slots.append(p.id)
        self.pts.append(p)
        return p.id

    def set_parent(self, k, parent):
        if self.kfs[k].parent is not None:
            self.kfs[self.kfs[k].parent].children.discard(k)
        self.kfs[k].parent = parent
        if parent is not None:
            self.kfs[parent].children.add(k)


# ---- flatten ----
def vote_points(sc):
    if sc.vote_last:
        return [p for p in sc.src if p is not None]
    return [sc.src[m] for m in sc.match if m >= 0 and sc.src[m] is not None]


def flatten(sc):
    """(item dict of orb.local_map_batch, table [kf ids in table order], points [point ids in point order])."""
    voting = sorted(set(p for p in sc.src if p is not None))      # every entry: which ones vote is the pose step's business
    observers = set(k for p in voting for k in sc.pts[p].obs)
    table = set(observers)
    for k in observers:
        kf = sc.kfs[k]
        table |= set(kf.cov[:10]) | kf.children | ({kf.parent} if kf.parent is not None else set())
    if sc.inertial:
        t = sc.last_kf
        for _ in range(20):
            if t is None:
                break
            table.add(t)
            t = sc.kfs[t].prev
    table = sorted(table, key=lambda k: sc.kfs[k].key)
    ti = {k: i for i, k in enumerate(table)}
    points = sorted(set(voting) | set(p for k in table for p in sc.kfs[k].slots if p is not None) | set(p for p in sc.src if p is not None))
    pi = {p: i for i, p in enumerate(points)}
    vset = set(voting)
    it = dict(kfFlags=[orb.KF_BAD if sc.kfs[k].bad else 0 for k in table], covStart=[0], covKF=[], childStart=[0], childKF=[],
              parent=[], prevKF=[], slotStart=[0], slotPoint=[], obsStart=[0], obsKF=[])
    for k in table:
        kf = sc.kfs[k]
        if k in observers:
            it['covKF'] += [ti[c] for c in kf.cov[:10]]
            it['childKF'] += sorted(ti[c] for c in kf.children)
        it['covStart'].append(len(it['covKF'])); it['childStart'].append(len(it['childKF']))
        it['parent'].append(ti[kf.parent] if k in observers and kf.parent is not None else -1)
        it['prevKF'].append(ti.get(kf.prev, -1) if kf.prev is not None else -1)
        it['slotPoint'] += [pi[p] for p in kf.slots if p is not None]
        it['slotStart'].append(len(it['slotPoint']))
    for p in points:
        if p in vset:
            it['obsKF'] += sorted(ti[k] for k in sc.pts[p].obs)
        it['obsStart'].append(len(it['obsKF']))
    P = [sc.pts[p] for p in points]
    it.update(pointBad=[p.bad for p in P], worldPos=np.array([p.worldPos for p in P], F32).reshape(-1, 3),
              normal=np.array([p.normal for p in P], F32).reshape(-1, 3), minDistInv=[p.minDistInv for p in P], maxDistInv=[p.maxDistInv for p in P],
              maxDistance=[p.maxDistance for p in P], mpDesc=np.array([p.desc for p in P], np.uint8).reshape(-1, 32), hasObs=[p.hasObs for p in P],
              srcPoint=[pi[p] if p is not None else -1 for p in sc.src], voteLastFrame=int(sc.vote_last), inertial=int(sc.inertial),
              lastKF=ti[sc.last_kf] if sc.inertial and sc.last_kf is not None else -1)
    if not sc.vote_last:
        it['match'] = list(sc.match)
    return it, table, points


# ---- the oracle ----
def oracle(d):
    """orbo_update_local_map on batch dict `d` (orb.local_map_batch): the outputs of orb.local_map_outputs."""
    L = O.lib()
    out = orb.local_map_outputs(d)
    keep = {n: np.ascontiguousarray(d[n], dt) for n, dt in orb.LOCAL_MAP_ARRAYS if d.get(n) is not None}
    s, r = orb.local_map_structs(d, out, lambda n: keep[n].ctypes.data if n in keep else None)
    L.orbo_update_local_map.argtypes = [C.c_void_p, C.c_void_p]
    L.orbo_update_local_map.restype = None
    L.orbo_update_local_map(C.byref(s), C.byref(r))
    return out


# ---- the Python restatement ----
def restate(sc):
    """UpdateLocalKeyFrames + UpdateLocalPoints on the model: dict(localKF, refKF, localPoint (ids), frame (the voting frame's points
    after the bad ones are NULLed), marked_kf, marked_pt)."""
    frame = list(sc.src) if sc.vote_last else [sc.src[m] if m >= 0 else None for m in sc.match]
    votes = {}
    for i, p in enumerate(frame):
        if p is None:
            continue
        if sc.pts[p].bad:
            frame[i] = None
            continue
        for k in sc.pts[p].obs:
            votes[k] = votes.get(k, 0) + 1
    local, marked = [], set()

    def take(k):
        local.append(k)
        marked.add(k)
    ref, best = None, 0
    for k in sorted(votes, key=lambda k: sc.kfs[k].key):
        if sc.kfs[k].bad:
            continue
        if votes[k] > best:
            best, ref = votes[k], k
        take(k)
    for k in list(local):
        if len(local) > 80:
            break
        kf = sc.kfs[k]
        c = next((c for c in kf.cov[:10] if not sc.kfs[c].bad and c not in marked), None)
        if c is not None:
            take(c)
        c = next((c for c in sorted(kf.children, key=lambda c: sc.kfs[c].key) if not sc.kfs[c].bad and c not in marked), None)
        if c is not None:
            take(c)
        if kf.parent is not None and kf.parent not in marked:
            take(kf.parent)
            break
    if sc.inertial and len(local) < 80:
        t, steps = sc.last_kf, 0
        while steps < 20 and t is not None:
            if t not in marked:
                take(t)
                t = sc.kfs[t].prev
            steps += 1
    points, seen = [], set()
    for k in reversed(local):
        for p in sc.kfs[k].slots:
            if p is not None and p not in seen and not sc.pts[p].bad:
                points.append(p)
                seen.add(p)
    return dict(localKF=local, refKF=ref, localPoint=points, frame=frame, marked_kf=marked, marked_pt=seen)


def replay(sc, table, points, res):
    """The host shim's replay of one stream's result (orb.local_map_split) on the model, in restate's terms."""
    frame = list(sc.src) if sc.vote_last else [sc.src[m] if m >= 0 else None for m in sc.match]
    frame = [None if p is not None and sc.pts[p].bad else p for p in frame]
    local = [table[k] for k in res['localKF']]
    pts = [points[p] for p in res['localPoint']]
    return dict(localKF=local, refKF=table[res['refKF']] if res['refKF'] >= 0 else None, localPoint=pts, frame=frame, marked_kf=set(local),
                marked_pt=set(pts))


def run_oracle(scenes, mcap=4096, kcap=None, mcapLast=None):
    """Flatten every scene into one batch and run the oracle: (batch dict, outputs, [(table, points)])."""
    flat = [flatten(sc) for sc in scenes]
    d = orb.local_map_batch([f[0] for f in flat], mcap, kcap, mcapLast)
    return d, oracle(d), [(f[1], f[2]) for f in flat]


# ---- seeded scenes ----
def scene(seed, n_kf=40, n_pts=600, window=(2, 6), n_src=250, p_null=0.15, p_dup=0.05, p_bad_kf=0.05, p_bad_pt=0.04, vote_last=False,
          inertial=False, trk_space=False, n_kp=None, recent=6):
    """A corridor of n_kf keyframes in time order (mnId = id) whose pointer keys are shuffled; each point is seen by a window of consecutive
    keyframes, the covisibles are ordered by shared points, the spanning tree links each keyframe to one of the three before it and mPrevKF
    to the one before it.  The frame's index space holds points of the `recent` newest keyframes (NULL and bad entries among them; with trk_space a
    block of keyframe features first); the current frame's row matches n_kp keypoints into it with some points held twice."""
    sc = Scene(seed)
    rng = sc.rng
    keys = rng.permutation(n_kf) * 8 + 4096
    for j in range(n_kf):
        sc.add_kf(int(keys[j]), bad=bool(j < n_kf - 1 and rng.random() < p_bad_kf))
    for _ in range(n_pts):
        w = int(rng.integers(window[0], window[1] + 1))
        j = int(rng.integers(0, n_kf))
        sc.add_point(range(j, min(j + w, n_kf)), bad=bool(rng.random() < p_bad_pt))
    for kf in sc.kfs:                                     # NULL slots interleaved
        for _ in range(int(rng.integers(0, 4))):
            kf.slots.insert(int(rng.integers(0, len(kf.slots) + 1)), None)
        for i, p in enumerate(kf.slots):
            if p is not None:
                sc.pts[p].obs[kf.id] = i
    shared = np.zeros((n_kf, n_kf), int)
    for p in sc.pts:
        o = list(p.obs)
        for a in o:
            for b in o:
                if a != b:
                    shared[a, b] += 1
    for kf in sc.kfs:
        nb = [k for k in range(n_kf) if shared[kf.id, k] > 0]
        kf.cov = sorted(nb, key=lambda k: (-shared[kf.id, k], sc.kfs[k].key))
    for j in range(1, n_kf):
        sc.set_parent(j, int(rng.integers(max(0, j - 3), j)))
        sc.kfs[j].prev = j - 1
    recent = [p for k in range(max(0, n_kf - recent), n_kf) for p in sc.kfs[k].slots if p is not None]
    src = [int(rng.choice(recent)) if recent and rng.random() > p_null else None for _ in range(n_src)]
    if trk_space:
        src = [p if rng.random() > 0.3 else None for p in sc.kfs[n_kf - 1].slots] + src
    sc.src = src
    n_kp = n_kp or int(n_src * 1.2)
    hit = [j for j, p in enumerate(src) if p is not None]
    match = [-1] * n_kp
    if hit:
        for i in range(n_kp):
            if rng.random() < 0.7:
                match[i] = int(rng.choice(hit))
        for i in rng.choice(n_kp, int(n_kp * p_dup), replace=False):
            j = int(rng.integers(0, n_kp))
            match[int(i)] = match[j]
    sc.match = match
    sc.vote_last, sc.inertial = vote_last, inertial
    sc.last_kf = n_kf - 1
    return sc


def chain(n, key=None, **kw):
    """n keyframes in a prev chain, keys in id order unless given."""
    sc = Scene(kw.get('seed', 0))
    for j in range(n):
        sc.add_kf(None if key is None else key(j))
        if j:
            sc.kfs[j].prev = j - 1
    return sc


def vote_for(sc, counts, last=False):
    """Points so that keyframe k gets counts[k] votes from the current frame (or the last frame): one point per vote, seen by k alone."""
    for k, c in counts.items():
        for _ in range(c):
            p = sc.add_point([k])
            sc.src.append(p)
    sc.match = list(range(len(sc.src)))
    sc.vote_last = last


def planted():
    """One scene per rule the kernel has a path for (the GPU tests compare them with the oracle; the CPU tests with the restatement):
    more than 80 voters, the 80 cap ending the expansion (size 81, not 80), the parent break with a bad parent, bad voters / neighbours,
    children order, a count tie, duplicate votes, the stalled walk, points shared by local keyframes, more than 32 children, and tables of
    more than 256 rows with the largest count in the second chunk and a tie across chunks."""
    out = []
    sc = scene(3, n_kf=200, n_pts=3000, window=(2, 4), n_src=900)
    sc.src = [p for k in range(200) for p in sc.kfs[k].slots[:3] if p is not None]
    sc.match = list(range(len(sc.src)))
    out.append(sc)                                      # more than 80 voters: no expansion
    sc = chain(120)
    vote_for(sc, {k: 1 for k in range(78)})
    for k in range(78):
        sc.kfs[k].cov = [78 + (k % 40)]
    out.append(sc)                                      # 78 voters + covisibles: the expansion stops at 81
    sc = chain(10)
    vote_for(sc, {0: 1, 1: 1, 2: 1})
    sc.kfs[1].cov = [5]
    sc.set_parent(1, 6)
    sc.kfs[6].bad = True
    sc.kfs[2].cov = [7]
    out.append(sc)                                      # parent break, bad parent added
    sc = chain(12, key=lambda j: 1000 - 8 * j)
    vote_for(sc, {3: 2, 4: 2, 5: 1, 6: 3})
    sc.kfs[6].bad = True
    sc.kfs[3].cov = [6, 8, 9]
    for c in (9, 10, 11):
        sc.set_parent(c, 4)
    out.append(sc)                                      # bad voter / neighbour, children in key order, tie
    sc = chain(6)
    vote_for(sc, {1: 2, 2: 3})
    sc.match = [0, 0, 0, 1, 2, 3, 4]
    sc.pts[sc.src[3]].bad = True
    out.append(sc)                                      # duplicate votes, a bad voting point
    sc = chain(30)
    sc.inertial, sc.last_kf = True, 29
    vote_for(sc, {27: 1}, last=True)
    out.append(sc)                                      # the stalled temporal walk
    sc = chain(4)
    vote_for(sc, {0: 1, 1: 1})
    sc.add_point([0, 1])
    sc.add_point([1])
    out.append(sc)                                      # reverse order decides shared points
    sc = chain(60, key=lambda j: 4096 + 8 * ((j * 37) % 60))
    vote_for(sc, {0: 1, 50: 1})
    for c in range(1, 46):
        sc.set_parent(c, 0)
    kids = sorted(range(1, 46), key=lambda c: sc.kfs[c].key)
    for c in kids[:38]:
        sc.kfs[c].bad = True                            # the first good child in key order is the 39th: push_first's second chunk
    sc.set_parent(50, 1)
    out.append(sc)
    for tie in (False, True):
        sc = chain(400)
        counts = {k: 1 for k in range(400)}
        counts[270], counts[300], counts[20] = 3, 3, 3 if tie else 2
        vote_for(sc, counts)
        out.append(sc)                                  # 400 voters: a three-chunk voter scan, pKFmax in a later chunk or tied across chunks
    return out
