"""LocalMapping::SearchInNeighbors (reference src/LocalMapping.cc:878-1021, monocular) after the target selection, written out over a small
map model and pluggable backends for the searches of ORBmatcher::Fuse (src/ORBmatcher.cc:1148-1338):
- OracleBackend: the CPU oracle, one search per call;
- GpuChainBackend: orbm_fuse_search, one upload / launch / download per target keyframe;
- GpuBatchBackend: orbm_fuse_search_batch, one launch per round of the lockstep driver.
Two drivers: `sequential` runs every keyframe's SearchInNeighbors in turn (the reference's order); `lockstep` runs the keyframes of
different maps in rounds -- round r searches target r of every keyframe in one call, then walks each keyframe's results in map-point order
-- and pass 2 (Fuse(mpCurrentKeyFrame, vpFuseCandidates)) of all keyframes in one more call (DESIGN.md §4).
The map model: keyframes with mvpMapPoints; map points with observations {keyframe id: index}, nObs, the bad flag, the descriptor, found /
visible and mnFuseCandidateForKF; MapPoint::Replace walks the observations in keyframe-id order (the stand-in for KeyFrame* order) and
ends in ComputeDistinctiveDescriptors.  Point geometry (position, normal, distances) is what the scene seeded: SearchInNeighbors' final
UpdateNormalAndDepth and UpdateConnections are host code this model leaves out.  Also: seeded scenes with duplicate points planted."""
import numpy as np

import oracle_lib as O

F32 = np.float32
TH_LOW = 50
FUSE_KEYS = ('kps', 'desc', 'bounds', 'sf', 'isg', 'log_sf', 'Tcw', 'Ow', 'cam', 'state', 'xyz', 'normal', 'min_d', 'max_d', 'mp_desc')


def globals_():
    tab = O.OracleExtractor().tables()
    from orb_slam3_modified_b200 import synth
    return dict(bounds=(0.0, 0.0, 640.0, 480.0), sf=tab['scale'], isg=tab['inv_sigma2'], log_sf=F32(np.log(F32(1.2))), cam=synth.camera())


# ---- map model ----
class KeyFrame:
    def __init__(self, kid, kps, desc, Tcw, Ow):
        self.id, self.kps, self.desc, self.Tcw, self.Ow = kid, kps, desc, Tcw, Ow
        self.mp = np.full(len(kps), -1, np.int64)          # mvpMapPoints as point ids, -1 = NULL
        self.bad = False


class MapPoint:
    def __init__(self, pid, xyz, desc):
        self.id, self.xyz, self.desc = pid, np.asarray(xyz, F32), np.array(desc, np.uint8)
        self.normal, self.min_d, self.max_d = np.zeros(3, F32), F32(0), F32(0)
        self.obs = {}                                      # keyframe id -> keypoint index
        self.nObs = 0
        self.bad = False
        self.found = self.visible = 1
        self.fuse_cand = -1                                # mnFuseCandidateForKF

    def AddObservation(self, kf, idx):
        if kf.id in self.obs:
            return
        self.obs[kf.id] = int(idx)
        self.nObs += 1

    def IsInKeyFrame(self, kf):
        return kf.id in self.obs


def host_distinctive(descs):
    """MapPoint::ComputeDistinctiveDescriptors' choice on the host (the oracle's transcription): index of the row with the least median distance."""
    return O.distinctive_descriptor(descs)


class Map:
    def __init__(self, g):
        self.g, self.kfs, self.pts = g, [], []

    def observed_descriptors(self, p):
        return [self.kfs[k].desc[i] for k, i in sorted(p.obs.items()) if not self.kfs[k].bad]

    def ComputeDistinctiveDescriptors(self, p):
        if p.bad:
            return
        d = self.observed_descriptors(p)
        if d:
            p.desc = d[host_distinctive(np.stack(d))].copy()

    def Replace(self, p, q):
        """p->Replace(q) (src/MapPoint.cc)."""
        if p.id == q.id:
            return
        obs, p.obs, p.bad = p.obs, {}, True
        for kid in sorted(obs):
            kf, idx = self.kfs[kid], obs[kid]
            if not q.IsInKeyFrame(kf):
                kf.mp[idx] = q.id                          # ReplaceMapPointMatch
                q.AddObservation(kf, idx)
            else:
                kf.mp[idx] = -1                            # EraseMapPointMatch
        q.found += p.found
        q.visible += p.visible
        self.ComputeDistinctiveDescriptors(q)

    def fuse_item(self, kf, cands, th=3.0, desc_of=None):
        """The search of Fuse(kf, cands, th) as an item (FUSE_KEYS): state 1 searched, 2 isBad(), 3 IsInKeyFrame(kf)."""
        M = len(cands)
        state = np.zeros(M, np.uint8); xyz = np.zeros((M, 3), F32); normal = np.zeros((M, 3), F32)
        min_d = np.zeros(M, F32); max_d = np.zeros(M, F32); mpd = np.zeros((M, 32), np.uint8)
        for i, pid in enumerate(cands):
            p = self.pts[pid]
            state[i] = 2 if p.bad else 3 if p.IsInKeyFrame(kf) else 1
            xyz[i], normal[i], min_d[i], max_d[i] = p.xyz, p.normal, p.min_d, p.max_d
            mpd[i] = p.desc if desc_of is None else desc_of[pid]
        g = self.g
        return dict(kps=kf.kps, desc=kf.desc, bounds=g['bounds'], sf=g['sf'], isg=g['isg'], log_sf=g['log_sf'], Tcw=kf.Tcw, Ow=kf.Ow, cam=g['cam'],
                    state=state, xyz=xyz, normal=normal, min_d=min_d, max_d=max_d, mp_desc=mpd, th=th)

    def fuse_walk(self, kf, cands, bi, bd, ev):
        """Fuse's bookkeeping (src/ORBmatcher.cc:1310-1330) in map-point order.  isBad() / IsInKeyFrame(kf) are tested again when the walk
        reaches a point: the search read them at the start of the round."""
        n = 0
        for i in np.nonzero(bd <= TH_LOW)[0]:
            p = self.pts[cands[i]]
            if p.bad or p.IsInKeyFrame(kf):
                ev['retest'] += 1
                continue
            idx = int(bi[i])
            pin_id = kf.mp[idx]
            if pin_id >= 0:
                pin = self.pts[pin_id]
                if not pin.bad:
                    if pin.nObs > p.nObs:
                        self.Replace(p, pin); ev['replace_into_kf'] += 1
                    else:
                        self.Replace(pin, p); ev['replace_from_kf'] += 1
                else:
                    ev['pin_bad'] += 1
            else:
                p.AddObservation(kf, idx)
                kf.mp[idx] = p.id                          # AddMapPoint
                ev['add'] += 1
            n += 1
        return n

    def state(self):
        """Everything SearchInNeighbors may change, for comparisons."""
        return ([kf.mp.tolist() for kf in self.kfs],
                [(sorted(p.obs.items()), p.nObs, p.bad, p.desc.tobytes(), p.found, p.visible, p.fuse_cand) for p in self.pts])


# ---- backends ----
class OracleBackend:
    def fuse(self, items):
        return [O.fuse_search(it, it['th']) for it in items]

    def distinctive(self, lists):
        return [O.distinctive_descriptor(d) for d in lists]


class GpuChainBackend:
    """orbm_fuse_search once per target keyframe; the final ComputeDistinctiveDescriptors once per keyframe."""
    def __init__(self, matcher):
        self.m, self.calls = matcher, 0

    def fuse(self, items):
        self.calls += len(items)
        return [self.m.FuseSearch(*[it[k] for k in FUSE_KEYS], it['th']) for it in items]

    def distinctive(self, lists):
        return list(self.m.ComputeDistinctiveDescriptors(lists)) if lists else []


class GpuBatchBackend(GpuChainBackend):
    """orbm_fuse_search_batch once per round; the final ComputeDistinctiveDescriptors once per batch."""
    def fuse(self, items):
        if not items:
            return []
        self.calls += 1
        out = self.m.fuse_search_batch(items)
        assert self.m.last_launch_count() == (1 if any(len(it['state']) and len(it['kps']) for it in items) else 0)
        return out


# ---- SearchInNeighbors after the target selection ----
# A job is one new keyframe: dict(map, cur (keyframe id), targets (keyframe ids in vpTargetKFs order), abort (mbAbortBA after pass 1)).
def _events():
    return dict(retest=0, replace_into_kf=0, replace_from_kf=0, pin_bad=0, add=0, in_kf_later=0, pass2_dup=0, pass2_bad=0, items=0, empty_items=0)


def _pass1_cands(job):
    return [int(p) for p in job['map'].kfs[job['cur']].mp if p >= 0]       # GetMapPointMatches() without the NULLs (Fuse skips them)


def _pass2_cands(job, ev):
    mp, cur = job['map'], job['cur']
    out = []
    for t in job['targets']:
        for pid in mp.kfs[t].mp:
            if pid < 0:
                continue
            p = mp.pts[pid]
            if p.bad:
                ev['pass2_bad'] += 1
                continue
            if p.fuse_cand == cur:
                ev['pass2_dup'] += 1
                continue
            p.fuse_cand = cur
            out.append(int(pid))
    return out


def _item(job, kf, cands, ev, desc_of):
    mp = job['map']
    it = mp.fuse_item(mp.kfs[kf], cands, desc_of=None if desc_of is None else desc_of[id(mp)])
    it['map'], it['pids'] = mp, cands                      # for backends that inspect the items (tests)
    ev['items'] += 1
    ev['empty_items'] += len(cands) == 0
    first = job['first_obs']
    ev['in_kf_later'] += sum(1 for i, pid in enumerate(cands) if it['state'][i] == 3 and kf not in first[pid])
    return it


def _final(be, jobs):
    """The final loop (:1004-1017): ComputeDistinctiveDescriptors of the new keyframe's good points, all jobs in one backend call."""
    todo = [(job['map'], job['map'].pts[pid]) for job in jobs for pid in job['map'].kfs[job['cur']].mp if pid >= 0 and not job['map'].pts[pid].bad]
    lists = [(mp, p, mp.observed_descriptors(p)) for mp, p in todo]
    lists = [x for x in lists if x[2]]
    for (mp, p, d), b in zip(lists, be.distinctive([np.stack(d) for _, _, d in lists])):
        p.desc = d[b].copy()


def _prepare(jobs):
    for job in jobs:
        job['first_obs'] = {p.id: set(p.obs) for p in job['map'].pts}


def sequential(be, jobs):
    """The reference's order: one keyframe after the other, one search per target."""
    _prepare(jobs)
    ev = _events()
    for job in jobs:
        mp = job['map']
        cands = _pass1_cands(job)
        for t in job['targets']:
            bi, bd = be.fuse([_item(job, t, cands, ev, None)])[0]
            mp.fuse_walk(mp.kfs[t], cands, bi, bd, ev)
        if job.get('abort'):
            continue
        c2 = _pass2_cands(job, ev)
        bi, bd = be.fuse([_item(job, job['cur'], c2, ev, None)])[0]
        mp.fuse_walk(mp.kfs[job['cur']], c2, bi, bd, ev)
        _final(be, [job])
    return ev


def lockstep(be, jobs, stale=False):
    """The keyframes (one per map) in lockstep rounds: max(|targets|) + 1 backend calls.  stale=True feeds every search the descriptors the
    points had before the first round (what a single all-targets launch would read): not the reference."""
    assert len({id(j['map']) for j in jobs}) == len(jobs), 'at most one keyframe per map in a batch'
    _prepare(jobs)
    ev = _events()
    desc_of = {id(j['map']): {p.id: p.desc.copy() for p in j['map'].pts} for j in jobs} if stale else None
    cands = [_pass1_cands(j) for j in jobs]
    for r in range(max([len(j['targets']) for j in jobs], default=0)):
        live = [s for s, j in enumerate(jobs) if r < len(j['targets'])]
        res = be.fuse([_item(jobs[s], jobs[s]['targets'][r], cands[s], ev, desc_of) for s in live])
        for s, (bi, bd) in zip(live, res):
            mp = jobs[s]['map']
            mp.fuse_walk(mp.kfs[jobs[s]['targets'][r]], cands[s], bi, bd, ev)
    live = [j for j in jobs if not j.get('abort')]
    c2 = [_pass2_cands(j, ev) for j in live]
    res = be.fuse([_item(j, j['cur'], c, ev, desc_of) for j, c in zip(live, c2)])
    for j, c, (bi, bd) in zip(live, c2, res):
        j['map'].fuse_walk(j['map'].kfs[j['cur']], c, bi, bd, ev)
    _final(be, live)
    return ev


# ---- seeded scenes ----
def _update_normal_and_depth(mp, p, ref_kf, ref_idx):
    g = mp.g
    n = np.zeros(3)
    for k in p.obs:
        v = p.xyz.astype(np.float64) - mp.kfs[k].Ow
        n += v / np.linalg.norm(v)
    p.normal = (n / np.linalg.norm(n)).astype(F32)
    dist = np.linalg.norm(p.xyz.astype(np.float64) - mp.kfs[ref_kf].Ow)
    p.max_d = F32(dist * g['sf'][mp.kfs[ref_kf].kps['octave'][ref_idx]])
    p.min_d = F32(p.max_d / g['sf'][-1])


def make_map(g, seed, t0, n_kf=5, step=1, frac_new=0.45, frac_track=0.5, frac_bad=0.03, cur_points=True):
    """Keyframes at frames t0, t0 + step, ... of the synthetic stream.  Keyframe j first tracks the points of keyframe j-1 (the oracle's
    Fuse search; a random frac_track of the hits become observations), then creates points on a random frac_new of its free keypoints.
    The hits not tracked leave two points on one physical point: the duplicates SearchInNeighbors fuses.  frac_bad of the points are bad
    but still in their keyframes' slots.  cur_points=False: the last keyframe holds no point."""
    import matcher_scenes
    from orb_slam3_modified_b200 import synth
    rng = np.random.default_rng(seed)
    mp = Map(g)
    ref = {}
    for j in range(n_kf):
        t = t0 + step * j
        kps, desc = matcher_scenes.extract(t)
        T = synth.pose(t)
        w, x, y, z = T[:4]
        R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                      [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])
        kf = KeyFrame(j, kps, desc, T.astype(F32), (-R.T @ T[4:]).astype(F32))
        mp.kfs.append(kf)
        last = j == n_kf - 1
        if j and (cur_points or not last):
            prev = [int(p) for p in mp.kfs[j - 1].mp if p >= 0]
            bi, bd = O.fuse_search(mp.fuse_item(kf, prev), 3.0)
            for i in np.nonzero(bd <= TH_LOW)[0]:
                p = mp.pts[prev[i]]
                if kf.mp[bi[i]] < 0 and not p.IsInKeyFrame(kf) and rng.random() < frac_track:
                    p.AddObservation(kf, bi[i]); kf.mp[bi[i]] = p.id
        if cur_points or not last:
            free = np.nonzero((kf.mp < 0) & (rng.random(len(kps)) < frac_new))[0]
            P = synth.backproject(np.stack([kps['x'][free], kps['y'][free]], 1), t) + rng.normal(0, 0.004, (len(free), 3))
            for k, X in zip(free, P):
                p = MapPoint(len(mp.pts), X, desc[k])
                p.AddObservation(kf, k); kf.mp[k] = p.id
                p.found, p.visible = int(rng.integers(1, 5)), int(rng.integers(5, 9))
                mp.pts.append(p)
                ref[p.id] = (j, int(k))
                _update_normal_and_depth(mp, p, j, k)
    for p in mp.pts:
        _update_normal_and_depth(mp, p, *ref[p.id])
        mp.ComputeDistinctiveDescriptors(p)
    for p in mp.pts:
        if rng.random() < frac_bad:
            p.bad = True
    return mp


def make_jobs(g, n, seed=0, n_targets=None, abort=(), no_points=()):
    """n keyframes of n different maps; keyframe s of map s is its last, its targets the others newest first (the covisibility order of
    a forward-moving camera), n_targets[s] of them."""
    jobs = []
    for s in range(n):
        nt = 4 if n_targets is None else n_targets[s]
        mp = make_map(g, seed * 1000 + s, 2 + (7 * s + seed) % 24, n_kf=max(nt, 1) + 1, cur_points=s not in no_points)
        cur = len(mp.kfs) - 1
        jobs.append(dict(map=mp, cur=cur, targets=list(range(cur - 1, cur - 1 - nt, -1)), abort=s in abort))
    return jobs
