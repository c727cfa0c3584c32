"""Place-recognition queries for LoopClosing::DetectCommonRegionsFromBoW's BoW sweep (orbm_common_regions_bow_batch), seeded, and an
independent Python restatement of the candidate loop (src/LoopClosing.cc, v1.0) with plain lists, dicts and a set.

A query is the dict ORBmatcher.common_regions_bow_batch takes: kfs (entry 0 the current keyframe), pointBad, cand, cov.  Keyframes observe
the points of a small world: a feature of point w carries w's descriptor with a few bits flipped, w's vocabulary node and w's angle plus
the keyframe's rotation, so SearchByBoW matches the features two keyframes share; clutter features (random descriptors, nodes and
angles) and features with a random angle give the ratio test and the rotation histogram something to reject.  The per-pair search is
the oracle's SearchByBoW(KeyFrame*, KeyFrame*) (oracle_lib.search_by_bow_kf, pinned to the reference's body); the restatement covers
steps 1-5 around it.  `oracle` runs the C++ oracle of the whole loop on a query."""
import ctypes as C

import numpy as np

import oracle_lib as O

SKIPPED, ABORTED_NEAR, RAN = range(3)
MAX_COV = 11
FIELDS = ('status', 'covList', 'nmatches', 'numBoWMatches', 'matchedCov', 'matchedPoint')


def world(rng, W, n_nodes):
    """W map points: descriptor, vocabulary node and angle."""
    return dict(desc=rng.integers(0, 256, (W, 32), dtype=np.uint8), node=rng.integers(0, n_nodes, W).astype(np.int32),
                angle=rng.uniform(0, 360, W).astype(np.float32), n_nodes=n_nodes)


def _flip(rng, desc, max_flips):
    """desc with 0..max_flips random bits flipped per row."""
    desc = desc.copy()
    nf = rng.integers(0, max_flips + 1, len(desc))
    for f in range(max_flips):
        rows = np.flatnonzero(nf > f)
        b = rng.integers(0, 256, len(rows))
        np.bitwise_xor.at(desc, (rows, b >> 3), (1 << (b & 7)).astype(np.uint8))
    return desc


def keyframe(rng, wd, ids, n_clutter=0, rot=0.0, p_null=0.1, bad_angle=0.06, max_flips=6, noise=3.0, bad=False, connected=False):
    """A keyframe observing the world points `ids` (its map points, each NULL with probability p_null) plus n_clutter clutter features,
    in shuffled feature order."""
    ids = np.asarray(ids, np.int64)
    m, n = len(ids), len(ids) + n_clutter
    desc = np.concatenate([_flip(rng, wd['desc'][ids], max_flips), rng.integers(0, 256, (n_clutter, 32), dtype=np.uint8)])
    node = np.concatenate([wd['node'][ids], rng.integers(0, wd['n_nodes'], n_clutter)]).astype(np.int32)
    ang = np.concatenate([wd['angle'][ids] + rot + rng.uniform(-noise, noise, m), rng.uniform(0, 360, n_clutter)])
    wild = rng.random(n) < bad_angle
    ang[wild] = rng.uniform(0, 360, int(wild.sum()))
    point = np.concatenate([np.where(rng.random(m) < p_null, -1, ids), np.full(n_clutter, -1)]).astype(np.int32)
    perm = rng.permutation(n)
    kps = np.zeros(n, O.KP_DTYPE)
    kps['x'] = rng.uniform(0, 640, n); kps['y'] = rng.uniform(0, 480, n)
    kps['angle'] = np.mod(ang[perm], 360.0).astype(np.float32)
    kps['octave'] = rng.integers(0, 8, n); kps['size'] = 31.0; kps['class_id'] = -1
    node = node[perm]
    order = np.lexsort((np.arange(n), node))           # DBoW2::FeatureVector: node ids ascending, features in index order inside a node
    return dict(kps=kps, desc=desc[perm], fv=(node[order].astype(np.int32), order.astype(np.int32)), point=point[perm], bad=bool(bad),
                connected=bool(connected))


def random_query(seed, n_cand=6, n_feat=300, n_cov=(0, 10), share=0.3, p_bad_cand=0.1, p_bad_cov=0.08, p_conn=0.03, p_null_cand=0.0):
    """A query with n_cand candidates, each with n_cov covisibles drawn from new keyframes and (with probability `share`) from the
    entries of earlier candidates.  Bad and connected keyframes with the given probabilities."""
    rng = np.random.default_rng(seed)
    W = 4 * n_feat
    wd = world(rng, W, max(W // 4, 1))
    pbad = (rng.random(W) < 0.03).astype(np.uint8)
    cur = rng.choice(W, n_feat, replace=False)
    kfs = [keyframe(rng, wd, cur, n_clutter=n_feat // 10, rot=float(rng.uniform(0, 360)))]

    def new_kf():
        ov = rng.uniform(0.1, 0.6)
        ids = np.union1d(rng.choice(cur, int(ov * n_feat), replace=False), rng.choice(W, n_feat - int(ov * n_feat), replace=False))
        kfs.append(keyframe(rng, wd, ids, n_clutter=n_feat // 10, rot=float(rng.uniform(0, 360)), bad=rng.random() < p_bad_cov,
                            connected=rng.random() < p_conn))
        return len(kfs) - 1

    cand, cov = [], []
    for _ in range(n_cand):
        if rng.random() < p_null_cand:
            cand.append(-1); cov.append([])
            continue
        c = new_kf()
        kfs[c]['bad'] = bool(rng.random() < p_bad_cand)
        lst = []
        for _ in range(int(rng.integers(n_cov[0], n_cov[1] + 1))):
            pool = [e for e in range(1, len(kfs)) if e != c and e not in lst]
            lst.append(int(rng.choice(pool)) if pool and rng.random() < share else new_kf())
        cand.append(c); cov.append(lst)
    return dict(kfs=kfs, pointBad=pbad, cand=cand, cov=cov)


def exact_query(seed, counts=(19, 20), n_feat=120):
    """Candidates without covisibles whose numBoWMatches are exactly `counts`: the current keyframe's points sit on distinct nodes with
    one feature each, and candidate i observes counts[i] of them with the same descriptors and angles (no NULL slot, no bad point)."""
    rng = np.random.default_rng(seed)
    W = 4 * n_feat
    wd = world(rng, W, 1 << 20)
    wd['node'] = rng.permutation(1 << 20)[:W].astype(np.int32)
    cur = rng.choice(W, n_feat, replace=False)
    kw = dict(p_null=0.0, bad_angle=0.0, max_flips=0, noise=0.0)
    kfs = [keyframe(rng, wd, cur, **kw)]
    for n in counts:
        kfs.append(keyframe(rng, wd, rng.choice(cur, n, replace=False), n_clutter=40, **kw))
    return dict(kfs=kfs, pointBad=np.zeros(W, np.uint8), cand=list(range(1, len(counts) + 1)), cov=[[] for _ in counts])


# ---------------------------------------------------------------------------------------------
# the CPU oracle (oracle/common_regions_oracle.cpp)
# ---------------------------------------------------------------------------------------------
def oracle(q):
    """orbo_common_regions_bow: LoopClosing::DetectCommonRegionsFromBoW up to the Sim3Solver on query dict `q`
    (ORBmatcher.common_regions_bow_batch's form); returns the record as the binding does."""
    import orb_slam3_modified_b200 as orb
    s, out, keep = orb.common_regions_struct(q)
    L = O.lib()
    L.orbo_common_regions_bow.restype = None
    L.orbo_common_regions_bow.argtypes = [C.c_void_p]
    L.orbo_common_regions_bow(C.byref(s))
    return out


# ---------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------
def flags(q, e):
    """SearchByBoW's view of keyframe e's slots: 0 NULL, 1 a map point, 2 a bad one."""
    pt = q['kfs'][e]['point']
    return np.array([0 if p < 0 else 2 if q['pointBad'][p] else 1 for p in pt], np.uint8)


def search(q, e):
    """ORBmatcher(0.9, true).SearchByBoW(mpCurrentKF, kf e): (nmatches, match12 [N0] = feature of e or -1)."""
    a, b = q['kfs'][0], q['kfs'][e]
    return O.search_by_bow_kf(a['kps'], a['desc'], flags(q, 0), a['fv'], b['kps'], b['desc'], flags(q, e), b['fv'], nnratio=0.9, check_ori=True)


def restate(q, events=None):
    """Steps 1-5 of DetectCommonRegionsFromBoW for every candidate: the record as lists (one dict per candidate).  `events`, if given,
    counts what the merge met: 'overwrite' (a later j replaced slot k), 'seen_same_k' / 'seen_diff_k' (a point already inserted, at the
    same / another k)."""
    kfs, N0 = q['kfs'], len(q['kfs'][0]['kps'])
    connected = {e for e, kf in enumerate(kfs) if kf['connected']}
    memo = {}
    out = []
    for c, cand in enumerate(q['cand']):
        rec = dict(status=SKIPPED, covList=[-1] * MAX_COV, nmatches=[-1] * MAX_COV, numBoWMatches=0, matchedCov=[-1] * N0, matchedPoint=[-1] * N0)
        out.append(rec)
        if cand < 0 or kfs[cand]['bad']:
            continue
        cov = list(q['cov'][c])
        lst = [cand] if not cov else [cand] + cov[1:] + [cov[0]]
        rec['covList'][:len(lst)] = lst
        if any(e in connected for e in lst):
            rec['status'] = ABORTED_NEAR
            continue
        rec['status'] = RAN
        matched = []
        for j, e in enumerate(lst):
            if kfs[e]['bad']:
                matched.append([])
                continue
            if e not in memo:
                memo[e] = search(q, e)
            n, m12 = memo[e]
            rec['nmatches'][j] = int(n)
            matched.append([int(kfs[e]['point'][i2]) if i2 >= 0 else -1 for i2 in m12])
        seen, first_k = set(), {}
        for j, row in enumerate(matched):
            for k, p in enumerate(row):
                if p < 0 or q['pointBad'][p]:
                    continue
                if p in seen:
                    if events is not None:
                        events['seen_same_k' if first_k[p] == k else 'seen_diff_k'] += 1
                    continue
                seen.add(p)
                first_k[p] = k
                if events is not None and rec['matchedPoint'][k] >= 0:
                    events['overwrite'] += 1
                rec['numBoWMatches'] += 1
                rec['matchedPoint'][k] = p
                rec['matchedCov'][k] = j
    return out


def as_arrays(recs, N0):
    """The restatement's records in the binding's layout (one dict of arrays per query)."""
    n = len(recs)
    return dict(status=np.array([r['status'] for r in recs], np.uint8).reshape(n),
                covList=np.array([r['covList'] for r in recs], np.int32).reshape(n, MAX_COV),
                nmatches=np.array([r['nmatches'] for r in recs], np.int32).reshape(n, MAX_COV),
                numBoWMatches=np.array([r['numBoWMatches'] for r in recs], np.int32).reshape(n),
                matchedCov=np.array([r['matchedCov'] for r in recs], np.int32).reshape(n, N0),
                matchedPoint=np.array([r['matchedPoint'] for r in recs], np.int32).reshape(n, N0))


def same(a, b):
    return all(np.array_equal(a[f], b[f]) for f in FIELDS)


# ---------------------------------------------------------------------------------------------
# planted merge cases (slot points relabelled after the searches: SearchByBoW reads only whether a slot holds a good point)
# ---------------------------------------------------------------------------------------------
def _ran_lists(q):
    rec = restate(q)
    return [(c, r['covList'][:r['covList'].index(-1) if -1 in r['covList'] else MAX_COV]) for c, r in enumerate(rec) if r['status'] == RAN]


def _good_matches(q, e):
    """[(k, i2, p)] of SearchByBoW(current, e) with a good point p."""
    _, m12 = search(q, e)
    pt = q['kfs'][e]['point']
    return [(k, int(i2), int(pt[i2])) for k, i2 in enumerate(m12) if i2 >= 0 and pt[i2] >= 0 and not q['pointBad'][pt[i2]]]


def plant_shared_diff_k(q, rng):
    """A point two entries of one RAN candidate bring at different k: the later one's slot takes the earlier one's point."""
    for _, lst in _ran_lists(q):
        good = [e for e in lst if not q['kfs'][e]['bad']]
        for a in range(len(good)):
            for b in range(a + 1, len(good)):
                ma, mb = _good_matches(q, good[a]), _good_matches(q, good[b])
                pa = {p for _, _, p in ma}
                for (k1, _, p1) in ma:
                    for (k2, i2, p2) in mb:
                        if k2 != k1 and p2 not in pa:
                            q['kfs'][good[b]]['point'][i2] = p1
                            return True
    return False


def plant_overwrite(q, rng):
    """Slot k overwritten: a later entry of a RAN candidate matches the same current feature k as an earlier one, with a new point."""
    for _, lst in _ran_lists(q):
        good = [e for e in lst if not q['kfs'][e]['bad']]
        for a in range(len(good)):
            for b in range(a + 1, len(good)):
                ka = {k for k, _, _ in _good_matches(q, good[a])}
                for (k, i2, _) in _good_matches(q, good[b]):
                    if k in ka:
                        q['pointBad'] = np.append(q['pointBad'], np.uint8(0))
                        q['kfs'][good[b]]['point'][i2] = len(q['pointBad']) - 1
                        return True
    return False


def planted_queries(seed):
    """The queries of the planted cases (see tests/test_common_regions_cpu.py)."""
    qs = []
    q = random_query(seed, n_cand=6, n_cov=(2, 10), share=0.5, p_bad_cand=0.0, p_bad_cov=0.0, p_conn=0.0)
    rng = np.random.default_rng(seed + 100)
    assert plant_shared_diff_k(q, rng) and plant_overwrite(q, rng)
    qs.append(q)
    # a bad candidate, a NULL candidate, a bad covisible, an empty covisible list, aborts by a connected covisible and a connected candidate
    q = random_query(seed + 1, n_cand=6, n_cov=(1, 4), share=0.0, p_bad_cand=0.0, p_bad_cov=0.0, p_conn=0.0)
    q['kfs'][q['cand'][0]]['bad'] = True
    q['cov'][1] = []
    q['kfs'][q['cov'][2][-1]]['bad'] = True
    q['kfs'][q['cov'][3][0]]['connected'] = True
    q['kfs'][q['cand'][4]]['connected'] = True
    q['cand'][5] = -1
    qs.append(q)
    # a current keyframe with no map points; zero-feature keyframes (a covisible, then the current keyframe)
    q = random_query(seed + 2, n_cand=3, n_cov=(1, 3), p_bad_cand=0.0, p_bad_cov=0.0, p_conn=0.0)
    q['kfs'][0]['point'][:] = -1
    qs.append(q)
    q = random_query(seed + 3, n_cand=3, n_cov=(2, 3), p_bad_cand=0.0, p_bad_cov=0.0, p_conn=0.0)
    q['kfs'][q['cov'][0][1]] = empty_kf()
    qs.append(q)
    q = random_query(seed + 4, n_cand=2, n_cov=(1, 3), p_bad_cand=0.0, p_bad_cov=0.0, p_conn=0.0)
    q['kfs'][0] = empty_kf()
    qs.append(q)
    qs.append(exact_query(seed + 5))
    return qs


def empty_kf():
    return dict(kps=np.zeros(0, O.KP_DTYPE), desc=np.zeros((0, 32), np.uint8), fv=(np.zeros(0, np.int32), np.zeros(0, np.int32)),
                point=np.zeros(0, np.int32), bad=False, connected=False)
