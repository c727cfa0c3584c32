"""KeyFrameDatabase (src/KeyFrameDatabase.cc) for the tests: scenes, operation sequences, the CPU oracle's driver and an independent
restatement of both detections.

The restatement does not walk lists: a keyframe shares the words of the set intersection of the two BowVectors, lKFsSharingWords is the
sharing keyframes ordered by (first shared query word, add order), and the score is the common words' L1 terms summed in ascending word
order.  Phase 2 is restated over per-keyframe marks and scores that persist across queries, replayed from each query's record as the
host shim does (INTEGRATION.md §2)."""
import ctypes as C

import numpy as np

import oracle_lib as O

RELOC, NBEST = 0, 1
SPIN = 1            # the NBEST selection loop would spin on a bad keyframe (oracle_lib: ORBO_KFDB_SPIN)


def random_bow(rng, n, vocab, lo=0):
    """n distinct random word ids in [lo, lo + vocab), ascending, with L1-normalised positive values."""
    ids = np.sort(rng.choice(vocab, n, replace=False)).astype(np.int32) + lo
    v = rng.uniform(0.05, 1.0, n)
    return ids, v / np.abs(v).sum()


class Scene:
    """Keyframes of one SLAM system: BowVectors, map of each, isBad(), ordered covisibility lists; maps with IsBad()."""

    def __init__(self, voc_words, bows, kf_map, kf_bad, cov, map_bad):
        self.voc_words, self.bows, self.kf_map, self.kf_bad, self.cov, self.map_bad = voc_words, bows, kf_map, kf_bad, cov, map_bad
        self.n = len(bows)
        used = np.concatenate([np.asarray(b[0], np.int64) for b in bows]) if bows else np.zeros(0, np.int64)
        self.unused = np.setdiff1d(np.arange(voc_words), used)[:1000].astype(np.int32)   # ids no keyframe holds

    def key(self, k, db=0):
        """A pointer-like key, unique within the database."""
        return np.uint64(0x7F3A00000000 + 0x2C0 * k + 8 * db)


def _covisibility(rng, n, deg):
    cov = []
    for k in range(n):
        nb = [j for j in rng.permutation(n)[:deg + 1].tolist() if j != k][:deg]
        cov.append(nb)
    return cov


def scene(seed, n_kf=40, vocab=300, words=(20, 60), n_maps=3, frac_bad=0.0, voc_words=None, deg=12):
    """Random BowVectors over a small vocabulary (much sharing), a random covisibility graph, keyframes of several maps (the last map
    bad).  Keyframe 0 holds many words; keyframes 1 and 2 hold the same BowVector and have no neighbours, so their accumulated scores tie."""
    rng = np.random.default_rng(seed)
    bows = [random_bow(rng, int(rng.integers(*words)), vocab) for _ in range(n_kf)]
    bows[0] = random_bow(rng, min(vocab, 4 * words[1]), vocab)                    # a keyframe shared by many words
    bows[2] = (bows[1][0].copy(), bows[1][1].copy())                              # equal scores: equal accumulated scores when unconnected
    kf_map = rng.integers(0, n_maps, n_kf).astype(np.int32)
    kf_bad = (rng.random(n_kf) < frac_bad).astype(np.uint8)
    cov = _covisibility(rng, n_kf, deg)
    cov[1], cov[2] = [], []                                                       # ... and no neighbours to tell them apart
    map_bad = np.zeros(n_maps, np.uint8)
    if n_maps > 2:
        map_bad[n_maps - 1] = 1
    return Scene(voc_words or vocab + 1000, bows, kf_map, kf_bad, cov, map_bad)


def planted_scene(seed=0):
    """Keyframes whose counters against the queries of `planted_queries` are max and max * 0.8 exactly, for max = 5, 10, 15, 20 (the
    float product sits on an integer; words > min is strict), and one keyframe one above."""
    rng = np.random.default_rng(seed)
    bows = []
    for j, m in enumerate((5, 10, 15, 20)):
        base = 5000 + 100 * j
        for c in (m, m * 4 // 5, m * 4 // 5 + 1):
            ids = np.arange(base, base + c, dtype=np.int32)
            extra = np.arange(base + 50, base + 50 + int(rng.integers(0, 10)), dtype=np.int32)
            ids = np.concatenate([ids, extra])
            v = rng.uniform(0.1, 1.0, len(ids))
            bows.append((ids, v / v.sum()))
    n = len(bows)
    return Scene(6000, bows, np.zeros(n, np.int32), np.zeros(n, np.uint8), _covisibility(rng, n, 3), np.zeros(1, np.uint8))


def planted_queries(first_id):
    rng = np.random.default_rng(first_id)
    out = []
    for j, m in enumerate((5, 10, 15, 20)):
        ids = np.arange(5000 + 100 * j, 5000 + 100 * j + m, dtype=np.int32)
        v = rng.uniform(0.1, 1.0, m)
        out.append(dict(id=first_id + j, kind=RELOC if j % 2 else NBEST, word_id=ids, word_value=v / v.sum(), connected=[], map=0))
    return out


def frame_scene(seed, n_kf=24, frames=6, k=10, L=3):
    """Keyframes from ORB features of matcher_scenes frames, BoW-transformed by the oracle over O.synthetic_vocabulary: each keyframe
    takes a random subset of one frame's descriptors.  Returns (scene, vocabulary, each keyframe's descriptors)."""
    import matcher_scenes
    rng = np.random.default_rng(seed)
    voc = O.synthetic_vocabulary(k, L, seed=k + L)
    descs = [matcher_scenes.extract(t)[1] for t in range(frames)]
    bows, kf_desc = [], []
    for i in range(n_kf):
        d = descs[i % frames]
        sel = np.sort(rng.choice(len(d), int(rng.integers(len(d) // 3, len(d))), replace=False))
        kf_desc.append(d[sel])
        w, v, _, _ = O.bow_transform(voc, d[sel])
        bows.append((w, v))
    kf_map = rng.integers(0, 2, n_kf).astype(np.int32)
    return Scene(voc['n_words'], bows, kf_map, np.zeros(n_kf, np.uint8), _covisibility(rng, n_kf, 8), np.zeros(2, np.uint8)), voc, kf_desc


def large_scene(seed, n_kf=1000, words=500, voc_words=10 ** 6):
    """ORBvoc-sized: BowVectors drawn directly (random ascending ids of a 10^6-word vocabulary, L1-normalised values); neighbouring
    keyframes share a third of their words, so lists are long and scores differ."""
    rng = np.random.default_rng(seed)
    bows = []
    prev = None
    for k in range(n_kf):
        n = int(rng.integers(words - 50, words + 50))
        ids = rng.choice(voc_words, n, replace=False)
        if prev is not None:
            keep = prev[rng.random(len(prev)) < 0.33]
            ids = np.unique(np.concatenate([keep, ids[:n - len(keep)]]))
        ids = np.sort(ids).astype(np.int32)
        v = rng.uniform(0.05, 1.0, len(ids))
        bows.append((ids, v / v.sum()))
        prev = ids
    kf_map = (np.arange(n_kf) * 3 // n_kf).astype(np.int32)
    return Scene(voc_words, bows, kf_map, np.zeros(n_kf, np.uint8), _covisibility(rng, n_kf, 15), np.zeros(3, np.uint8))


def query_from(rng, sc, qid, kind, n_words=(20, 60), vocab=300):
    """A query: mostly a perturbed copy of a keyframe's BowVector (large lists, close scores), sometimes a random one; NBEST queries get
    connected keyframes (some of which share words) and a map."""
    r = rng.random()
    if r < 0.1:
        ids = np.sort(rng.choice(sc.unused, 10, replace=False)).astype(np.int32)        # shares no word
        v = np.full(10, 0.1)
    elif r < 0.4:
        ids, v = random_bow(rng, int(rng.integers(*n_words)), vocab)
    else:
        b = sc.bows[int(rng.integers(sc.n))]
        keep = rng.random(len(b[0])) < 0.8
        ids, v = b[0][keep], b[1][keep] * rng.uniform(0.8, 1.2, int(keep.sum()))
        v = v / v.sum() if len(v) else v
    conn = sorted(rng.choice(sc.n, int(rng.integers(0, 8)), replace=False).tolist()) if kind == NBEST else []
    return dict(id=qid, kind=kind, word_id=np.asarray(ids, np.int32), word_value=np.asarray(v, np.float64), connected=conn,
                map=int(rng.integers(len(sc.map_bad))))


def operations(seed, sc, n_ops=60, first_id=1):
    """A random sequence of add / erase / clear / clearMap / query (1-4 queries per step) that includes an erase followed by a re-add,
    queries of an empty database and, mid-way, a clear."""
    rng = np.random.default_rng(seed)
    live, ops, qid = [], [], first_id
    ops.append(('query', [query_from(rng, sc, qid, RELOC)]))                        # the empty database
    qid += 1
    for step in range(n_ops):
        r = rng.random()
        out = [k for k in range(sc.n) if k not in live]
        if step == n_ops // 2:
            ops.append(('clear',)); live = []
        elif (r < 0.35 or len(live) < 3) and out:
            ks = rng.choice(out, min(len(out), int(rng.integers(1, 6))), replace=False).tolist()
            ops.append(('add', ks)); live += ks
        elif r < 0.5 and live:
            k = live[int(rng.integers(len(live)))]
            ops.append(('erase', [k, int(rng.choice(out)) if out else k]))             # the second may be absent: a no-op
            live.remove(k)
            if rng.random() < 0.6:
                ops.append(('add', [k])); live.append(k)                                # re-added: to the ends of its lists
        elif r < 0.55 and live:
            m = int(rng.integers(len(sc.map_bad)))
            ops.append(('clearMap', m)); live = [k for k in live if sc.kf_map[k] != m]
        else:
            qs = []
            for _ in range(int(rng.integers(1, 5))):
                qs.append(query_from(rng, sc, qid, RELOC if rng.random() < 0.5 else NBEST)); qid += 1
            ops.append(('query', qs))
    return ops


# ---------------------------------------------------------------------------------------------
# the CPU oracle (oracle/keyframe_database_oracle.cpp)
# ---------------------------------------------------------------------------------------------
def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _lib():
    L = O.lib()
    if not getattr(L, '_kfdb_set', False):
        L.orbo_kfdb_create.restype = C.c_void_p
        L.orbo_kfdb_create.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 7 + [C.c_int, C.c_void_p]
        for n in ('orbo_kfdb_destroy', 'orbo_kfdb_clear'):
            getattr(L, n).argtypes = [C.c_void_p]
        for n in ('orbo_kfdb_add', 'orbo_kfdb_erase', 'orbo_kfdb_clear_map'):
            getattr(L, n).argtypes = [C.c_void_p, C.c_int]
        L.orbo_kfdb_list.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.orbo_kfdb_detect_reloc.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 8
        L.orbo_kfdb_detect_nbest.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int,
                                             C.c_int] + [C.c_void_p] * 10
        L._kfdb_set = True
    return L


def flat_bows(bows):
    start = np.zeros(len(bows) + 1, np.int32)
    start[1:] = np.cumsum([len(b[0]) for b in bows])
    ids = np.concatenate([np.asarray(b[0], np.int32) for b in bows]) if bows else np.zeros(0, np.int32)
    vals = np.concatenate([np.asarray(b[1], np.float64) for b in bows]) if bows else np.zeros(0)
    return start, np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(vals, np.float64)


class Oracle:
    """One KeyFrameDatabase of the CPU oracle over a scene."""

    def __init__(self, sc):
        self.sc = sc
        L = _lib()
        start, ids, vals = flat_bows(sc.bows)
        cs = np.zeros(sc.n + 1, np.int32)
        cs[1:] = np.cumsum([len(c) for c in sc.cov])
        cov = np.array([j for c in sc.cov for j in c] or [0], np.int32)
        self._keep = [start, ids, vals, cs, cov, np.ascontiguousarray(sc.kf_map, np.int32), np.ascontiguousarray(sc.kf_bad, np.uint8),
                      np.ascontiguousarray(sc.map_bad, np.uint8)]
        self.h = L.orbo_kfdb_create(sc.voc_words, sc.n, _p(start), _p(ids), _p(vals), _p(self._keep[5]), _p(self._keep[6]), _p(cs), _p(cov),
                                    len(sc.map_bad), _p(self._keep[7]))

    def __del__(self):
        if getattr(self, 'h', None):
            _lib().orbo_kfdb_destroy(self.h)

    def apply(self, op):
        L = _lib()
        if op[0] == 'add':
            for k in op[1]:
                L.orbo_kfdb_add(self.h, k)
        elif op[0] == 'erase':
            for k in op[1]:
                L.orbo_kfdb_erase(self.h, k)
        elif op[0] == 'clear':
            L.orbo_kfdb_clear(self.h)
        elif op[0] == 'clearMap':
            L.orbo_kfdb_clear_map(self.h, op[1])

    def word_list(self, w):
        out = np.zeros(self.sc.n, np.int32)
        n = _lib().orbo_kfdb_list(self.h, w, len(out), _p(out))
        return out[:n].tolist()

    def query(self, q, n_candidates=3):
        """Both phases: (record, candidates) with record = dict(kf, words, scored, score, nSharing, maxCommonWords) and candidates =
        list (RELOC), (loop list, merge list) (NBEST) or SPIN."""
        L = _lib()
        n = self.sc.n
        kf = np.zeros(n, np.int32); words = np.zeros(n, np.int32); scored = np.zeros(n, np.uint8); score = np.zeros(n, np.float32)
        ns = C.c_int(0); mx = C.c_int(0)
        wid, wv = np.ascontiguousarray(q['word_id'], np.int32), np.ascontiguousarray(q['word_value'], np.float64)
        if q['kind'] == RELOC:
            cand = np.zeros(n, np.int32); nc = C.c_int(0)
            rc = L.orbo_kfdb_detect_reloc(self.h, q['id'], len(wid), _p(wid), _p(wv), q['map'], n, _p(kf), _p(words), _p(scored), _p(score),
                                          C.byref(ns), C.byref(mx), _p(cand), C.byref(nc))
            cands = cand[:nc.value].tolist()
        else:
            conn = np.ascontiguousarray(q['connected'] or [0], np.int32)
            loop = np.zeros(n, np.int32); merge = np.zeros(n, np.int32); nl = C.c_int(0); nm = C.c_int(0)
            rc = L.orbo_kfdb_detect_nbest(self.h, q['id'], len(wid), _p(wid), _p(wv), len(q['connected']), _p(conn), q['map'], n_candidates, n,
                                          _p(kf), _p(words), _p(scored), _p(score), C.byref(ns), C.byref(mx), _p(loop), C.byref(nl), _p(merge),
                                          C.byref(nm))
            cands = SPIN if rc == SPIN else (loop[:nl.value].tolist(), merge[:nm.value].tolist())
        m = ns.value
        rec = dict(kf=kf[:m].copy(), words=words[:m].copy(), scored=scored[:m].copy(), score=score[:m].copy(), nSharing=m, maxCommonWords=mx.value)
        return rec, cands


# ---------------------------------------------------------------------------------------------
# the restatement
# ---------------------------------------------------------------------------------------------
def l1_score(a, b):
    """L1Scoring::score: the common words' terms in ascending word order, one running double, -score / 2 rounded to float."""
    ia = {int(w): i for i, w in enumerate(a[0])}
    s = 0.0
    for j, w in enumerate(b[0]):
        i = ia.get(int(w))
        if i is not None:
            vi, wi = float(a[1][i]), float(b[1][j])
            s += abs(vi - wi) - abs(vi) - abs(wi)
    return np.float32(-s / 2.0)


class Restatement:
    """One database: its keyframes in add order, and the keyframes' marks, counters and scores across queries."""

    def __init__(self, sc):
        self.sc = sc
        self.live = []
        self.mark = {RELOC: np.zeros(sc.n, np.uint64), NBEST: np.zeros(sc.n, np.uint64)}
        self.score = {RELOC: np.zeros(sc.n, np.float32), NBEST: np.zeros(sc.n, np.float32)}
        self.stale_reads = 0        # phase 2 read the score of a neighbour marked by the query but not scored by it
        self.ties = 0               # equal accumulated scores next to each other after the stable sort

    def apply(self, op):
        if op[0] == 'add':
            self.live += list(op[1])
        elif op[0] == 'erase':
            gone = set(op[1])
            self.live = [k for k in self.live if k not in gone]
        elif op[0] == 'clear':
            self.live = []
        elif op[0] == 'clearMap':
            self.live = [k for k in self.live if self.sc.kf_map[k] != op[1]]

    def phase1(self, q):
        qset = {int(w): r for r, w in enumerate(q['word_id'])}
        conn = set(q['connected']) if q['kind'] == NBEST else set()
        rows = []
        for seq, k in enumerate(self.live):
            shared = [qset[int(w)] for w in self.sc.bows[k][0] if int(w) in qset]
            if shared and k not in conn:
                rows.append((min(shared), seq, k, len(shared)))
        rows.sort()
        mx = max((r[3] for r in rows), default=0)
        mn = int(np.float32(mx) * np.float32(0.8))
        kf = np.array([r[2] for r in rows], np.int32)
        words = np.array([r[3] for r in rows], np.int32)
        scored = (words > mn).astype(np.uint8)
        score = np.array([l1_score((q['word_id'], q['word_value']), self.sc.bows[k]) if s else 0 for k, s in zip(kf, scored)], np.float32)
        return dict(kf=kf, words=words, scored=scored, score=score, nSharing=len(rows), maxCommonWords=mx)

    def phase1_np(self, q):
        """phase1 over numpy arrays, for databases of thousands of keyframes: the live rows concatenated, each word's rank in the query
        by a binary search, the counter and the first rank per keyframe by bincount / minimum.at, the list by a stable sort on the first
        rank of the sharing keyframes in add order; a score is the common words' terms from intersect1d summed by add.accumulate (one
        running double, in ascending word order).  The record also holds `rank`, each entry's first shared rank."""
        qw, qv = np.asarray(q['word_id'], np.int64), np.asarray(q['word_value'], np.float64)
        conn = set(q['connected']) if q['kind'] == NBEST else set()
        live = [k for k in self.live if k not in conn]
        lens = np.array([len(self.sc.bows[k][0]) for k in live], np.int64)
        ids = np.concatenate([np.asarray(self.sc.bows[k][0], np.int64) for k in live]) if live else np.zeros(0, np.int64)
        owner = np.repeat(np.arange(len(live)), lens)
        pos = np.minimum(np.searchsorted(qw, ids), max(len(qw) - 1, 0))
        hit = qw[pos] == ids if len(qw) else np.zeros(len(ids), bool)
        cnt = np.bincount(owner[hit], minlength=len(live))
        first = np.full(len(live), len(qw), np.int64)
        np.minimum.at(first, owner[hit], pos[hit])
        sel = np.flatnonzero(cnt > 0)
        sel = sel[np.argsort(first[sel], kind='stable')]
        mx = int(cnt.max()) if len(sel) else 0
        mn = int(np.float32(mx) * np.float32(0.8))
        words = cnt[sel].astype(np.int32)
        scored = (words > mn).astype(np.uint8)
        score = np.zeros(len(sel), np.float32)
        for j in np.flatnonzero(scored):
            b = self.sc.bows[live[sel[j]]]
            _, iq, ib = np.intersect1d(qw, np.asarray(b[0], np.int64), assume_unique=True, return_indices=True)
            vi, wi = qv[iq], np.asarray(b[1], np.float64)[ib]
            s = np.add.accumulate(np.abs(vi - wi) - np.abs(vi) - np.abs(wi))[-1]
            score[j] = np.float32(-s / 2.0)
        return dict(kf=np.array([live[i] for i in sel], np.int32), words=words, scored=scored, score=score, nSharing=len(sel),
                    maxCommonWords=mx, rank=first[sel])

    def phase2(self, q, rec, n_candidates=3):
        """Replays the record's marks and scores (as the host shim does), then the reference's phase 2."""
        kind, mark, sc_ = q['kind'], self.mark[q['kind']], self.score[q['kind']]
        for k, s, v in zip(rec['kf'], rec['scored'], rec['score']):
            mark[k] = q['id']
            if s:
                sc_[k] = v
        scored = [(np.float32(v), int(k)) for k, s, v in zip(rec['kf'], rec['scored'], rec['score']) if s]
        if not scored:
            return [] if kind == RELOC else ([], [])
        acc_list, best_acc = [], np.float32(0)
        scored_now = set(rec['kf'][rec['scored'] > 0].tolist())
        for si, k in scored:
            best, acc, best_kf = si, si, k
            for k2 in self.sc.cov[k][:10]:
                if mark[k2] != q['id']:
                    continue
                if k2 not in scored_now:
                    self.stale_reads += 1
                acc = np.float32(acc + sc_[k2])
                if sc_[k2] > best:
                    best_kf, best = k2, sc_[k2]
            acc_list.append((acc, best_kf))
            if acc > best_acc:
                best_acc = acc
        if kind == RELOC:
            keep = np.float32(np.float32(0.75) * best_acc)
            out = []
            for a, k in acc_list:
                if a > keep and self.sc.kf_map[k] == q['map'] and k not in out:
                    out.append(k)
            return out
        acc_list = sorted(acc_list, key=lambda e: -e[0])                               # list::sort(compFirst): stable, descending
        self.ties += sum(int(a[0] == b[0]) for a, b in zip(acc_list, acc_list[1:]))
        loop, merge, seen = [], [], set()
        for a, k in acc_list:
            if len(loop) >= n_candidates and len(merge) >= n_candidates:
                break
            if self.sc.kf_bad[k]:
                return SPIN
            if k not in seen:
                if self.sc.kf_map[k] == q['map'] and len(loop) < n_candidates:
                    loop.append(k)
                elif self.sc.kf_map[k] != q['map'] and len(merge) < n_candidates and not self.sc.map_bad[self.sc.kf_map[k]]:
                    merge.append(k)
                seen.add(k)
        return loop, merge


def same_record(a, b):
    return (a['nSharing'] == b['nSharing'] and a['maxCommonWords'] == b['maxCommonWords'] and
            all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in ('kf', 'words', 'scored', 'score')))
