"""KeyFrameDatabase scenes at the shapes orbv_db_query_batch launches with (csrc/keyframe_database.cu), for the CPU oracle, the
restatement and the device (CPU only, seeded).

The kernels take their launch shape from the call: kfdb_share_kernel and kfdb_score_kernel run bpq = min(ceil(maxN / 8), 128) CTAs of
8 warps per query (maxN = the largest queried database), so past 1024 keyframes a warp loops over several list positions or scored
entries; kfdb_order_kernel compacts and radix-sorts each sharing list in one 512-thread CTA, one block_prefix per bit of
ceil(log2(nW)), in tiles of 512 entries; the score kernel takes 12 * nW bytes of shared memory for the largest query of the call,
past 48 KB (nW > 4096) by opt-in.

A case is one database of a handle: a Scene (keyframe_database_lib), the add / erase operations that fill it and its queries.  The
cases of a handle are loaded one after the other, case i into database i.  Two handles serve them: NARROW (many slots, rows of
NARROW_WORDS) and WIDE (64 slots, rows of 8192 words, MAX_WORDS).  Every query carries a fresh id (the reference's mnId mark) within
its case; a query's `connected` holds scene indices, possibly repeated or not in the database, and `absent` holds keys that no
database of the handle holds."""
import functools

import numpy as np

import keyframe_database_lib as K

VOC = 20000                  # vocabularyWords of both handles
MAX_WORDS = 8192             # kfdb::MAX_WORDS: orbv_db_create's largest maxWords
NARROW_SLOTS, NARROW_WORDS = 12800, 1536
WIDE_SLOTS, WIDE_WORDS = 64, MAX_WORDS
SH_WARPS, MAX_BPQ, OR_NT = 8, 128, 512
SWEEP_SIZES = (0, 1, 3, 7, 8, 9, 511, 512, 513, 1023, 1024, 1025)
SWEEP_NW = (1, 2, 31, 32, 33, 511, 512, 513, NARROW_WORDS)
WIDE_NW = (8192, 4097, 4096, 513, 512, 511, 33, 32, 31, 2, 1, 0)
TIED_FIRST = (3, 17, 40)     # the first shared query ranks of the tied keyframes
NARROW_NAMES = ['size%d' % n for n in SWEEP_SIZES] + ['wide', 'tied', 'pair_a', 'pair_b']
WIDE_NAMES = ['top_ranks', 'stale', 'empty']


class Case:
    def __init__(self, name, sc, ops, queries, key_db=None):
        self.name, self.sc, self.ops, self.queries = name, sc, ops, queries
        self.key_db = key_db             # the `db` of Scene.key; None: the case's own database index
        assert len({q['id'] for q in queries}) == len(queries) and all(q['id'] > 0 for q in queries)

    def live(self):
        r = K.Restatement(self.sc)
        for op in self.ops:
            r.apply(op)
        return r.live


def keys(sc, kfs, key_db):
    """Scene.key of every keyframe index of `kfs`, as uint64."""
    return np.array([sc.key(int(k), key_db) for k in kfs], np.uint64)


def values(rng, n):
    """BowVector values with magnitudes log-uniform over 1e-9..1, about 5 % of them zero and 10 % negative (check_bow takes any
    value; L1Scoring::score takes fabs of each)."""
    v = 10.0 ** rng.uniform(-9, 0, n)
    v[rng.random(n) < 0.05] = 0.0
    v[rng.random(n) < 0.1] *= -1
    return v


def bow(rng, ids):
    ids = np.unique(np.asarray(ids, np.int64)).astype(np.int32)
    return ids, values(rng, len(ids))


def _scene(rng, bows, n_maps=2, deg=10):
    n = len(bows)
    cov = []
    for k in range(n):
        nb = np.unique(rng.integers(0, n, deg + 2))
        cov.append(rng.permutation(nb[nb != k])[:deg].tolist())
    return K.Scene(VOC, bows, rng.integers(0, n_maps, n).astype(np.int32), np.zeros(n, np.uint8), cov, np.zeros(n_maps, np.uint8))


def _query(rng, qid, kind, ids, connected=(), absent=(), n_maps=2):
    ids, v = bow(rng, ids)
    return dict(id=qid, kind=kind, word_id=ids, word_value=v, connected=[int(k) for k in connected],
                absent=[np.uint64(a) for a in absent], map=int(rng.integers(n_maps)))


def cycled(rng, pool, n):
    """Operations that leave exactly pool[:n] live, in an add order the slots do not follow: pool[:n] and e more keyframes are added
    (shuffled, in up to three calls), the e and r of pool[:n] are erased, and the r are added again.  The free list hands the erased
    slots out again, last freed first, so the re-added keyframes, last in add order, take slots freed in the middle of the pool."""
    pool = [int(k) for k in pool]
    e, r = min(n // 6 + 1, 200), min(n, n // 4 + 1)
    assert len(pool) >= n + e
    first = rng.permutation(pool[:n + e]).tolist()
    ops = [('add', c.tolist()) for c in np.array_split(np.array(first, np.int64), 3) if len(c)]
    back = rng.permutation(pool[:n])[:r].tolist()
    ops.append(('erase', rng.permutation(pool[n:n + e] + back).tolist()))
    if back:
        ops.append(('add', rng.permutation(back).tolist()))
    return ops


def slots(cases, n_slots):
    """The handle's slot of every keyframe, as orbv_db_create / add / erase hand them out for `cases` loaded one after the other
    (case i in database i): the free slots are a stack that starts as n_slots - 1, ..., 0 (top last), an add takes the top, an erase
    pushes the keyframe's slot.  Returns (per case: {keyframe: slot} of the live keyframes in add order, every add as (case, kf,
    slot)).  Raises IndexError where the handle would run out of slots."""
    free = list(range(n_slots - 1, -1, -1))
    out, adds = [], []
    for i, c in enumerate(cases):
        live = {}
        for op in c.ops:
            if op[0] == 'add':
                for k in op[1]:
                    live[k] = free.pop()
                    adds.append((i, k, live[k]))
            elif op[0] == 'erase':
                for k in op[1]:
                    if k in live:
                        free.append(live.pop(k))
        out.append(live)
    return out, adds


# ---------------------------------------------------------------------------------------------
# the NARROW handle
# ---------------------------------------------------------------------------------------------
def _sweep_queries(rng, sc, live, i, lo=0, hi=3000):
    """A perturbed copy of a live keyframe (RELOC), two random queries of SWEEP_NW word counts (NBEST with connected keyframes, live or
    not, and RELOC), one sharing no word and, on every third database, one of no word."""
    qs, qid = [], 1
    if live:
        b = sc.bows[live[int(rng.integers(len(live)))]][0]
        qs.append(_query(rng, qid, K.RELOC, b[rng.random(len(b)) < 0.8])); qid += 1
    for j, nw in enumerate((SWEEP_NW[(2 * i) % len(SWEEP_NW)], SWEEP_NW[(2 * i + 1) % len(SWEEP_NW)])):
        conn = rng.permutation(live)[:5].tolist() + rng.integers(0, sc.n, 3).tolist() if j == 0 else []
        qs.append(_query(rng, qid, K.NBEST if j == 0 else K.RELOC, rng.choice(np.arange(lo, hi), nw, replace=False), conn)); qid += 1
    qs.append(_query(rng, qid, K.NBEST, rng.choice(np.arange(hi, VOC), 10, replace=False))); qid += 1
    if i % 3 == 0:
        qs.append(_query(rng, qid, K.RELOC, [])); qid += 1
    return qs


def sweep_cases(seed=1):
    """Databases of SWEEP_SIZES keyframes of one scene (1200 keyframes of 20..80 words over ids [0, 3000))."""
    rng = np.random.default_rng(seed)
    sc = _scene(rng, [bow(rng, rng.choice(3000, int(rng.integers(20, 81)), replace=False)) for _ in range(1200)])
    out = []
    for i, n in enumerate(SWEEP_SIZES):
        ops = cycled(rng, rng.permutation(sc.n), n)
        c = Case('size%d' % n, sc, ops, [])
        c.queries = _sweep_queries(rng, sc, c.live(), i)
        out.append(c)
    return out


def wide_case(seed=2):
    """5000 live keyframes of about 200 words over ids [0, 3000) (5200 in the scene, cycled), queries of 1400, 1500 and NARROW_WORDS
    random words: nearly every keyframe shares a word (nSharing > 1024) and about half of them are scored."""
    rng = np.random.default_rng(seed)
    sc = _scene(rng, [bow(rng, rng.choice(3000, int(rng.integers(190, 211)), replace=False)) for _ in range(5200)])
    ops = cycled(rng, rng.permutation(sc.n), 5000)
    c = Case('wide', sc, ops, [])
    live = c.live()
    b = sc.bows[live[7]][0]
    c.queries = [_query(rng, 1, K.RELOC, rng.choice(3000, 1500, replace=False)),
                 _query(rng, 2, K.NBEST, rng.choice(3000, NARROW_WORDS, replace=False), rng.permutation(live)[:40]),
                 _query(rng, 3, K.NBEST, rng.choice(3000, 1400, replace=False), rng.permutation(live)[:1100]),
                 _query(rng, 4, K.RELOC, b[rng.random(len(b)) < 0.8])]
    return c


def tied_case(seed=3):
    """1200 live keyframes, about 1130 of which share exactly 6 of the 64 query words (counter == maxCommonWords, all scored), their
    first shared rank drawn from TIED_FIRST so that keyframes of one first word sit in every 512-entry tile of the add-order list,
    interleaved with those of the others; the rest share 1..4 words.  Each keyframe also holds 20..40 words the query lacks."""
    rng = np.random.default_rng(seed)
    qids = np.sort(rng.choice(np.arange(10000, 10500), 64, replace=False))
    other = np.arange(10500, 11000)
    bows = []
    for k in range(1420):
        if rng.random() < 0.95:
            f = int(rng.choice(TIED_FIRST))
            ranks = [f] + rng.choice(np.arange(f + 1, 64), 5, replace=False).tolist()
        else:
            ranks = rng.choice(64, int(rng.integers(1, 5)), replace=False).tolist()
        bows.append(bow(rng, np.concatenate([qids[ranks], rng.choice(other, int(rng.integers(20, 41)), replace=False)])))
    sc = _scene(rng, bows)
    ops = cycled(rng, rng.permutation(sc.n), 1200)
    c = Case('tied', sc, ops, [])
    live = c.live()
    c.queries = [_query(rng, 1, K.RELOC, qids), _query(rng, 2, K.NBEST, qids, rng.permutation(live)[:30]), _query(rng, 3, K.RELOC, qids)]
    return c


def pair_cases(seed=4):
    """Two databases of one scene (1700 keyframes of 20..60 words over [0, 3000)) under the same keys: A holds 1100 of keyframes
    0..1399, B 600 of 500..1699, so that many keyframes are in both.  NBEST queries list more than 1024 connected keys: keyframes of
    the database, keyframes only the other database holds, repeats, and keys no database holds."""
    rng = np.random.default_rng(seed)
    sc = _scene(rng, [bow(rng, rng.choice(3000, int(rng.integers(20, 61)), replace=False)) for _ in range(1700)])
    a = Case('pair_a', sc, cycled(rng, rng.permutation(1400), 1100), [], key_db=0)
    b = Case('pair_b', sc, cycled(rng, 500 + rng.permutation(1200), 600), [], key_db=0)
    absent = [sc.key(sc.n + j, 0) for j in range(40)]
    for me, other in ((a, b), (b, a)):
        mine, theirs = me.live(), sorted(set(other.live()) - set(me.live()))
        conn = rng.permutation(mine)[:len(mine) * 3 // 5].tolist() + rng.permutation(theirs)[:700].tolist()
        conn += rng.choice(conn, 200).tolist()                                  # repeats
        src = sc.bows[mine[3]][0]
        me.queries = [_query(rng, 1, K.NBEST, rng.choice(3000, 400, replace=False), rng.permutation(conn), absent),
                      _query(rng, 2, K.RELOC, src[rng.random(len(src)) < 0.8]),
                      _query(rng, 3, K.NBEST, src, [theirs[0]], absent[:1]),
                      _query(rng, 4, K.NBEST, rng.choice(3000, 200, replace=False), theirs)]
    return [a, b]


@functools.lru_cache(maxsize=None)
def narrow_cases():
    return sweep_cases() + [wide_case(), tied_case()] + pair_cases()


# ---------------------------------------------------------------------------------------------
# the WIDE handle
# ---------------------------------------------------------------------------------------------
def top_ranks_case(seed=5):
    """Keyframes against one 8192-word query Q whose first shared rank uses the radix sort's top bits: 8191 (twice), 4096, 4095 (twice),
    0; rows of 8192 words (all of Q; Q's upper half and 4096 other words; 8192 words not in Q); 20 keyframes of random first rank.
    Queries of every WIDE_NW word count draw their words from Q."""
    rng = np.random.default_rng(seed)
    q = np.sort(rng.choice(VOC, MAX_WORDS, replace=False))
    other = np.setdiff1d(np.arange(VOC), q)

    def kf(ranks, n_other):
        return bow(rng, np.concatenate([q[np.asarray(ranks, np.int64)], rng.choice(other, n_other, replace=False)]))

    above = lambda r, n: [r] + rng.choice(np.arange(r + 1, MAX_WORDS), n, replace=False).tolist()
    bows = [kf(np.arange(MAX_WORDS), 0), kf(np.arange(4096, MAX_WORDS), 4096), kf([8191], 50), kf(above(4096, 20), 30),
            kf(above(4095, 10), 5), kf([4095], 0), kf([8191], 0), bow(rng, rng.choice(other, MAX_WORDS, replace=False)), kf(above(0, 3), 9)]
    for _ in range(20):
        r = int(rng.integers(0, MAX_WORDS - 70))
        bows.append(kf(above(r, int(rng.integers(0, 60))), int(rng.integers(0, 100))))
    sc = _scene(rng, bows)
    ops = cycled(rng, np.arange(sc.n), 24)                                       # the nine above and 15 of the random ones
    queries = []
    for i, nw in enumerate(WIDE_NW):
        ids = q if nw == MAX_WORDS else rng.choice(q, nw, replace=False)
        queries.append(_query(rng, i + 1, K.NBEST if i % 2 else K.RELOC, ids, [3, 20] if i % 2 else []))
    queries.append(_query(rng, len(queries) + 1, K.NBEST, q, [0, 1]))
    return Case('top_ranks', sc, ops, queries)


def stale_case(seed=6):
    """A slot that held an 8192-word row, then a 3-word keyframe: keyframe 0 (8192 words) is added and erased, and keyframe 1 (three
    of its words) takes its slot, whose row still holds keyframe 0's ids past the third.  The queries hold all of keyframe 0's words."""
    rng = np.random.default_rng(seed)
    big = bow(rng, rng.choice(VOC, MAX_WORDS, replace=False))
    small = bow(rng, big[0][[100, 5000, 8000]])
    extra = bow(rng, rng.choice(big[0], 12, replace=False))
    sc = _scene(rng, [big, small, extra])
    ops = [('add', [2, 0]), ('erase', [0]), ('add', [1])]
    return Case('stale', sc, ops, [_query(rng, 1, K.RELOC, big[0]), _query(rng, 2, K.NBEST, big[0], [2])])


def empty_case(seed=7):
    """A database whose keyframes were all erased, queried with 8192, 1 and 0 words."""
    rng = np.random.default_rng(seed)
    sc = _scene(rng, [bow(rng, rng.choice(VOC, 40, replace=False)) for _ in range(3)])
    ops = [('add', [0, 1, 2]), ('erase', [1, 0, 2])]
    return Case('empty', sc, ops, [_query(rng, 1, K.RELOC, rng.choice(VOC, MAX_WORDS, replace=False)),
                                   _query(rng, 2, K.NBEST, sc.bows[0][0][:1]), _query(rng, 3, K.RELOC, [])])


@functools.lru_cache(maxsize=None)
def wide_cases():
    return [top_ranks_case(), stale_case(), empty_case()]
