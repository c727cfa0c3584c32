"""GPU tests of orbv_db_query_batch at the launch shapes of tests/kfdb_scenes.py, byte for byte against the CPU oracle in every field
(key, words, scored, score, nSharing, maxCommonWords): databases of 0 to 5000 keyframes (bpq = min(ceil(maxN / 8), 128) CTAs per
query, warps that loop past 1024 keyframes or scored entries), sharing lists of 5000 entries and tied first ranks over several 512-entry
tiles of the order kernel's radix sort, queries of 0 to 8192 words (the score kernel's shared memory past 48 KB, 13 radix passes),
slots reused out of add order and one whose row still holds an 8192-word keyframe's ids past a 3-word one, two databases under equal
keys.  Each case alone, each query alone, every query of a handle in one call in two orders and repeated; a query whose bpq and
shared-memory size come from another query of the call; outputs past nSharing written 0, cap == nSharing, the first cap entries on
ORB_ERR_CAPACITY, cap 0 with null outputs; maxWords 8192 and 8193 at creation."""
import numpy as np
import pytest

import kfdb_scenes as S
import keyframe_database_lib as K

pytestmark = pytest.mark.gpu

FIELDS = ('key', 'words', 'scored', 'score')


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


class Loaded:
    """A handle with its cases loaded (case i in database i), and per query: the device query, the oracle's record with keys, the
    (case, query id) and the result of a call of that query alone."""

    def __init__(self, orb, cases, n_slots, n_words):
        self.db = db = orb.KeyFrameDatabase(S.VOC, max_databases=len(cases), max_keyframes=n_slots, max_words=n_words)
        self.queries, self.expect, self.where, self.case_of = [], [], [], []
        for d, c in enumerate(cases):
            kd = d if c.key_db is None else c.key_db
            o = K.Oracle(c.sc)
            for op in c.ops:
                o.apply(op)
                if op[0] == 'add':
                    db.add(d, S.keys(c.sc, op[1], kd), [c.sc.bows[k] for k in op[1]])
                    assert db.last_launch_count() == 1
                else:
                    db.erase(d, S.keys(c.sc, op[1], kd))
            assert db.size(d) == len(c.live())
            for q in c.queries:
                rec, _ = o.query(q)
                self.expect.append(dict(key=S.keys(c.sc, rec['kf'], kd), words=rec['words'], scored=rec['scored'], score=rec['score'],
                                        nSharing=rec['nSharing'], maxCommonWords=rec['maxCommonWords']))
                conn = np.concatenate([S.keys(c.sc, q['connected'], kd), np.array(q['absent'], np.uint64)])
                self.queries.append(dict(db=d, kind=q['kind'], word_id=q['word_id'], word_value=q['word_value'], connected=conn))
                self.where.append((c.name, q['id']))
                self.case_of.append(c.name)
        self.single = [run(db, [q])[0] for q in self.queries]

    def index(self, name, qid):
        return self.where.index((name, qid))


def run(db, queries, cap=None):
    got = db.query_batch(queries, cap)
    assert db.last_launch_count() == 3
    return got


def same(g, e):
    return all(np.asarray(g[f]).tobytes() == np.asarray(e[f]).tobytes() for f in FIELDS) and \
        (int(g['nSharing']), int(g['maxCommonWords'])) == (e['nSharing'], e['maxCommonWords'])


@pytest.fixture(scope='module')
def narrow(orb):
    L = Loaded(orb, S.narrow_cases(), S.NARROW_SLOTS, S.NARROW_WORDS)
    yield L
    L.db.close()


@pytest.fixture(scope='module')
def wide(orb):
    L = Loaded(orb, S.wide_cases(), S.WIDE_SLOTS, S.WIDE_WORDS)
    yield L
    L.db.close()


def _handle(request, name):
    return request.getfixturevalue('wide' if name in S.WIDE_NAMES else 'narrow')


@pytest.mark.parametrize('name', S.NARROW_NAMES + S.WIDE_NAMES)
def test_case_alone(request, name):
    """The case's queries in one call, and each alone, equal the oracle."""
    L = _handle(request, name)
    idx = [i for i, c in enumerate(L.case_of) if c == name]
    got = run(L.db, [L.queries[i] for i in idx])
    for i, g in zip(idx, got):
        assert same(L.single[i], L.expect[i]), L.where[i]
        assert same(g, L.expect[i]), L.where[i]


@pytest.mark.parametrize('order', ['forward', 'shuffled'])
@pytest.mark.parametrize('handle', ['narrow', 'wide'])
def test_all_queries_in_one_call(request, handle, order):
    """Every query of the handle in one call: each record equals the oracle's and its single-query call's, byte for byte."""
    L = request.getfixturevalue(handle)
    idx = list(range(len(L.queries)))
    if order == 'shuffled':
        idx = np.random.default_rng(len(idx)).permutation(idx).tolist()
    got = run(L.db, [L.queries[i] for i in idx])
    for i, g in zip(idx, got):
        assert same(g, L.expect[i]) and same(g, L.single[i]), L.where[i]


def _sentinel(out):
    out['key'][:] = np.uint64(0xA5A5A5A5A5A5A5A5)
    out['words'][:] = -0x5A5A5A5B
    out['scored'][:] = 0xA5
    out['score'].view(np.uint32)[:] = 0x7FC0A5A5
    out['nSharing'][:] = -7
    out['maxCommonWords'][:] = -7


def raw_call(orb, db, queries, caps, null=()):
    """orbv_db_query_batch over db_query_struct outputs of width caps[j], filled with a sentinel first; the queries of `null` get null
    output arrays.  Returns (status, outputs)."""
    built = [orb.db_query_struct(q, c) for q, c in zip(queries, caps)]
    for j, (s, out, _) in enumerate(built):
        _sentinel(out)
        if j in null:
            s.key = s.words = s.scored = s.score = None
    arr = (orb.OrbvDbQuery * len(built))(*[b[0] for b in built])
    rc = orb.lib().orbv_db_query_batch(db._h, len(built), arr)
    assert db.last_launch_count() == 3
    return rc, [b[1] for b in built]


def _head(out, e, n):
    return all(out[f][:n].tobytes() == np.asarray(e[f])[:n].tobytes() for f in FIELDS) and \
        (int(out['nSharing'][0]), int(out['maxCommonWords'][0])) == (e['nSharing'], e['maxCommonWords'])


@pytest.mark.parametrize('handle', ['narrow', 'wide'])
def test_repeat_is_byte_identical(orb, request, handle):
    """The whole call twice, every output byte up to cap (the entries past nSharing included)."""
    L = request.getfixturevalue(handle)
    caps = [e['nSharing'] + 17 for e in L.expect]
    rc1, a = raw_call(orb, L.db, L.queries, caps)
    rc2, b = raw_call(orb, L.db, L.queries, caps)
    assert rc1 == rc2 == orb.ORB_OK
    for i, (x, y) in enumerate(zip(a, b)):
        assert all(x[f].tobytes() == y[f].tobytes() for f in x), L.where[i]
        assert _head(x, L.expect[i], L.expect[i]['nSharing']), L.where[i]


def test_shapes_from_another_query(narrow, wide):
    """bpq and the shared-memory size of a call come from its largest query: an 8192-word query next to a 1-word query and one of an
    empty database; the 5000-keyframe database's 1536-word query next to 3-, 1- and 0-keyframe databases."""
    for L, picks, words in ((wide, [('top_ranks', 1), ('top_ranks', 11), ('empty', 1), ('empty', 3)], (S.MAX_WORDS, 1, S.MAX_WORDS, 0)),
                            (narrow, [('wide', 2), ('size3', 1), ('size3', 3), ('size1', 1), ('size0', 4)], (S.NARROW_WORDS, None, 511, None, 0))):
        idx = [L.index(*p) for p in picks]
        assert all(w is None or len(L.queries[i]['word_id']) == w for i, w in zip(idx, words))
        for order in (idx, idx[::-1], idx[1:] + idx[:1]):
            got = run(L.db, [L.queries[i] for i in order])
            for i, g in zip(order, got):
                assert same(g, L.expect[i]) and same(g, L.single[i]), L.where[i]


@pytest.mark.parametrize('handle', ['narrow', 'wide'])
def test_caps(orb, request, handle):
    """Outputs pre-filled with a sentinel, every query of the handle in one call: cap past nSharing gives 0 in [nSharing, cap) of all
    four arrays; cap == nSharing succeeds; cap == nSharing - 1 returns ORB_ERR_CAPACITY with the oracle's first cap entries (scores
    included) and nSharing / maxCommonWords exact; cap 0 with null outputs succeeds for the queries that share nothing."""
    L = request.getfixturevalue(handle)
    ns = [e['nSharing'] for e in L.expect]
    rc, outs = raw_call(orb, L.db, L.queries, [n + 40 for n in ns])
    assert rc == orb.ORB_OK
    for i, (out, n) in enumerate(zip(outs, ns)):
        assert _head(out, L.expect[i], n), L.where[i]
        assert all(not out[f][n:].view(np.uint8).any() for f in FIELDS), L.where[i]
    rc, outs = raw_call(orb, L.db, L.queries, ns)
    assert rc == orb.ORB_OK
    assert all(_head(out, e, n) for out, e, n in zip(outs, L.expect, ns))
    sharing = [i for i, n in enumerate(ns) if n > 0]
    assert len(sharing) < len(ns)
    rc, outs = raw_call(orb, L.db, [L.queries[i] for i in sharing], [ns[i] - 1 for i in sharing])
    assert rc == orb.ORB_ERR_CAPACITY
    for i, out in zip(sharing, outs):
        assert _head(out, L.expect[i], ns[i] - 1), L.where[i]
    empty = [i for i, n in enumerate(ns) if n == 0]
    rc, outs = raw_call(orb, L.db, [L.queries[i] for i in empty], [0] * len(empty), null=range(len(empty)))
    assert rc == orb.ORB_OK
    assert all(int(o['nSharing'][0]) == 0 and int(o['maxCommonWords'][0]) == 0 for o in outs)
    if handle == 'narrow':                                       # long lists whose scored entries go past the score kernel's 1024 warps
        big = [i for i in sharing if ns[i] > 1024 and int(L.expect[i]['scored'][1024:].sum()) > 0]
        assert len(big) >= 3


def test_max_words(orb, wide):
    """orbv_db_create takes maxWords = 8192 and refuses 8193; a BowVector of exactly maxWords words goes through add and query."""
    with pytest.raises(orb.OrbError) as ei:
        orb.KeyFrameDatabase(S.VOC, max_keyframes=4, max_words=S.MAX_WORDS + 1)
    assert ei.value.code == orb.ORB_ERR_ARG
    db = orb.KeyFrameDatabase(S.VOC, max_keyframes=4, max_words=S.MAX_WORDS)
    rng = np.random.default_rng(1)
    full = S.bow(rng, rng.choice(S.VOC, S.MAX_WORDS, replace=False))
    db.add(0, [7], [full])
    g = run(db, [dict(db=0, kind=K.RELOC, word_id=full[0], word_value=full[1])])[0]
    assert g['nSharing'] == 1 and g['maxCommonWords'] == S.MAX_WORDS and g['key'].tolist() == [7]
    over = (np.arange(S.MAX_WORDS + 1, dtype=np.int32), np.ones(S.MAX_WORDS + 1))
    with pytest.raises(orb.OrbError) as ei:
        db.add(0, [8], [over])
    assert ei.value.code == orb.ORB_ERR_ARG
    with pytest.raises(orb.OrbError) as ei:
        db.query_batch([dict(db=0, kind=K.RELOC, word_id=over[0], word_value=over[1])])
    assert ei.value.code == orb.ORB_ERR_ARG
    db.close()
    i = wide.index('top_ranks', 1)
    assert len(wide.queries[i]['word_id']) == S.MAX_WORDS and wide.expect[i]['maxCommonWords'] == S.MAX_WORDS
