"""GPU tests of orbv_db_*: after every operation of random add / erase / clear / clearMap sequences over 1, 7 and 24 databases of one
handle, every query's record (keys, counters, scored flags, float scores), with RELOC and NBEST mixed in one call, equals the CPU
oracle's phase-1 record byte for byte, and the record through the restatement's phase 2 gives the oracle's candidates; a batch equals
per-query calls byte for byte; three launches whatever the query count; an ORBvoc-sized database (10^6 words, 1000 keyframes of ~500
words); the argument and capacity errors, each leaving the handle usable; the C++ mirror's digest equals the Python binding's."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import keyframe_database_lib as K

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


def _gpu_query(q, sc, d):
    return dict(db=d, kind=q['kind'], word_id=q['word_id'], word_value=q['word_value'], connected=[sc.key(k, d) for k in q['connected']])


def _as_record(g, sc, d):
    """A GPU result with keys turned back into keyframe indices."""
    back = {int(sc.key(k, d)): k for k in range(sc.n)}
    return dict(kf=np.array([back[int(x)] for x in g['key']], np.int32), words=g['words'], scored=g['scored'], score=g['score'],
                nSharing=g['nSharing'], maxCommonWords=g['maxCommonWords'])


def _apply(db, sc, d, op):
    if op[0] == 'add':
        db.add(d, [sc.key(k, d) for k in op[1]], [sc.bows[k] for k in op[1]])
    elif op[0] == 'erase':
        db.erase(d, [sc.key(k, d) for k in op[1]])
    elif op[0] == 'clear':
        db.clear(d)
    elif op[0] == 'clearMap':                                     # clearMap(pMap) == erase of the map's keyframes
        db.erase(d, [sc.key(k, d) for k in range(sc.n) if sc.kf_map[k] == op[1]])


@pytest.mark.parametrize('D', [1, 7, 24])
def test_sequences_equal_oracle(orb, D):
    scenes = [K.scene(300 * D + d, frac_bad=0.15 if d % 3 == 2 else 0.0) for d in range(D)]
    seqs = [K.operations(11 * D + d, sc, n_ops=40) for d, sc in enumerate(scenes)]
    oracles, rests = [K.Oracle(sc) for sc in scenes], [K.Restatement(sc) for sc in scenes]
    db = orb.KeyFrameDatabase(scenes[0].voc_words, max_databases=D, max_keyframes=D * 40, max_words=512)
    n_checked = kinds = 0
    single_checked = False
    for t in range(max(len(s) for s in seqs)):
        batch = []
        for d, sc in enumerate(scenes):
            if t >= len(seqs[d]):
                continue
            op = seqs[d][t]
            oracles[d].apply(op)
            rests[d].apply(op)
            _apply(db, sc, d, op)
            assert db.size(d) == len(rests[d].live)
            if op[0] == 'query':
                batch += [(d, q) for q in op[1]]
        if not batch:
            continue
        got = db.query_batch([_gpu_query(q, scenes[d], d) for d, q in batch])
        assert db.last_launch_count() == 3
        for _, q in batch:
            kinds |= 1 << q['kind']
        for (d, q), g in zip(batch, got):
            rec, cands = oracles[d].query(q)
            mine = _as_record(g, scenes[d], d)
            assert K.same_record(mine, rec), (d, q['id'])
            assert rests[d].phase2(q, mine) == cands, (d, q['id'])
            n_checked += 1
        if not single_checked and len(batch) > 1:                 # the batch equals per-query calls
            single_checked = True
            for (d, q), g in zip(batch, got):
                one = db.query_batch([_gpu_query(q, scenes[d], d)])[0]
                assert all(one[k].tobytes() == g[k].tobytes() for k in ('key', 'words', 'scored', 'score'))
                assert (one['nSharing'], one['maxCommonWords']) == (g['nSharing'], g['maxCommonWords'])
    assert n_checked > 10 * D and kinds == 3 and single_checked


def test_planted_thresholds_equal_oracle(orb):
    sc = K.planted_scene()
    o = K.Oracle(sc)
    o.apply(('add', list(range(sc.n))))
    db = orb.KeyFrameDatabase(sc.voc_words, max_keyframes=sc.n, max_words=64)
    _apply(db, sc, 0, ('add', list(range(sc.n))))
    qs = K.planted_queries(1)
    got = db.query_batch([_gpu_query(q, sc, 0) for q in qs])
    for q, g in zip(qs, got):
        assert K.same_record(_as_record(g, sc, 0), o.query(q)[0])


def test_frame_scene_equals_oracle(orb):
    """The chain the shim runs: keyframes' ORB descriptors through orbv_transform_batch on the device (== the oracle's DBoW2 transform
    bit for bit), those BowVectors into the database sized from the device vocabulary, queries against the oracle."""
    sc, voc, kf_desc = K.frame_scene(5)
    v = orb.ORBVocabulary(voc['L'], voc['child_start'], voc['children'], voc['desc'], voc['weight'], voc['word_id'])
    assert v.n_words == sc.voc_words
    gpu_bows = [(w, val) for w, val, _, _ in v.transform(kf_desc)]
    for g, b in zip(gpu_bows, sc.bows):
        assert g[0].tobytes() == b[0].tobytes() and g[1].tobytes() == b[1].tobytes()
    sc.bows = gpu_bows
    o = K.Oracle(sc)
    db = orb.KeyFrameDatabase(v, max_keyframes=64, max_words=1024)
    for op in K.operations(9, sc, n_ops=30):
        o.apply(op)
        _apply(db, sc, 0, op)
        if op[0] == 'query':
            got = db.query_batch([_gpu_query(q, sc, 0) for q in op[1]])
            for q, g in zip(op[1], got):
                assert K.same_record(_as_record(g, sc, 0), o.query(q)[0])


def test_launch_count_constant_in_queries(orb):
    sc = K.scene(77, n_kf=60)
    db = orb.KeyFrameDatabase(sc.voc_words, max_keyframes=60, max_words=512)
    _apply(db, sc, 0, ('add', list(range(sc.n))))
    assert db.last_launch_count() == 1
    rng = np.random.default_rng(1)
    for n in (1, 8, 48):
        db.query_batch([_gpu_query(K.query_from(rng, sc, i + 1, i % 2), sc, 0) for i in range(n)])
        assert db.last_launch_count() == 3
    db.query_batch([])
    assert db.last_launch_count() == 0


def test_orbvoc_sized_database(orb):
    """vocabularyWords = 10^6, 1000 keyframes of about 500 words, queries from perturbed keyframes: long lists, many scores."""
    sc = K.large_scene(3)
    o = K.Oracle(sc)
    o.apply(('add', list(range(sc.n))))
    db = orb.KeyFrameDatabase(sc.voc_words, max_databases=2, max_keyframes=sc.n, max_words=600)
    _apply(db, sc, 1, ('add', list(range(sc.n))))
    rng = np.random.default_rng(5)
    qs = [K.query_from(rng, sc, 1 + i, i % 2) for i in range(16)]
    got = db.query_batch([_gpu_query(q, sc, 1) for q in qs])
    longest = 0
    for q, g in zip(qs, got):
        assert K.same_record(_as_record(g, sc, 1), o.query(q)[0])
        longest = max(longest, g['nSharing'])
    assert longest > 100


def test_bad_arguments_and_capacity(orb):
    L = orb.lib()
    sc = K.scene(8, n_kf=30)
    db = orb.KeyFrameDatabase(sc.voc_words, max_databases=2, max_keyframes=30, max_words=256)
    _apply(db, sc, 0, ('add', list(range(20))))
    rng = np.random.default_rng(2)
    q0 = _gpu_query(K.query_from(rng, sc, 1, K.NBEST), sc, 0)
    ref = db.query_batch([q0])[0]

    def still_usable():
        g = db.query_batch([q0])[0]
        assert all(g[k].tobytes() == ref[k].tobytes() for k in ('key', 'words', 'scored', 'score')) and db.size(0) == 20

    def add_fails(code, dbs, keys, bows):
        with pytest.raises(orb.OrbError) as ei:
            db.add(dbs, keys, bows)
        assert ei.value.code == code
        still_usable()

    b0 = sc.bows[25]
    add_fails(orb.ORB_ERR_ARG, 2, [sc.key(25)], [b0])                                      # database index out of range
    add_fails(orb.ORB_ERR_ARG, -1, [sc.key(25)], [b0])
    add_fails(orb.ORB_ERR_ARG, 0, [sc.key(3)], [b0])                                       # already present
    add_fails(orb.ORB_ERR_ARG, 0, [sc.key(25), sc.key(25)], [b0, b0])                      # added twice by one call
    add_fails(orb.ORB_ERR_ARG, 0, [sc.key(25)], [(np.array([1, sc.voc_words], np.int32), np.ones(2))])   # id >= vocabularyWords
    add_fails(orb.ORB_ERR_ARG, 0, [sc.key(25)], [(np.array([5, 4], np.int32), np.ones(2))])              # not ascending
    add_fails(orb.ORB_ERR_ARG, 0, [sc.key(25)], [(np.array([5, 5], np.int32), np.ones(2))])
    add_fails(orb.ORB_ERR_ARG, 0, [sc.key(25)], [(np.arange(257, dtype=np.int32), np.ones(257))])        # more than maxWords
    add_fails(orb.ORB_ERR_CAPACITY, 1, [sc.key(k, 1) for k in range(11)], [sc.bows[k] for k in range(11)])   # 10 free slots
    keys = np.array([sc.key(25)], np.uint64); dbs = np.zeros(1, np.int32); ids = np.array([1, 2], np.int32); vals = np.ones(2)
    for start in (np.array([1, 2], np.int32), np.array([0, -1], np.int32)):                                # bad CSR
        assert L.orbv_db_add_batch(db._h, 1, orb._ptr(dbs), orb._ptr(keys), orb._ptr(start), orb._ptr(ids), orb._ptr(vals)) == orb.ORB_ERR_ARG
    assert L.orbv_db_add_batch(db._h, 1, orb._ptr(dbs), orb._ptr(keys), None, orb._ptr(ids), orb._ptr(vals)) == orb.ORB_ERR_ARG
    still_usable()
    assert L.orbv_db_erase_batch(db._h, 1, orb._ptr(np.array([5], np.int32)), orb._ptr(keys)) == orb.ORB_ERR_ARG
    assert L.orbv_db_clear(db._h, 2) == orb.ORB_ERR_ARG
    db.erase(0, [sc.key(29)])                                                              # absent: a no-op
    still_usable()

    def query_fails(code, edit=None, struct_edit=None, cap=30):
        q = dict(q0)
        if edit:
            edit(q)
        s, out, keep = orb.db_query_struct(q, cap)
        if struct_edit:
            struct_edit(s)
        assert L.orbv_db_query_batch(db._h, 1, C.byref(s)) == code
        still_usable()
        return out

    query_fails(orb.ORB_ERR_ARG, lambda q: q.update(db=2))
    query_fails(orb.ORB_ERR_ARG, lambda q: q.update(kind=2))
    query_fails(orb.ORB_ERR_ARG, lambda q: q.update(word_id=np.array([3, sc.voc_words], np.int32), word_value=np.ones(2)))
    query_fails(orb.ORB_ERR_ARG, lambda q: q.update(word_id=np.array([7, 3], np.int32), word_value=np.ones(2)))
    query_fails(orb.ORB_ERR_ARG, lambda q: q.update(word_id=np.arange(257, dtype=np.int32), word_value=np.ones(257)))
    for f in ('key', 'words', 'scored', 'score', 'nSharing', 'maxCommonWords', 'wordId'):
        query_fails(orb.ORB_ERR_ARG, struct_edit=lambda s, f=f: setattr(s, f, None))
    query_fails(orb.ORB_ERR_ARG, struct_edit=lambda s: setattr(s, 'nConnected', -1))
    query_fails(orb.ORB_ERR_ARG, struct_edit=lambda s: setattr(s, 'cap', -1))
    assert L.orbv_db_query_batch(db._h, 2, None) == orb.ORB_ERR_ARG
    one = (orb.OrbvDbQuery * 1)(orb.db_query_struct(q0, 30)[0])
    assert L.orbv_db_query_batch(db._h, 1 << 24, one) == orb.ORB_ERR_ARG                   # nQueries above 2^24 - 1
    assert ref['nSharing'] > 3
    out = query_fails(orb.ORB_ERR_CAPACITY, cap=ref['nSharing'] - 1)                       # the list is wider than cap
    assert int(out['nSharing'][0]) == ref['nSharing'] and out['key'].tobytes() == ref['key'][:ref['nSharing'] - 1].tobytes()
    with pytest.raises(orb.OrbError) as ei:
        db.query_batch([q0], cap=2)
    assert ei.value.code == orb.ORB_ERR_CAPACITY
    still_usable()
    db.add(1, [sc.key(k, 1) for k in range(10)], [sc.bows[k] for k in range(10)])         # every failed add left its slots free
    assert db.size(1) == 10
    add_fails(orb.ORB_ERR_CAPACITY, 1, [sc.key(10, 1)], [sc.bows[10]])


def _digest(outs, cap):
    h = 14695981039346656037
    for o in outs:
        for b in o['key'].tobytes() + o['words'].tobytes() + o['scored'].tobytes() + o['score'].tobytes() + o['nSharing'].tobytes() + \
                o['maxCommonWords'].tobytes():
            h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def test_cpp_keyframe_database_equals_python(orb, tmp_path):
    """ORB_SLAM3::KeyFrameDatabase (include/orb_b200/orb_slam3.hpp) from a g++-built caller gives the Python binding's digest."""
    D, cap = 3, 64
    scenes = [K.scene(500 + d, n_kf=30) for d in range(D)]
    adds = [(d, k) for d in range(D) for k in np.random.default_rng(d).permutation(scenes[d].n)[:25].tolist()]
    rng = np.random.default_rng(9)
    qs = [(d, _gpu_query(K.query_from(rng, scenes[d], 1 + i, i % 2), scenes[d], d)) for i in range(12) for d in [i % D]]
    start, ids, vals = K.flat_bows([scenes[d].bows[k] for d, k in adds])
    raw = dict(add_db=np.array([d for d, _ in adds], np.int32), add_key=np.array([scenes[d].key(k, d) for d, k in adds], np.uint64),
               add_start=start, add_id=ids, add_val=vals,
               q_meta=np.array([[d, q['kind'], len(q['word_id']), len(q['connected'])] for d, q in qs], np.int32),
               q_id=np.concatenate([q['word_id'] for _, q in qs]).astype(np.int32), q_val=np.concatenate([q['word_value'] for _, q in qs]),
               q_conn=np.array([c for _, q in qs for c in q['connected']], np.uint64))
    for n, a in raw.items():
        (tmp_path / (n + '.raw')).write_bytes(np.ascontiguousarray(a).tobytes())
    (tmp_path / 'dims.txt').write_text('%d %d %d %d %d\n' % (scenes[0].voc_words, D, 100, 256, cap))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'keyframe_database_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'keyframe_database_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    db = orb.KeyFrameDatabase(scenes[0].voc_words, max_databases=D, max_keyframes=100, max_words=256)
    db.add(raw['add_db'], raw['add_key'], [scenes[d].bows[k] for d, k in adds])
    built = [orb.db_query_struct(q, cap) for _, q in qs]
    arr = (orb.OrbvDbQuery * len(built))(*[b[0] for b in built])
    assert orb.lib().orbv_db_query_batch(db._h, len(built), arr) == orb.ORB_OK
    assert out['digest'] == '%016x' % _digest([b[1] for b in built], cap)
    assert int(out['sharing']) == sum(int(b[1]['nSharing'][0]) for b in built) > 20
    assert out['launches'] == '3'


def test_threads_of_different_systems_share_one_handle(orb):
    """Two threads, one database each, run add / erase / clear / query sequences on one handle at the same time (ctypes releases the
    GIL for the C calls): every record equals the oracle's, as when the calls run one after the other."""
    import threading
    scenes = [K.scene(900 + d, n_kf=40) for d in range(2)]
    seqs = [K.operations(70 + d, sc, n_ops=120) for d, sc in enumerate(scenes)]
    db = orb.KeyFrameDatabase(scenes[0].voc_words, max_databases=2, max_keyframes=80, max_words=512)
    got, errors = [[], []], []

    def run(d):
        try:
            sc = scenes[d]
            for op in seqs[d]:
                _apply(db, sc, d, op)
                if op[0] == 'query':
                    got[d].append(db.query_batch([_gpu_query(q, sc, d) for q in op[1]]))
        except Exception as e:                                    # reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=run, args=(d,)) for d in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    for d, sc in enumerate(scenes):
        o = K.Oracle(sc)
        results = iter(got[d])
        n = 0
        for op in seqs[d]:
            o.apply(op)
            if op[0] == 'query':
                for q, g in zip(op[1], next(results)):
                    assert K.same_record(_as_record(g, sc, d), o.query(q)[0]), (d, q['id'])
                    n += 1
        assert n > 50

