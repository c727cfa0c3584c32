"""CPU tests of KeyFrameDatabase: the oracle (oracle/keyframe_database_oracle.cpp, the reference's text over a pointer model) equals the
independent restatement of tests/keyframe_database_lib.py -- phase-1 records and both detections' candidates -- on random add / erase /
clear / clearMap / query sequences, with the thresholds, ties, stale scores and the NBEST spin planted; clearMap equals erase of the
map's keyframes; without a device orbv_db_create fails with ORB_ERR_CUDA."""
import numpy as np
import pytest

import keyframe_database_lib as K


def _run(sc, ops):
    """Drives the oracle and the restatement through `ops`; returns the restatement and what the sequence covered."""
    o, r = K.Oracle(sc), K.Restatement(sc)
    seen = dict(empty_db=0, no_share=0, connected_sharing=0, readd=0, spin=0, scored=0, unscored=0)
    last_erased = set()
    for op in ops:
        o.apply(op)
        r.apply(op)
        if op[0] == 'erase':
            last_erased = set(op[1])
        elif op[0] == 'add':
            seen['readd'] += bool(last_erased & set(op[1]))
        if op[0] != 'query':
            continue
        for q in op[1]:
            rec, cands = o.query(q)
            mine = r.phase1(q)
            assert K.same_record(rec, mine), (q['id'], rec, mine)
            assert r.phase2(q, mine) == cands, q['id']
            seen['empty_db'] += not r.live
            seen['no_share'] += bool(r.live) and rec['nSharing'] == 0
            seen['spin'] += cands == K.SPIN
            seen['scored'] += int(rec['scored'].sum())
            seen['unscored'] += int((rec['scored'] == 0).sum())
            if q['kind'] == K.NBEST:
                qw = set(q['word_id'].tolist())
                seen['connected_sharing'] += any(k in r.live and qw & set(sc.bows[k][0].tolist()) for k in q['connected'])
    # the inverted file itself: each word's list is the live keyframes that hold it, in add order
    for w in range(0, sc.voc_words, 7):
        assert o.word_list(w) == [k for k in r.live if w in set(sc.bows[k][0].tolist())]
    return r, seen


@pytest.mark.parametrize('D', [1, 7, 24])
def test_oracle_equals_restatement(D):
    total = dict(ties=0, stale=0)
    seen_all = {}
    for d in range(D):
        sc = K.scene(100 * D + d, frac_bad=0.15 if d % 3 == 2 else 0.0)
        r, seen = _run(sc, K.operations(7 * D + d, sc, n_ops=50))
        total['ties'] += r.ties
        total['stale'] += r.stale_reads
        for k, v in seen.items():
            seen_all[k] = seen_all.get(k, 0) + v
    for k in ('empty_db', 'no_share', 'connected_sharing', 'readd', 'scored', 'unscored'):
        assert seen_all[k] > 0, (k, seen_all)
    assert total['ties'] > 0 and total['stale'] > 0, total
    if D > 2:
        assert seen_all['spin'] > 0


def test_planted_thresholds():
    """max = 5, 10, 15, 20: max * 0.8f is an integer, and a keyframe with exactly that many common words is not scored."""
    sc = K.planted_scene()
    o, r = K.Oracle(sc), K.Restatement(sc)
    op = ('add', list(range(sc.n)))
    o.apply(op)
    r.apply(op)
    for j, q in enumerate(K.planted_queries(1)):
        m = (5, 10, 15, 20)[j]
        rec, cands = o.query(q)
        mine = r.phase1(q)
        assert K.same_record(rec, mine)
        assert r.phase2(q, mine) == cands
        assert rec['maxCommonWords'] == m and rec['nSharing'] == 3
        by_words = dict(zip(rec['words'].tolist(), rec['scored'].tolist()))
        assert by_words == {m: 1, m * 4 // 5: 0, m * 4 // 5 + 1: 1}


def test_clear_map_equals_erase_of_its_keyframes():
    sc = K.scene(5, n_kf=40)
    rng = np.random.default_rng(11)
    order = rng.permutation(sc.n).tolist()
    gone = order[5:15]
    ops = [('add', order[:20]), ('add', order[20:]), ('erase', gone), ('add', gone[::2])]       # erased, some re-added
    a, b, r = K.Oracle(sc), K.Oracle(sc), K.Restatement(sc)
    for op in ops:
        a.apply(op); b.apply(op); r.apply(op)
    m = int(sc.kf_map[r.live[0]])
    a.apply(('clearMap', m))
    b.apply(('erase', [k for k in range(sc.n) if sc.kf_map[k] == m]))
    for w in range(sc.voc_words):
        assert a.word_list(w) == b.word_list(w)
    for i in range(20):
        q = K.query_from(rng, sc, 100 + i, i % 2)
        assert K.same_record(a.query(q)[0], b.query(q)[0])


def test_frame_scene_oracle_equals_restatement():
    """BowVectors of real ORB features (matcher_scenes frames) through the oracle's DBoW2 transform."""
    sc, _, _ = K.frame_scene(2)
    _, seen = _run(sc, K.operations(4, sc, n_ops=30))
    assert seen['scored'] > 0


def test_no_device_is_an_error():
    import ctypes as C
    import torch
    import orb_slam3_modified_b200 as orb
    if torch.cuda.is_available():
        pytest.skip('GPU present')
    h = C.c_void_p()
    assert orb.lib().orbv_db_create(C.byref(h), 1000, 1, 16, 64, 0) == orb.ORB_ERR_CUDA
    with pytest.raises(orb.OrbError) as ei:
        orb.KeyFrameDatabase(1000)
    assert ei.value.code == orb.ORB_ERR_CUDA
