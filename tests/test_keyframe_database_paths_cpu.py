"""CPU tests of the KeyFrameDatabase scenes of tests/kfdb_scenes.py: on every case the oracle's phase-1 record and candidates equal the
restatement's (its numpy form, itself equal to the list-walking form on the smaller cases), and the cases reach the shapes they are
built for -- database sizes around the share kernel's 8 warps, the order kernel's 512-entry tile and bpq = 128, about 5000 keyframes;
nSharing > 1024; more than 1024 scored entries, of tied first ranks spread over several tiles; every word count of SWEEP_NW / WIDE_NW
up to 8192; first ranks 4095, 4096 and 8191; rows of 8192 words; slot orders that differ from add order, and a slot reused by a
3-word keyframe after an 8192-word one; two databases under equal keys; NBEST queries of more than 1024 connected keys."""
import functools

import numpy as np
import pytest

import kfdb_scenes as S
import keyframe_database_lib as K

NARROW, WIDE = S.NARROW_NAMES, S.WIDE_NAMES


def _case(name):
    return next(c for c in S.narrow_cases() + S.wide_cases() if c.name == name)


@functools.lru_cache(maxsize=None)
def _run(name):
    """Oracle and restatement through the case: per query (query, oracle record, restatement record)."""
    c = _case(name)
    o, r = K.Oracle(c.sc), K.Restatement(c.sc)
    for op in c.ops:
        o.apply(op)
        r.apply(op)
    out = []
    for q in c.queries:
        rec, cands = o.query(q)
        mine = r.phase1_np(q)
        assert K.same_record(rec, mine), (name, q['id'])
        assert r.phase2(q, mine) == cands, (name, q['id'])
        if len(r.live) <= 600:
            assert K.same_record(r.phase1(q), mine), (name, q['id'])
        out.append((q, rec, mine))
    return r.live, out


@pytest.mark.parametrize('name', NARROW + WIDE)
def test_oracle_equals_restatement(name):
    live, out = _run(name)
    c = _case(name)
    assert live == c.live()
    wide = name in WIDE
    assert all(len(q['word_id']) <= (S.WIDE_WORDS if wide else S.NARROW_WORDS) for q, _, _ in out)
    assert all(len(c.sc.bows[k][0]) <= (S.WIDE_WORDS if wide else S.NARROW_WORDS) for k in live)


def test_database_sizes():
    assert [c.name for c in S.narrow_cases()] == NARROW and [c.name for c in S.wide_cases()] == WIDE
    sizes = {c.name: len(c.live()) for c in S.narrow_cases() + S.wide_cases()}
    for n in S.SWEEP_SIZES:
        assert sizes['size%d' % n] == n
    assert sizes['wide'] == 5000 and sizes['empty'] == 0
    big = max(sizes.values())
    assert min(-(-big // S.SH_WARPS), S.MAX_BPQ) == S.MAX_BPQ and big > S.MAX_BPQ * S.SH_WARPS       # warps loop in the share kernel


def test_word_counts_and_ranks():
    nw = {len(q['word_id']) for n in NARROW + WIDE for q, _, _ in _run(n)[1]}
    assert set(S.SWEEP_NW) | set(S.WIDE_NW) <= nw and {S.NARROW_WORDS, S.MAX_WORDS} <= nw
    assert any(12 * n > 48 * 1024 for n in nw) and 12 * 4096 == 48 * 1024                              # the score kernel's opt-in edge
    _, out = _run('top_ranks')
    full = [rec for q, _, rec in out if len(q['word_id']) == S.MAX_WORDS]
    assert full and all({0, 4095, 4096, 8191} <= set(rec['rank'].tolist()) for rec in full[:1])
    ranks = full[0]['rank'].tolist()
    assert ranks.count(4095) == 2 and ranks.count(8191) == 2                                           # ties in the top bits
    rows = [len(_case('top_ranks').sc.bows[k][0]) for k in _case('top_ranks').live()]
    assert rows.count(S.MAX_WORDS) == 3


def test_long_lists_and_many_scores():
    _, out = _run('wide')
    assert max(rec['nSharing'] for _, _, rec in out) > 4500
    assert max(int(rec['scored'].sum()) for _, _, rec in out) > 1024
    _, out = _run('tied')
    q, _, rec = out[0]
    assert rec['nSharing'] > 1024 and int((rec['words'] == rec['maxCommonWords']).sum()) > 1024 and int(rec['scored'].sum()) > 1024
    # keyframes of one first word spread over the tiles of the add-order list, between keyframes of the others
    c = _case('tied')
    pos = {k: i for i, k in enumerate(k for k in c.live() if k in set(rec['kf'].tolist()))}
    rank = dict(zip(rec['kf'].tolist(), rec['rank'].tolist()))
    add_order = sorted(pos, key=pos.get)
    for f in S.TIED_FIRST:
        tiles = {pos[k] // S.OR_NT for k in add_order if rank[k] == f}
        assert len(tiles) >= 3, (f, tiles)
    runs = sum(1 for a, b in zip(add_order, add_order[1:]) if rank[a] != rank[b])
    assert runs > 500


def test_score_values():
    """Scored keyframes and queries hold values from 1e-9 to 0.1 and above, zeros and negative values."""
    v = np.concatenate([np.concatenate([q['word_value'], *[c.sc.bows[k][1] for k in rec['kf'][rec['scored'] > 0]]])
                        for c in (_case('tied'), _case('top_ranks')) for q, _, rec in _run(c.name)[1]])
    a = np.abs(v[v != 0])
    assert (v == 0).any() and (v < 0).any() and a.min() < 1e-8 and a.max() > 0.1
    scores = np.concatenate([rec['score'][rec['scored'] > 0] for n in NARROW + WIDE for _, _, rec in _run(n)[1]])
    assert len(np.unique(scores)) > 1000 and (scores < 1e-6).any() and (scores > 1e-2).any()


@pytest.mark.parametrize('handle', ['narrow', 'wide'])
def test_slot_order_differs_from_add_order(handle):
    cases, n_slots = (S.narrow_cases(), S.NARROW_SLOTS) if handle == 'narrow' else (S.wide_cases(), S.WIDE_SLOTS)
    live, adds = S.slots(cases, n_slots)                          # IndexError if the handle ran out of slots
    for c, l in zip(cases, live):
        assert list(l) == c.live()
        if len(l) > 8:
            s = list(l.values())
            assert s != sorted(s), c.name
    if handle == 'wide':
        st = [i for i, c in enumerate(cases) if c.name == 'stale'][0]
        slot = {k: s for i, k, s in adds if i == st}
        c = cases[st]
        assert slot[0] == slot[1] and len(c.sc.bows[0][0]) == S.MAX_WORDS and len(c.sc.bows[1][0]) == 3
        assert set(c.sc.bows[0][0].tolist()) <= set(c.queries[0]['word_id'].tolist())


def test_pair_shares_keys_and_rows():
    a, b = _case('pair_a'), _case('pair_b')
    assert a.sc is b.sc and a.key_db == b.key_db
    la, lb = set(a.live()), set(b.live())
    assert len(la & lb) > 100
    for me, other in ((la, lb), (lb, la)):
        c = a if me is la else b
        nb = [q for q in c.queries if q['kind'] == K.NBEST]
        big = nb[0]
        conn = big['connected']
        assert len(conn) + len(big['absent']) > 1024 and len(set(conn)) < len(conn)
        assert set(conn) & me and set(conn) & (other - me) and big['absent']
        assert any(set(q['connected']) and set(q['connected']) <= other - me for q in nb)
    _, out = _run('pair_a')
    assert all(set(rec['kf'].tolist()) <= la for _, _, rec in out)
