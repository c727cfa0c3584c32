"""GPU tests of orbm_common_regions_bow_batch (LoopClosing::DetectCommonRegionsFromBoW's BoW sweep) against the CPU oracle
orbo_common_regions_bow: records byte for byte at 1 / 7 / 24 queries with the planted cases, per-pair counts against orbm_search_by_bow_kf,
batch against per-query calls and another query order, the launch count, every argument error and a g++-built C++ caller."""
import copy
import os
import subprocess

import numpy as np
import pytest

import common_regions_lib as CR
import oracle_lib as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def matcher(orb):
    return orb.ORBmatcher(0.6, False, max_batch=1, max_keypoints=2048, max_mappoints=2048)


def _queries(n, seed):
    """n queries: the planted ones first, then random queries of up to 6 candidates x 11 entries."""
    qs = CR.planted_queries(seed)[:n]
    rng = np.random.default_rng(seed)
    while len(qs) < n:
        qs.append(CR.random_query(seed * 1000 + len(qs), n_cand=int(rng.integers(1, 7)), n_feat=int(rng.integers(150, 400)), p_null_cand=0.05))
    return qs


def _same(got, want):
    for f in CR.FIELDS:
        assert got[f].dtype == want[f].dtype and np.array_equal(got[f], want[f]), f


@pytest.mark.parametrize('n', [1, 7, 24])
def test_batch_equals_oracle(matcher, n):
    qs = _queries(n, 5 + n)
    got = matcher.common_regions_bow_batch(qs)
    assert matcher.last_launch_count() == 2
    for q, g in zip(qs, got):
        _same(g, CR.oracle(q))
    if n == 24:
        assert sum(int((g['status'] == CR.RAN).sum()) for g in got) > 50
        assert max(int(g['numBoWMatches'].max(initial=0)) for g in got) >= 20


def test_nmatches_equal_single_searches(orb, matcher):
    """Each RAN entry's count is what orbm_search_by_bow_kf gives that pair alone with ORBmatcher(0.9, true)."""
    single = orb.ORBmatcher(0.9, True, max_batch=1, max_keypoints=2048, max_mappoints=2048)
    qs = _queries(7, 3)
    for q, g in zip(qs, matcher.common_regions_bow_batch(qs)):
        a = q['kfs'][0]
        for c in np.flatnonzero(g['status'] == CR.RAN):
            for j, e in enumerate(g['covList'][c]):
                if e < 0 or q['kfs'][e]['bad']:
                    continue
                b = q['kfs'][e]
                n, _ = single.SearchByBoWKF(a['kps'], a['desc'], CR.flags(q, 0), a['fv'], b['kps'], b['desc'], CR.flags(q, e), b['fv'])
                assert g['nmatches'][c][j] == n, (c, j)


def test_batch_equals_per_query_calls_and_any_order(orb, matcher):
    qs = _queries(7, 21)
    batch = matcher.common_regions_bow_batch(qs)
    for q, b in zip(qs, batch):
        _same(matcher.common_regions_bow_batch([q])[0], b)
    perm = np.random.default_rng(0).permutation(len(qs))
    for i, r in zip(perm, matcher.common_regions_bow_batch([qs[i] for i in perm])):
        _same(r, batch[i])
    # after other calls on the handle (the staging holds their data)
    a, b = qs[0]['kfs'][0], qs[0]['kfs'][1]
    matcher.SearchByBoWKF(a['kps'], a['desc'], CR.flags(qs[0], 0), a['fv'], b['kps'], b['desc'], CR.flags(qs[0], 1), b['fv'])
    matcher.common_regions_bow_batch(_queries(24, 8))
    for r, want in zip(matcher.common_regions_bow_batch(qs), batch):
        _same(r, want)


def test_launch_count_zero_without_a_ran_candidate(matcher):
    matcher.common_regions_bow_batch(_queries(1, 2))
    assert matcher.last_launch_count() == 2
    q = CR.planted_queries(4)[1]
    q['cand'] = [q['cand'][i] for i in (0, 3, 4, 5)]
    q['cov'] = [q['cov'][i] for i in (0, 3, 4, 5)]
    r = matcher.common_regions_bow_batch([q])[0]
    assert matcher.last_launch_count() == 0
    _same(r, CR.oracle(q))
    assert list(r['status']) == [CR.SKIPPED, CR.ABORTED_NEAR, CR.ABORTED_NEAR, CR.SKIPPED]
    assert matcher.common_regions_bow_batch([]) == [] and matcher.last_launch_count() == 0


def _bad_queries(orb):
    base = CR.random_query(1, n_cand=3, n_cov=(1, 3), p_bad_cand=0.0, p_bad_cov=0.0, p_conn=0.0)

    def edit(fn):
        q = copy.deepcopy(base)
        fn(q)
        return q

    def big(q, e, n):
        q['kfs'][e] = CR.keyframe(np.random.default_rng(0), CR.world(np.random.default_rng(1), n, 64), np.arange(n), p_null=1.0)

    def unsorted(q):
        nodes, feats = q['kfs'][1]['fv']
        q['kfs'][1]['fv'] = (nodes[::-1].copy(), feats)

    return {
        'cand out of range': edit(lambda q: q['cand'].__setitem__(0, len(q['kfs']))),
        'cand is the current keyframe': edit(lambda q: q['cand'].__setitem__(0, 0)),
        'cand below -1': edit(lambda q: q['cand'].__setitem__(0, -2)),
        'cov out of range': edit(lambda q: q['cov'][0].append(len(q['kfs']))),
        'cov is the current keyframe': edit(lambda q: q['cov'][0].append(0)),
        'more than 10 covisibles': edit(lambda q: q['cov'].__setitem__(0, [len(q['kfs']) - 1] * 11)),
        'point out of range': edit(lambda q: q['kfs'][1]['point'].__setitem__(0, len(q['pointBad']))),
        'point below -1': edit(lambda q: q['kfs'][0]['point'].__setitem__(0, -2)),
        'unsorted feature vector': edit(unsorted),
        'feature index out of range': edit(lambda q: q['kfs'][2]['fv'][1].__setitem__(0, len(q['kfs'][2]['kps']))),
        'current keyframe over max_mappoints': edit(lambda q: big(q, 0, 2049)),
        'covisible over max_keypoints': edit(lambda q: big(q, 1, 2049)),
        'no keyframe': edit(lambda q: q.__setitem__('kfs', [])),
    }


def test_argument_errors_before_any_launch(orb, matcher):
    bad = _bad_queries(orb)
    assert len(bad) == 13
    good = _queries(2, 9)
    for name, q in bad.items():
        matcher.common_regions_bow_batch(good)
        assert matcher.last_launch_count() == 2
        s, out, keep = orb.common_regions_struct(q)
        for v in out.values():
            v.fill(7)
        arr = (orb.OrbmCommonRegionsQuery * 2)(orb.common_regions_struct(good[0])[0], s)
        rc = orb.lib().orbm_common_regions_bow_batch(matcher._h, 2, arr)
        assert rc == orb.ORB_ERR_ARG, name
        assert matcher.last_launch_count() == 2, name
        assert all((v == 7).all() for v in out.values()), name
    L = orb.lib()
    assert L.orbm_common_regions_bow_batch(matcher._h, -1, None) == orb.ORB_ERR_ARG
    assert L.orbm_common_regions_bow_batch(matcher._h, 1, None) == orb.ORB_ERR_ARG
    assert L.orbm_common_regions_bow_batch(None, 0, None) == orb.ORB_ERR_ARG


def _digest(recs):
    h = 14695981039346656037
    for r in recs:
        for f in CR.FIELDS:
            for b in r[f].tobytes():
                h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def test_cpp_common_regions_bow_batch_equals_python(orb, matcher, tmp_path):
    """ORBmatcher::CommonRegionsBoWBatch (include/orb_b200/orb_slam3.hpp) from a g++-built caller gives the Python binding's digest."""
    qs = _queries(7, 13)
    lines = [str(len(qs))]
    for i, q in enumerate(qs):
        lines.append('%d %d %d' % (len(q['kfs']), len(q['pointBad']), len(q['cand'])))
        lines.append(' '.join(str(int(c)) for c in q['cand']))
        lines.append(' '.join(str(len(c)) for c in q['cov']))
        lines.append(' '.join(str(int(e)) for c in q['cov'] for e in c))
        (tmp_path / ('q%d_pointBad.raw' % i)).write_bytes(np.ascontiguousarray(q['pointBad'], np.uint8).tobytes())
        for e, kf in enumerate(q['kfs']):
            lines.append('%d %d %d %d' % (len(kf['kps']), len(kf['fv'][0]), int(kf['bad']), int(kf['connected'])))
            for name, a in (('kps', np.ascontiguousarray(kf['kps'], O.KP_DTYPE)), ('desc', np.ascontiguousarray(kf['desc'], np.uint8)),
                            ('fvNode', np.ascontiguousarray(kf['fv'][0], np.int32)), ('fvFeature', np.ascontiguousarray(kf['fv'][1], np.int32)),
                            ('point', np.ascontiguousarray(kf['point'], np.int32))):
                (tmp_path / ('q%d_kf%d_%s.raw' % (i, e, name))).write_bytes(a.tobytes())
    (tmp_path / 'dims.txt').write_text('\n'.join(lines) + '\n')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'common_regions_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'common_regions_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    res = matcher.common_regions_bow_batch(qs)
    assert out['digest'] == '%016x' % _digest(res)
    assert int(out['ran']) == sum(int((r['status'] == CR.RAN).sum()) for r in res) > 5
    assert out['launches'] == '2'
