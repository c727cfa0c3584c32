"""CPU tests of LoopClosing::DetectCommonRegionsFromBoW's oracle (oracle/common_regions_oracle.cpp) against the Python restatement of
tests/common_regions_lib.py, on seeded queries and on the planted cases of the candidate loop and the merge.  No GPU needed."""
import collections

import numpy as np
import pytest

import common_regions_lib as CR
import oracle_lib as O


def check(q, events=None):
    """Oracle == restatement on every record field; returns the oracle's record."""
    got = CR.oracle(q)
    want = CR.as_arrays(CR.restate(q, events), len(q['kfs'][0]['kps']))
    for f in CR.FIELDS:
        assert np.array_equal(got[f], want[f]), f
    return got


@pytest.mark.parametrize('seed', range(6))
def test_oracle_equals_restatement_on_random_queries(seed):
    q = CR.random_query(seed, n_cand=6, n_feat=250, p_null_cand=0.1)
    rec = check(q)
    assert (rec['status'] == CR.RAN).any()


def test_planted_cases():
    """Every planted case of the loop and the merge is met, and the oracle equals the restatement on each query."""
    ev = collections.Counter()
    recs = [(q, check(q, ev)) for q in CR.planted_queries(11)]
    assert ev['overwrite'] > 0                 # a later j overwrote slot k with a new point
    assert ev['seen_diff_k'] > 0               # a point shared by two covisibles at different k: the later one ignored
    assert ev['seen_same_k'] > 0               # a later j bringing an already-seen point at the same k: ignored
    q, r = recs[1]
    assert list(r['status']) == [CR.SKIPPED, CR.RAN, CR.RAN, CR.ABORTED_NEAR, CR.ABORTED_NEAR, CR.SKIPPED]
    assert list(r['covList'][1]) == [q['cand'][1]] + [-1] * 10                        # empty covisible list: the candidate alone
    cov2 = q['cov'][2]
    assert list(r['covList'][2][:len(cov2) + 1]) == [q['cand'][2]] + cov2[1:] + [cov2[0]]   # cov0 moved to the end
    jb = list(r['covList'][2]).index(cov2[-1])                                        # the bad covisible is skipped
    assert r['nmatches'][2][jb] == -1 and (np.delete(r['nmatches'][2][:len(cov2) + 1], jb) >= 0).all()
    assert not (r['matchedCov'][2] == jb).any()
    assert (r['numBoWMatches'][[0, 3, 4, 5]] == 0).all() and (r['matchedCov'][[0, 3, 4, 5]] == -1).all()
    q, r = recs[2]                             # current keyframe without map points
    assert (r['status'] == CR.RAN).all() and (r['numBoWMatches'] == 0).all() and (r['nmatches'][r['covList'] >= 0] == 0).all()
    q, r = recs[3]                             # a zero-feature covisible
    e = q['cov'][0][1]
    j = list(r['covList'][0]).index(e)
    assert r['nmatches'][0][j] == 0
    q, r = recs[4]                             # a zero-feature current keyframe
    assert r['matchedCov'].shape == (2, 0) and (r['numBoWMatches'] == 0).all()
    q, r = recs[5]
    assert list(r['numBoWMatches']) == [19, 20]


def test_orientation_rejects_matches():
    """The rotation histogram removes matches: SearchByBoW with the orientation check finds fewer than without it on some entry."""
    q = CR.random_query(3, n_cand=2, n_cov=(2, 4), p_bad_cand=0.0, p_bad_cov=0.0, p_conn=0.0)
    a = q['kfs'][0]
    fewer = 0
    for e in range(1, len(q['kfs'])):
        b = q['kfs'][e]
        n1, _ = O.search_by_bow_kf(a['kps'], a['desc'], CR.flags(q, 0), a['fv'], b['kps'], b['desc'], CR.flags(q, e), b['fv'], nnratio=0.9, check_ori=True)
        n0, _ = O.search_by_bow_kf(a['kps'], a['desc'], CR.flags(q, 0), a['fv'], b['kps'], b['desc'], CR.flags(q, e), b['fv'], nnratio=0.9, check_ori=False)
        fewer += n1 < n0
    assert fewer > 0
    check(q)
