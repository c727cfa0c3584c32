"""LocalMapping::SearchInNeighbors for a batch of keyframes of different maps in lockstep rounds (tests/search_in_neighbors_lib.py) equals
the reference's keyframe-after-keyframe order, with the CPU oracle's Fuse search: every keyframe's mvpMapPoints and every point's
observations, bad flag, descriptor, found / visible and mnFuseCandidateForKF.  Each bookkeeping rule is shown to fire, and a driver
that searches with the descriptors of before the first round differs (a single launch for all targets would not be exact)."""
import numpy as np
import pytest

import oracle_lib as O
import search_in_neighbors_lib as SN


@pytest.fixture(scope='module')
def g():
    return SN.globals_()


class CountingOracle(SN.OracleBackend):
    def __init__(self):
        self.calls = 0

    def fuse(self, items):
        self.calls += bool(items)
        return super().fuse(items)


CASES = [  # (n keyframes, targets per keyframe, aborted, keyframes without points, seed)
    (1, [4], (), (), 0),
    (4, [3, 0, 5, 2], (), (), 1),
    (6, [2, 4, 1, 0, 3, 5], (4,), (2,), 2),
    (3, [0, 0, 0], (), (1,), 3),
]


@pytest.mark.parametrize('n,nt,abort,nopts,seed', CASES)
def test_lockstep_equals_sequential(g, n, nt, abort, nopts, seed):
    a = SN.make_jobs(g, n, seed, nt, abort, nopts)
    b = SN.make_jobs(g, n, seed, nt, abort, nopts)
    assert [j['map'].state() for j in a] == [j['map'].state() for j in b]        # the scenes are seeded
    be_a, be_b = CountingOracle(), CountingOracle()
    ev_a = SN.lockstep(be_a, a)
    ev_b = SN.sequential(be_b, b)
    for s, (ja, jb) in enumerate(zip(a, b)):
        assert ja['map'].state() == jb['map'].state(), s
    assert ev_a == ev_b
    live = [j for j in a if not j['abort']]
    assert be_a.calls == max(nt) + bool(live)                                    # max |T| + 1 searches ...
    assert be_b.calls == sum(nt) + len(live)                                     # ... instead of sum(|T| + 1)
    if sum(nt):                                                                  # the bookkeeping did something
        assert ev_a['add'] > 0 and ev_a['replace_into_kf'] + ev_a['replace_from_kf'] > 0


def test_every_rule_fires(g):
    jobs = SN.make_jobs(g, 4, 1, [3, 0, 5, 2])
    ev = SN.lockstep(SN.OracleBackend(), jobs)
    assert ev['replace_into_kf'] > 0                 # pMP->Replace(pMPinKF): pMPinKF has more observations
    assert ev['replace_from_kf'] > 0                 # pMPinKF->Replace(pMP)
    assert ev['pin_bad'] > 0                         # pMPinKF->isBad(): nothing happens, nFused still counts
    assert ev['add'] > 0                             # AddObservation + AddMapPoint
    assert ev['in_kf_later'] > 0                     # IsInKeyFrame became true for a later target (a Replace handed the point that keyframe)
    assert ev['pass2_dup'] > 0 and ev['pass2_bad'] > 0   # pass 2: mnFuseCandidateForKF deduplication and bad points left out
    assert ev['empty_items'] > 0                     # the keyframe without targets searches an empty candidate list


def test_pass2_candidates_are_unique(g):
    jobs = SN.make_jobs(g, 2, 5, [4, 3])
    seen = []

    class Spy(SN.OracleBackend):
        def fuse(self, items):
            seen.append(items)
            return super().fuse(items)
    SN.lockstep(Spy(), jobs)
    last = seen[-1]                                  # the pass-2 call
    assert len(last) == 2
    for it in last:
        assert len(it['pids']) == len(set(it['pids'])) and len(it['pids']) > 0


def test_stale_descriptors_change_later_results(g):
    """Replace recomputes the absorbing point's descriptor (MapPoint::Replace -> ComputeDistinctiveDescriptors).  Searching later targets
    with the descriptors of before the first round changes some search results, and the final map state."""
    live = SN.make_jobs(g, 4, 1, [3, 0, 5, 2])
    init = {(id(j['map']), p.id): p.desc.copy() for j in live for p in j['map'].pts}
    changed = []

    class Compare(SN.OracleBackend):
        def fuse(self, items):
            out = super().fuse(items)
            for it, (bi, bd) in zip(items, out):
                st = dict(it, mp_desc=np.array([init[(id(it['map']), p)] for p in it['pids']], np.uint8).reshape(-1, 32))
                sbi, sbd = O.fuse_search(st, it['th'])
                diff = (it['state'] == 1) & ((sbi != bi) | (sbd != bd))
                changed.append(int(diff.sum()))
            return out
    SN.lockstep(Compare(), live)
    assert sum(changed) > 0
    stale = SN.make_jobs(g, 4, 1, [3, 0, 5, 2])
    SN.lockstep(SN.OracleBackend(), stale, stale=True)
    differ = [a['map'].state() != b['map'].state() for a, b in zip(live, stale)]
    assert any(differ) and not differ[1]             # keyframe 1 has no targets: nothing can go stale


def test_one_keyframe_per_map(g):
    jobs = SN.make_jobs(g, 1, 0, [2])
    with pytest.raises(AssertionError):
        SN.lockstep(SN.OracleBackend(), jobs + [dict(jobs[0])])
