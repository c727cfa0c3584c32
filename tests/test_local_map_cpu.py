"""CPU tests of the UpdateLocalMap oracle (oracle/local_map_oracle.cpp): it equals the independent Python restatement on seeded scenes of
both vote branches, monocular and inertial, and on planted scenes for each rule of UpdateLocalKeyFrames / UpdateLocalPoints; its slabs
hold the local points' rows and lastToLocal their local indices."""
import numpy as np
import pytest

import local_map_lib as L
import orb_slam3_modified_b200 as orb


def _check(scenes, mcap=4096):
    """Oracle == restatement on every scene of one batch; returns the restatements."""
    d, out, orders = L.run_oracle(scenes, mcap)
    res = orb.local_map_split(d, out)
    got = []
    for sc, (table, points), r in zip(scenes, orders, res):
        want = L.restate(sc)
        assert L.replay(sc, table, points, r) == want
        pi = {p: i for i, p in enumerate(points)}
        local = {p: i for i, p in enumerate(want['localPoint'])}
        src = [pi[p] if p is not None else -1 for p in sc.src]
        assert r['lastToLocal'].tolist() == [local.get(points[j], -1) if j >= 0 else -1 for j in src]
        got.append(want)
    for b, sc in enumerate(scenes):                     # the slab rows are the points' fields
        nM = int(out['nM'][b])
        rows = out['localPoint'][b, :nM]
        p0 = int(d['pointStart'][b])
        for k in ('worldPos', 'normal', 'minDistInv', 'maxDistInv', 'maxDistance', 'mpDesc', 'hasObs'):
            assert out[k][b, :nM].tobytes() == np.ascontiguousarray(d[k][p0 + rows]).tobytes(), k
        assert not out['bad'][b].any() and (out['localPoint'][b, nM:] == -1).all() and not out['worldPos'][b, nM:].any()
    return got


@pytest.mark.parametrize('vote_last,inertial,trk', [(False, False, False), (False, True, False), (True, True, False), (False, False, True),
                                                     (True, False, False)])
def test_oracle_equals_restatement_on_seeded_scenes(vote_last, inertial, trk):
    scenes = [L.scene(100 * s + 7, n_kf=20 + 13 * s, vote_last=vote_last, inertial=inertial, trk_space=trk) for s in range(6)]
    got = _check(scenes)
    assert any(len(g['localKF']) > len(set(k for p in L.vote_points(sc) for k in sc.pts[p].obs if not sc.kfs[k].bad))
               for g, sc in zip(got, scenes))          # the expansion adds keyframes
    assert all(g['localPoint'] for g in got)


def test_the_80_cap_and_many_voters():
    sc = L.scene(3, n_kf=200, n_pts=3000, window=(2, 4), n_src=900)
    sc.src = [p for k in range(200) for p in sc.kfs[k].slots[:3] if p is not None]
    sc.match = list(range(len(sc.src)))
    g = _check([sc])[0]
    assert len(g['localKF']) > 81                       # more than 80 voters: no expansion at all
    few = L.chain(120)
    L.vote_for(few, {k: 1 for k in range(78)})
    for k in range(78):
        few.kfs[k].cov = [78 + (k % 40)]
    g = _check([few])[0]
    assert len(g['localKF']) == 81                      # expansion stops once the size passes 80


def test_parent_breaks_the_voter_loop_and_bad_parent_is_added():
    sc = L.chain(10)
    L.vote_for(sc, {0: 1, 1: 1, 2: 1})
    sc.kfs[1].cov = [5]
    sc.set_parent(1, 6)
    sc.kfs[6].bad = True                                # a bad parent is still added
    sc.kfs[2].cov = [7]                                 # never reached: the parent push of voter 1 breaks the loop
    g = _check([sc])[0]
    assert g['localKF'] == [0, 1, 2, 5, 6]


def test_bad_voters_and_neighbours_children_order_and_tie():
    sc = L.chain(12, key=lambda j: 1000 - 8 * j)        # pointer order is the reverse of the id order
    L.vote_for(sc, {3: 2, 4: 2, 5: 1, 6: 3})
    sc.kfs[6].bad = True                                # the largest count, but bad: skipped
    sc.kfs[3].cov = [6, 8, 9]                           # 6 bad, so 8
    for c in (9, 10, 11):
        sc.set_parent(c, 4)                             # children in key order: 11 first
    g = _check([sc])[0]
    assert g['refKF'] == 4                              # tie 3 / 4: 4 comes first in key order
    assert g['localKF'][:3] == [5, 4, 3] and 11 in g['localKF']


def test_duplicate_votes_and_bad_points_of_the_voting_frame():
    sc = L.chain(6)
    L.vote_for(sc, {1: 2, 2: 3})
    sc.match = [0, 0, 0, 1, 2, 3, 4]                    # keyframe 1's first point held three times: 4 votes against 3
    g = _check([sc])[0]
    assert g['refKF'] == 1
    sc.pts[sc.src[0]].bad = True                        # now NULLed and not voting
    g = _check([sc])[0]
    assert g['refKF'] == 2 and g['frame'][:3] == [None] * 3
    sc.vote_last = True                                 # the last frame votes: each entry once
    g = _check([sc])[0]
    assert g['refKF'] == 2 and g['frame'][0] is None


def test_stalled_temporal_walk():
    sc = L.chain(30)
    sc.inertial, sc.last_kf = True, 29
    L.vote_for(sc, {27: 1})                             # 27 is a voter: the walk adds 29, 28 and stalls at 27
    g = _check([sc])[0]
    assert g['localKF'] == [27, 29, 28]
    sc.inertial = False
    assert _check([sc])[0]['localKF'] == [27]


def test_reverse_order_decides_shared_points():
    sc = L.chain(4)
    L.vote_for(sc, {0: 1, 1: 1})
    shared = sc.add_point([0, 1])
    late = sc.add_point([1])
    g = _check([sc])[0]
    assert g['localKF'] == [0, 1]
    assert g['localPoint'] == [sc.src[1], shared, late, sc.src[0]]      # keyframe 1's slots first


def test_overflow_leaves_no_rows():
    sc = L.scene(5)
    d, out, _ = L.run_oracle([sc, L.scene(6)], mcap=20)
    assert (out['nM'] > 20).all() and (out['localPoint'] == -1).all() and (out['lastToLocal'] == -1).all() and not out['worldPos'].any()


def test_planted_scenes_of_the_gpu_tests():
    got = _check(L.planted())
    assert len(got[0]['localKF']) > 256 // 2 and len(got[1]['localKF']) == 81
    assert got[7]['localKF'][:3] == [0, 50, sorted(range(1, 46), key=lambda c: (c * 37) % 60)[38]]
    assert got[8]['refKF'] == 270 and got[9]['refKF'] == 20 and len(got[9]['localKF']) == 400
