"""CPU tests of the DBoW2 transform's oracle on the vocabularies and frames of tests/bow_scenes.py: the oracle (oracle/bow_oracle.cpp,
pinned to the reference's own DBoW2 by tests/test_ref_pins_oracle_cpu.py) equals bow_scenes' numpy restatement of the transform word for
word, value for value bit for bit (the L2 norm's fused multiply-adds rounded exactly) and entry for entry; every FeatureVector node is
its feature's leaf's ancestor at depth L - levelsup; L1-normalised values sum to 1."""
import math

import numpy as np
import pytest

import bow_scenes as B
import matcher_scenes as S
import oracle_lib as O

PAIRS = [(w, n) for w in range(4) for n in range(3)]        # weighting (TF_IDF, TF, IDF, BINARY) x norm (none, L1, L2)


def levelsups(voc):
    return (0, 1, voc['L'] - 1, voc['L'], voc['L'] + 3)


def check(voc, feats, levelsup, weighting, norm):
    """The three checks of this file on one frame; returns the oracle's result."""
    ref = O.bow_transform(voc, feats, levelsup, weighting, norm)
    got = B.transform(voc, feats, levelsup, weighting, norm)
    what = (len(feats), levelsup, weighting, norm)
    assert np.array_equal(got[0], ref[0]) and got[1].tobytes() == ref[1].tobytes(), what
    assert np.array_equal(got[2], ref[2]) and np.array_equal(got[3], ref[3]), what
    nid_level = voc['L'] - levelsup
    leaf = B.descend(voc, feats, levelsup)[0][ref[3]]
    if nid_level <= 0:
        assert not ref[2].any(), what
    else:
        deep = voc['depth'][leaf] >= nid_level       # leaves above nid_level: test_leaf_above_nid_level_is_filed_under_node_0
        assert np.array_equal(ref[2][deep], B.ancestor(voc, leaf[deep], nid_level)), what
    if norm == 1 and len(ref[1]):
        # the norm is a recursive sum of n positive terms (relative error below (n - 1) 2^-53) and each quotient adds half an ulp, so
        # the exact sum of the quotients is within n 2^-53 of 1 (a fixed 1e-15 fails: a 1000-word frame already sums to 1 + 1.1e-15)
        assert abs(math.fsum(ref[1]) - 1.0) <= len(ref[1]) * 2.0 ** -53, (what, math.fsum(ref[1]) - 1.0)
    return ref


@pytest.mark.parametrize('name', sorted(B.TREES))
def test_trees(name):
    voc = B.vocabulary(name)
    fr = B.frames(voc, seed=len(name))
    for feats in fr:
        for ls in levelsups(voc):
            check(voc, feats, ls, 0, 1)
        for w, n in PAIRS:
            check(voc, feats, 2, w, n)


@pytest.mark.parametrize('name', sorted(B.TREES))
def test_trees_are_what_they_claim(name):
    """Each tree has what its builder promises: the root's k children and one leaf, nodes with 1..k children, leaves at several depths,
    one directly under the root, child lists out of id order, stopped words at the asked fraction; every planted tie is reached and
    always resolved to its first position."""
    kw, voc = B.TREES[name], B.vocabulary(name)
    cs, ch = voc['child_start'], voc['children']
    count = np.diff(cs)
    leaves = np.flatnonzero(count == 0)
    assert count[0] == kw['k'] + 1 and count[count > 0].max() <= kw['k'] + 1 and count[1:][count[1:] > 0].max() <= kw['k']
    assert (voc['depth'][ch[:count[0]]] == 1).all() and (count[ch[:count[0]]] == 0).any()
    assert len(set(voc['depth'][leaves])) >= 2
    descending = np.diff(ch) < 0
    descending[cs[1:-1][cs[1:-1] < len(descending)] - 1] = False        # pairs across two lists
    assert descending.any() == kw.get('shuffle', True) or kw['k'] == 1
    assert (voc['weight'][leaves] == 0).sum() == round(kw.get('stop', 0.02) * len(leaves))
    assert sorted(voc['word_id'][leaves]) == list(range(len(leaves)))
    assert (np.diff(voc['word_id'][leaves]) < 0).any() == kw.get('permute_words', True) or kw['k'] == 1
    planted = [(p, q) for _, p, q in voc['ties']]
    assert (0, 1) in planted and ((15, 16) in planted) == (kw['k'] >= 16) and ((16, 32) in planted) == (kw['k'] >= 32)
    for (p, q), (hp, hq) in zip(planted, B.tie_hits(voc, np.concatenate(B.frames(voc, seed=len(name))))):
        assert hp > 0 and hq == 0, (p, q, hp, hq)


def test_orbvoc_shape():
    """ORBvoc.txt's shape (k = 10, L = 6, TF_IDF, L1) with ComputeBoW's levelsup = 4, on real ORB features."""
    voc = B.vocabulary('orbvoc')
    assert len(voc['parent']) == 1111111 and voc['n_words'] == 10 ** 6
    for nf in (1000, 2000, 5000):
        feats = S.extract(5, nf=nf)[1]
        ref = check(voc, feats, 4, 0, 1)
        assert len(ref[0]) > 0.8 * len(feats)


def test_leaf_above_nid_level_is_filed_under_node_0():
    """A leaf above depth L - levelsup: DBoW2 never assigns nid on that descent (its value is whatever the caller's variable held); the
    library and the oracle file the feature under node 0, the root."""
    voc = B.vocabulary('k16_L4')
    cs, ch = voc['child_start'], voc['children']
    root_leaf = [c for c in ch[:cs[1]] if cs[c + 1] == cs[c]]
    feats = np.concatenate([B.near(voc, root_leaf, 50, seed=1, max_flips=0), B.frames(voc, seed=2)[1]])
    leaf = B.descend(voc, feats, 0)[0]
    assert (voc['depth'][leaf[:50]] == 1).all() and (voc['depth'][leaf[50:]] > 2).any()
    for ls in (1, 2):
        ref = check(voc, feats, ls, 0, 1)
        above = voc['depth'][leaf[ref[3]]] < voc['L'] - ls
        assert above.any() and not ref[2][above].any()


def test_edge_frames():
    """Every word stopped (nWords = nEntries = 0), and one word receiving 16384 features (their weights summed in feature order)."""
    voc = B.vocabulary('k17_stop_half')
    for feats in (B.stopped_frame(voc, 500, seed=3), B.stopped_frame(voc, 1, seed=4)):
        for w, n in PAIRS:
            ref = check(voc, feats, 1, w, n)
            assert len(ref[0]) == 0 and len(ref[2]) == 0
    feats = B.one_word_frame(voc, 16384, seed=5)
    for w, n in ((0, 0), (0, 1), (1, 2), (2, 0), (3, 1)):
        ref = check(voc, feats, 2, w, n)
        assert len(ref[0]) == 1 and np.array_equal(ref[3], np.arange(16384))
    voc = B.vocabulary('k10_stop_all')
    for feats in B.frames(voc, seed=6):
        ref = check(voc, feats, 1, 0, 1)
        assert len(ref[0]) == 0 and len(ref[2]) == 0
