"""GPU paths of the DBoW2 transform (orbv_transform_batch and its device form) against the oracle on the vocabularies of
tests/bow_scenes.py: word ids, the values' bytes, FeatureVector nodes and features, and the counts, for every tree shape (1 to 65
children, so a half-warp takes a node's children in up to five strides; leaves at mixed depths; shuffled child lists; planted sibling
ties), all weighting x norm pairs, levelsup 0 to L + 3, every sort tile of the assembly (cap 1 to 16384), odd caps where one warp holds
the end of a frame and the start of the next, the ORBvoc shape, and the refusals of malformed vocabularies and counts."""
import numpy as np
import pytest

import bow_scenes as B
import matcher_scenes as S
import oracle_lib as O

pytestmark = pytest.mark.gpu

CAPS = (1, 2, 15, 16, 17, 31, 32, 33, 511, 512, 513, 8192, 8193, 16384)


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


def handle(orb, voc, weighting=0, norm=1):
    return orb.ORBVocabulary(voc['L'], voc['child_start'], voc['children'], voc['desc'], voc['weight'], voc['word_id'], weighting, norm)


def same(got, ref, what):
    assert np.array_equal(got[0], ref[0]) and got[1].tobytes() == ref[1].tobytes(), ('BowVector', what)
    assert np.array_equal(got[2], ref[2]) and np.array_equal(got[3], ref[3]), ('FeatureVector', what)


def padded(frames, cap, seed):
    """desc [B, cap, 32] with random bytes past each frame's n, and n [B]."""
    desc = np.random.default_rng(seed).integers(0, 256, (len(frames), cap, 32)).astype(np.uint8)
    for b, f in enumerate(frames):
        desc[b, :len(f)] = f
    return desc, np.array([len(f) for f in frames], np.int32)


def host_call(orb, v, desc, n, cap, levelsup):
    """orbv_transform_batch on [B, cap] rows; outputs start filled with a pattern.  Returns (status, outputs)."""
    B_ = len(n)
    outs = [np.full((B_, cap), -7, np.int32), np.full((B_, cap), -7.0), np.full(B_, -7, np.int32), np.full((B_, cap), -7, np.int32),
            np.full((B_, cap), -7, np.int32), np.full(B_, -7, np.int32)]
    rc = orb.lib().orbv_transform_batch(v._h, B_, orb._ptr(desc), orb._ptr(n), cap, levelsup, *[orb._ptr(o) for o in outs])
    return rc, outs


def rows(outs, b):
    wid, wv, nw, fn, ff, ne = outs
    return wid[b, :nw[b]], wv[b, :nw[b]], fn[b, :ne[b]], ff[b, :ne[b]]


def run_padded(orb, v, frames, cap, levelsup, seed=0):
    rc, outs = host_call(orb, v, *padded(frames, cap, seed), cap, levelsup)
    assert rc == orb.ORB_OK, orb.lib().orb_last_error()
    return [rows(outs, b) for b in range(len(frames))]


def check_frames(got, voc, frames, levelsup, weighting=0, norm=1):
    for b, (g, f) in enumerate(zip(got, frames)):
        same(g, O.bow_transform(voc, f, levelsup, weighting, norm), (b, len(f), levelsup, weighting, norm))


@pytest.mark.parametrize('name', sorted(B.TREES))
def test_trees(orb, name):
    """Every tree of bow_scenes at levelsup 0, 1, L - 1, L and L + 3, TF_IDF / L1, its frames in one call."""
    voc = B.vocabulary(name)
    v = handle(orb, voc)
    fr = B.frames(voc, seed=len(name))
    for ls in (0, 1, voc['L'] - 1, voc['L'], voc['L'] + 3):
        check_frames(v.transform(fr, ls), voc, fr, ls)


def test_weighting_norm_pairs(orb):
    """The 12 weighting x norm pairs on one tree (nodes of 34 children, ties at (0, 1), (15, 16), (16, 32)), levelsup 0 to L + 3."""
    voc = B.vocabulary('k33_L3')
    fr = B.frames(voc, seed=3)
    for w in range(4):
        for n in range(3):
            v = handle(orb, voc, w, n)
            for ls in (0, 1, voc['L'] - 1, voc['L'], voc['L'] + 3):
                check_frames(v.transform(fr, ls), voc, fr, ls, w, n)


def _features(voc, n, seed):
    """n features: near the planted ties, near random nodes and random, interleaved."""
    if n == 0:
        return np.zeros((0, 32), np.uint8)
    rng = np.random.default_rng(seed)
    pool = np.concatenate([B.near(voc, B.tie_targets(voc), min(n, 3000), seed), rng.integers(0, 256, (n, 32)).astype(np.uint8)])
    return pool[rng.integers(0, len(pool), n)]


@pytest.mark.parametrize('cap', CAPS)
def test_caps(orb, cap):
    """Frames of n = 0, 1, cap - 1 and cap in one call at each cap: the sort tile n2 runs 1 .. 16384 (12 n2 bytes of shared memory, up
    to 196,608), with random bytes in the slots past n."""
    voc = B.vocabulary('k17_L4')
    v = handle(orb, voc)
    ns = (cap, 0, cap - 1, 1, cap)
    frames = [_features(voc, n, seed=cap + i) for i, n in enumerate(ns)]
    check_frames(run_padded(orb, v, frames, cap, 2, seed=cap), voc, frames, 2)


@pytest.mark.parametrize('cap', (15, 17, 31, 33, 513))
def test_odd_caps_short_next_to_full(orb, cap):
    """An odd cap puts the last feature of a frame and the first of the next in one warp; short frames (whose half-warps leave at once)
    sit before and after full ones."""
    voc = B.vocabulary('k64_L3')
    v = handle(orb, voc)
    ns = (cap, 1, cap, cap // 2, cap, 0, cap, 2, 1, cap)
    frames = [_features(voc, n, seed=7 * cap + i) for i, n in enumerate(ns)]
    check_frames(run_padded(orb, v, frames, cap, 1, seed=cap), voc, frames, 1)


def test_300_frames(orb):
    """One call of 300 frames of 0 to 2000 features."""
    voc = B.vocabulary('k64_L3')
    v = handle(orb, voc)
    rng = np.random.default_rng(300)
    ns = np.concatenate([[0, 1, 2000, 2000, 1999], rng.integers(0, 2001, 295)])
    pool = _features(voc, 20000, seed=301)
    frames = [pool[rng.integers(0, len(pool), n)] for n in ns]
    check_frames(run_padded(orb, v, frames, 2000, 1, seed=302), voc, frames, 1)


def test_cap_grows_and_shrinks(orb):
    """One handle whose cap goes up past 48 KiB of sort tile (the kernel's dynamic shared memory limit is raised part way) to 16384 and
    back down; every call equals the oracle."""
    voc = B.vocabulary('k16_L4')
    v = handle(orb, voc)
    for i, cap in enumerate((1, 100, 4096, 4097, 8192, 16384, 513, 16, 16384, 1)):
        frames = [_features(voc, n, seed=i * 3 + j) for j, n in enumerate((cap, cap // 3))]
        check_frames(run_padded(orb, v, frames, cap, 2, seed=i), voc, frames, 2)


def test_edge_frames(orb):
    """16384 copies of one descriptor (one word's 16384 weights summed in feature order by one thread), frames whose every word is
    stopped, and a vocabulary whose every word is stopped."""
    voc = B.vocabulary('k17_stop_half')
    one = B.one_word_frame(voc, 16384, seed=5)
    stopped = [B.stopped_frame(voc, 500, seed=3), B.stopped_frame(voc, 1, seed=4)]
    for w, n in ((0, 0), (0, 1), (1, 2), (2, 0), (3, 1)):
        v = handle(orb, voc, w, n)
        got = v.transform([one] + stopped, 2)
        check_frames(got, voc, [one] + stopped, 2, w, n)
        assert len(got[0][0]) == 1 and len(got[0][2]) == 16384 and all(len(g[0]) == len(g[2]) == 0 for g in got[1:])
    voc = B.vocabulary('k10_stop_all')
    fr = B.frames(voc, seed=6)
    got = handle(orb, voc).transform(fr, 1)
    check_frames(got, voc, fr, 1)
    assert all(len(g[0]) == len(g[2]) == 0 for g in got)


def test_leaf_above_nid_level_is_filed_under_node_0(orb):
    """A feature whose leaf lies above depth L - levelsup (here: the root's leaf child) is filed under node 0, as the oracle files it;
    DBoW2 leaves that node id unset."""
    voc = B.vocabulary('k16_L4')
    cs, ch = voc['child_start'], voc['children']
    root_leaf = [c for c in ch[:cs[1]] if cs[c + 1] == cs[c]]
    feats = np.concatenate([B.near(voc, root_leaf, 50, seed=1, max_flips=0), B.frames(voc, seed=2)[1]])
    v = handle(orb, voc)
    for ls in (1, 2):
        got = v.transform([feats], ls)[0]
        same(got, O.bow_transform(voc, feats, ls), ls)
        assert set(range(50)) <= set(got[3][got[2] == 0].tolist())


@pytest.fixture(scope='module')
def orbvoc(orb):
    voc = B.vocabulary('orbvoc')
    return voc, handle(orb, voc)


@pytest.mark.parametrize('nf', (1000, 2000, 5000))
def test_orbvoc(orbvoc, nf):
    """ORBvoc.txt's shape (k = 10, L = 6, 1,111,111 nodes, TF_IDF, L1) with ComputeBoW's levelsup = 4 on real ORB features."""
    voc, v = orbvoc
    fr = [S.extract(t, nf=nf)[1] for t in (5, 6)]
    check_frames(v.transform(fr, 4), voc, fr, 4)


def _device_buffers(torch, B_, cap, fill=-7):
    i32 = dict(dtype=torch.int32, device='cuda')
    scratch = (torch.full((B_, cap), fill, **i32), torch.full((B_, cap), float(fill), dtype=torch.float64, device='cuda'),
               torch.full((B_, cap), fill, **i32))
    out = (torch.full((B_, cap), fill, **i32), torch.full((B_, cap), float(fill), dtype=torch.float64, device='cuda'), torch.full((B_,), fill, **i32),
           torch.full((B_, cap), fill, **i32), torch.full((B_, cap), fill, **i32), torch.full((B_,), fill, **i32))
    return scratch, out


def _device_rows(out):
    return [rows([t.cpu().numpy() for t in out], b) for b in range(out[0].shape[0])]


def test_orbvoc_device_form_into_search_by_bow(orb, orbvoc):
    """Frame::ComputeBoW by the device form for a keyframe and a frame, its FeatureVectors into SearchByBoW(KeyFrame*, Frame&), against
    the oracle's transform + SearchByBoW."""
    import torch
    voc, v = orbvoc
    (kk, dk), (kf, df) = S.extract(3), S.extract(4)
    cap = max(len(dk), len(df))
    desc, n = padded([dk, df], cap, seed=4)
    scratch, out = _device_buffers(torch, 2, cap)
    v.transform_device(torch.from_numpy(desc).cuda(), torch.from_numpy(n).cuda(), 4, scratch, out)
    torch.cuda.synchronize()
    got = _device_rows(out)
    refs = [O.bow_transform(voc, d, 4) for d in (dk, df)]
    for g, r in zip(got, refs):
        same(g, r, 'device form')
    kf_point = np.random.default_rng(3).choice([0, 1, 1, 1, 1, 2], len(kk)).astype(np.uint8)
    m = orb.ORBmatcher(0.7, True, max_batch=1, max_keypoints=2048, max_mappoints=2048)
    nm, match = m.SearchByBoW(kk, dk, kf_point, got[0][2:], kf, df, got[1][2:])
    on, om = O.search_by_bow(kk, dk, kf_point, refs[0][2:], kf, df, refs[1][2:], nnratio=0.7, check_ori=True)
    assert nm == on and np.array_equal(match, om) and nm > 20, (nm, on)


def test_device_form_on_a_side_stream(orb):
    """The device form enqueued on a side stream gives the host form's bytes (within nWords / nEntries) and the oracle's result."""
    import torch
    voc = B.vocabulary('k64_L3')
    v = handle(orb, voc)
    frames = [_features(voc, n, seed=40 + i) for i, n in enumerate((700, 0, 1, 513, 699))]
    cap = 700
    desc, n = padded(frames, cap, seed=41)
    host = run_padded(orb, v, frames, cap, 1, seed=41)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        d_desc, d_n = torch.from_numpy(desc).cuda(non_blocking=True), torch.from_numpy(n).cuda(non_blocking=True)
        scratch, out = _device_buffers(torch, len(frames), cap)
    v.transform_device(d_desc, d_n, 1, scratch, out, stream=side.cuda_stream)
    side.synchronize()
    got = _device_rows(out)
    for b, (g, h) in enumerate(zip(got, host)):
        assert all(x.tobytes() == y.tobytes() for x, y in zip(g, h)), b
    check_frames(got, voc, frames, 1)


def test_device_form_small_call_after_large_on_the_same_buffers(orb):
    """A call with large n, then one with small n on the same scratch and output tensors: the second gives its own oracle result."""
    import torch
    voc = B.vocabulary('k33_L3')
    v = handle(orb, voc)
    cap = 1024
    scratch, out = _device_buffers(torch, 3, cap)
    for ns, seed in (((1024, 1024, 1000), 50), ((3, 0, 17), 51)):
        frames = [_features(voc, k, seed=seed + i) for i, k in enumerate(ns)]
        desc, n = padded(frames, cap, seed=seed)
        v.transform_device(torch.from_numpy(desc).cuda(), torch.from_numpy(n).cuda(), 2, scratch, out)
        torch.cuda.synchronize()
        check_frames(_device_rows(out), voc, frames, 2)


# ---- refusals ----
def test_refuses_cap_above_16384(orb):
    import torch
    voc = B.vocabulary('k10_L5')
    v = handle(orb, voc)
    rc, _ = host_call(orb, v, *padded([_features(voc, 5, seed=1)], 16385, seed=1), 16385, 2)
    assert rc == orb.ORB_ERR_ARG
    scratch, out = _device_buffers(torch, 1, 16385)
    with pytest.raises(orb.OrbError):
        v.transform_device(torch.zeros((1, 16385, 32), dtype=torch.uint8, device='cuda'), torch.full((1,), 5, dtype=torch.int32, device='cuda'), 2,
                           scratch, out)


def test_refuses_negative_levelsup(orb):
    import torch
    voc = B.vocabulary('k10_L5')
    v = handle(orb, voc)
    with pytest.raises(orb.OrbError):
        v.transform([_features(voc, 5, seed=1)], -1)
    scratch, out = _device_buffers(torch, 1, 8)
    with pytest.raises(orb.OrbError):
        v.transform_device(torch.zeros((1, 8, 32), dtype=torch.uint8, device='cuda'), torch.full((1,), 5, dtype=torch.int32, device='cuda'), -1,
                           scratch, out)


def test_refuses_unknown_weighting_and_norm(orb):
    voc = B.vocabulary('k10_L5')
    for w, n in ((4, 1), (0, 3), (-1, 0), (0, -1)):
        with pytest.raises(orb.OrbError):
            handle(orb, voc, w, n)


@pytest.mark.parametrize('bad', (-1, 9))
def test_refuses_counts_outside_0_cap_before_staging(orb, bad):
    """n[f] < 0 or n[f] > cap in the host form: ORB_ERR_ARG and not one output element written."""
    voc = B.vocabulary('k10_L5')
    v = handle(orb, voc)
    frames = [_features(voc, k, seed=k) for k in (8, 3, 8)]
    desc, n = padded(frames, 8, seed=2)
    n[1] = bad
    rc, outs = host_call(orb, v, desc, n, 8, 2)
    assert rc == orb.ORB_ERR_ARG
    assert all((o == -7).all() for o in outs)


def _small_tree():
    """synthetic_vocabulary(3, 4): root 0; nodes 1-3 at depth 1, 4-12 at depth 2, 13-39 at depth 3, 40-120 leaves at depth 4."""
    voc = O.synthetic_vocabulary(3, 4, seed=1)
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in voc.items()}


def _self_loop(voc):
    x = 5                                                  # an inner node at depth 2
    voc['children'][voc['child_start'][x]] = x


def _grandparent_cycle(voc):
    x = 20                                                 # depth 3; its grandparent is at depth 1
    g = voc['parent'][voc['parent'][x]]
    assert g > 0
    voc['children'][voc['child_start'][x]] = g


def _listed_twice(voc):
    voc['children'][voc['child_start'][7]] = voc['children'][voc['child_start'][6]]


def _negative_word(voc):
    leaf = 60
    voc['word_id'][leaf], voc['weight'][leaf] = -1, 1.5


def _not_monotone(voc):
    voc['child_start'][5], voc['child_start'][6] = voc['child_start'][6], voc['child_start'][5]


def _root_without_children(voc):
    voc['child_start'][1] = 0


def _too_many_children(voc):
    """A root with 2^20 + 1 leaf children: more list positions than the descent's 20-bit rank holds."""
    n = (1 << 20) + 2
    voc.update(child_start=np.concatenate([[0], np.full(n, n - 1)]).astype(np.int32), children=np.arange(1, n, dtype=np.int32),
               desc=np.zeros((n, 32), np.uint8), weight=np.concatenate([[0.0], np.ones(n - 1)]),
               word_id=np.concatenate([[-1], np.arange(n - 1)]).astype(np.int32))


@pytest.mark.parametrize('defect', (_not_monotone, _root_without_children, _listed_twice, _self_loop, _grandparent_cycle, _negative_word,
                                    _too_many_children), ids=lambda f: f.__name__.strip('_'))
def test_refuses_malformed_vocabulary(orb, defect):
    """orbv_create refuses the table; none of these is ever transformed (a cycle would never reach a leaf)."""
    voc = _small_tree()
    handle(orb, voc)                                       # the intact tree is accepted
    defect(voc)
    with pytest.raises(orb.OrbError):
        handle(orb, voc)
