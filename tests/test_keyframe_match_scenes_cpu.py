"""The cases of tests/keyframe_match_scenes.py reach the shapes they are built for, shown from the oracle's outputs and the cases' own data,
and the SearchByBoW oracle (both overloads, rotation filter included) equals a set-based numpy restatement on every BoW case.  The
restatement is integer work plus the float32 rotation bin with round half away from zero, so these cases do not rest on
test_ref_pins_oracle_cpu.py alone (which needs the reference checkout).  The GPU side is tests/test_keyframe_match_paths_gpu.py."""
import numpy as np
import pytest

import keyframe_match_scenes as S
import new_points_lib as NP
import oracle_lib as O

BOW, TRI, FUSE = S.bow_cases(), S.tri_cases(), S.fuse_cases()
BY = {c['name']: c for c in BOW + FUSE}
BYT = {c['name']: c for c in TRI}
POP = np.array([bin(i).count('1') for i in range(256)], np.int32)
f32 = np.float32


def dist_matrix(a, b):
    return POP[np.bitwise_xor(a[:, None, :], b[None, :, :])].sum(-1)


def bow_restatement(c, kf_kf, ori):
    """SearchByBoW from sets: the nodes both vectors hold, in id order; in each node the keyframe features in list order take the closest
    frame feature not yet taken (first list position on equal distance), subject to TH_LOW (strict for KeyFrame-KeyFrame) and the ratio test
    in float32; then the rotation filter.  Returns (n, out) as the oracle does: match [nF] (KeyFrame-Frame) or match12 [nKF]."""
    (nk, fk), (nf, ff) = c['fvk'], c['fvf']
    taken = np.zeros(len(c['kf']), bool)
    usable = (c['fp'] == 1) if kf_kf else np.ones(len(c['kf']), bool)
    pairs = []
    for node in np.intersect1d(nk, nf):
        ks, fs = fk[nk == node], ff[nf == node]
        D = dist_matrix(c['dk'][ks], c['df'][fs])
        for r, i in enumerate(ks):
            if c['kp'][i] != 1:
                continue
            d = np.where(taken[fs] | ~usable[fs], 256, D[r])
            p = int(np.argmin(d))
            d1 = int(d[p])
            d2 = int(np.min(np.delete(d, p))) if len(d) > 1 else 256
            if d1 == 256:
                continue
            if (d1 < S.TH_LOW if kf_kf else d1 <= S.TH_LOW) and f32(d1) < f32(c['nnratio']) * f32(d2):
                pairs.append((int(i), int(fs[p])))
                taken[fs[p]] = True
    if ori:
        bins = [S.rot_bin(c['kk']['angle'][i], c['kf']['angle'][j]) for i, j in pairs]
        keep = S.three_maxima(np.bincount(bins, minlength=13)) if bins else ()
        pairs = [p for p, b in zip(pairs, bins) if b in keep]
    out = np.full(len(c['kk']) if kf_kf else len(c['kf']), -1, np.int32)
    for i, j in pairs:
        out[i if kf_kf else j] = j if kf_kf else i
    return len(pairs), out


def bow_oracle(c, kf_kf, ori):
    if kf_kf:
        return O.search_by_bow_kf(c['kk'], c['dk'], c['kp'], c['fvk'], c['kf'], c['df'], c['fp'], c['fvf'], nnratio=c['nnratio'], check_ori=ori)
    return O.search_by_bow(c['kk'], c['dk'], c['kp'], c['fvk'], c['kf'], c['df'], c['fvf'], nnratio=c['nnratio'], check_ori=ori)


@pytest.mark.parametrize('ori', (False, True))
@pytest.mark.parametrize('kf_kf', (False, True))
@pytest.mark.parametrize('c', BOW, ids=[c['name'] for c in BOW])
def test_bow_oracle_equals_restatement(c, kf_kf, ori):
    n, out = bow_oracle(c, kf_kf, ori)
    rn, rout = bow_restatement(c, kf_kf, ori)
    assert n == rn and np.array_equal(out, rout), (c['name'], n, rn)
    if not ori:
        assert n >= c['min_matches'], (c['name'], n)          # the byte compare cannot pass on empty outputs


def _kf_matches(c, ori=False):
    """The KeyFrame-Frame oracle's matches as (keyframe feature, frame feature)."""
    _, m = bow_oracle(c, False, ori)
    return {(int(m[j]), j) for j in np.flatnonzero(m >= 0)}


def test_bow_shapes():
    fv_nodes = lambda fv: np.unique(fv[0])
    assert len(BY['eKF_0']['fvk'][0]) == 0 and len(BY['eKF_0']['fvf'][0]) > 0
    c = BY['one_node_2048']
    assert len(fv_nodes(c['fvk'])) == len(fv_nodes(c['fvf'])) == 1 and len(c['fvk'][0]) == len(c['fvf'][0]) == S.N == len(c['kk']) == len(c['kf'])
    for g in (1, 7, 8, 9, 300):
        c = BY['groups_%d' % g]
        assert len(np.intersect1d(fv_nodes(c['fvk']), fv_nodes(c['fvf']))) == g      # node groups: 300 > 8 warps
    for s in (1, 31, 32, 33, 64, 65, 1000):
        _, counts = np.unique(BY['fnode_%d' % s]['fvf'][0], return_counts=True)
        assert (counts == s).all()
    c = BY['one_sided_nodes']
    k, f = set(fv_nodes(c['fvk'])), set(fv_nodes(c['fvf']))
    assert k - f and f - k and k & f
    c = BY['node_ids_ends']
    for fv in (c['fvk'], c['fvf']):
        assert fv[0][0] == 0 and fv[0][-1] == S.NODE_MAX
    c = BY['node_ids_ends_one_sided']
    assert c['fvk'][0][-1] == S.NODE_MAX and S.NODE_MAX not in c['fvf'][0] and 0 in c['fvk'][0] and 0 not in c['fvf'][0]
    c = BY['entries_lt_N']
    assert len(c['fvk'][0]) < S.N and len(c['fvf'][0]) < S.N
    c = BY['unsorted_node_lists']
    (nk, fk) = c['fvk']
    assert any((np.diff(fk[nk == n]) < 0).any() for n in np.unique(nk))
    c = BY['points_012']
    assert set(np.unique(c['kp'])) == set(np.unique(c['fp'])) == {0, 1, 2}


def test_bow_boundaries_decided_by_the_oracle():
    # 49 / 50 / 51: <= TH_LOW for KeyFrame-Frame, < TH_LOW for KeyFrame-KeyFrame
    c = BY['th_low_50_51']
    kf_frame = _kf_matches(c)
    _, m12 = bow_oracle(c, True, False)
    for i, j, d in c['plants']:
        assert S.hamming(c['dk'][i], c['df'][j]) == d
        assert ((i, j) in kf_frame) == (d <= 50) and (m12[i] == j) == (d < 50), (i, j, d)
    # the ratio test at equality: 30 vs 0.75 * 40 = 30 exactly in float32
    assert f32(0.75) * f32(40) == f32(30)
    c = BY['ratio_edge']
    got = _kf_matches(c)
    firsts = {}
    for i, j, d in c['plants']:
        firsts.setdefault(i, []).append((j, d))
    for i, pl in firsts.items():
        want = len(pl) == 1 or f32(pl[0][1]) < f32(0.75) * f32(pl[1][1])
        assert ((i, pl[0][0]) in got) == want, (i, pl)
    # equal best distances: the first list position wins
    c = BY['lane_ties']
    got = _kf_matches(c)
    (nf, ff) = c['fvf']
    for i, j, _ in c['plants'][::2]:
        node = c['fvk'][0][list(c['fvk'][1]).index(i)]
        fs = list(ff[nf == node])
        j2 = next(jj for ii, jj, _ in c['plants'] if ii == i and jj != j)
        assert (i, min(j, j2, key=fs.index)) in got
    # claims: some keyframe features end on their second choice, some fail the ratio test once the first choice is gone
    c = BY['claims']
    got = _kf_matches(c)
    plants = {}
    for i, j, d in c['plants']:
        plants.setdefault(i, []).append(j)
    second = sum((i, p[1]) in got for i, p in plants.items() if len(p) > 1)
    assert second >= 10 and sum(1 for i in plants if not any(k == i for k, _ in got)) >= 10


@pytest.mark.parametrize('kind', ('bow', 'tri'))
def test_rotation_plans(kind):
    """Each planted histogram has the bins, ties and bars of its plan; the k + 0.5 products are exact in float32 and decide the kept bins
    differently under round half to even."""
    for pname, plan in S.ROT_PLANS.items():
        c = (BY if kind == 'bow' else BYT)['rot_' + pname]
        if kind == 'bow':
            pairs = sorted(_kf_matches(c))
            ang = [(c['kk']['angle'][i], c['kf']['angle'][j]) for i, j in pairs]
        else:
            on, om = _tri(c, 0, False)
            ang = [(c['kf1']['kps']['angle'][i], c['kf2'][0]['kps']['angle'][om[i]]) for i in np.flatnonzero(om >= 0)]
        hist = list(np.bincount([S.rot_bin(a, b) for a, b in ang], minlength=13))
        assert hist == S.plan_hist(plan), (kind, pname, hist)
        keep = S.three_maxima(hist)
        if 'half' in plan:
            k = plan['half'][0]
            halves = [(a, b) for a, b in ang if S.rot_product(a, b) == f32(k + 0.5)]
            assert len(halves) == plan['half'][1] and all(S.rot_bin(a, b) == k + 1 and S.rot_bin(a, b, True) == k for a, b in halves)
            assert all((f32(a - b) < 0) == plan['half'][2] for a, b in halves)
            even = list(np.bincount([S.rot_bin(a, b, True) for a, b in ang], minlength=13))
            assert set(S.three_maxima(even)) != set(keep)
        if pname == 'wrap_0_12':
            assert all(f32(a - b) < 0 for a, b in ang if S.rot_bin(a, b) in (0, 12))
        n_ori = _tri(c, 0, True)[0] if kind == 'tri' else bow_oracle(c, False, True)[0]
        assert n_ori == sum(hist[b] for b in keep if b >= 0)
    assert S.three_maxima(S.plan_hist(S.ROT_PLANS['max2_10v1']))[1] == 6 and S.three_maxima(S.plan_hist(S.ROT_PLANS['max2_11v1']))[1] == -1
    assert S.three_maxima(S.plan_hist(S.ROT_PLANS['max3_10v1']))[2] == 9 and S.three_maxima(S.plan_hist(S.ROT_PLANS['max3_11v1']))[2] == -1
    assert S.three_maxima(S.plan_hist(S.ROT_PLANS['four_tied'])) == (1, 4, 7)
    assert S.three_maxima(S.plan_hist(S.ROT_PLANS['tie_max'])) == (3, 8, 1)


def _tri(c, k, ori):
    kf2 = c['kf2'][k]
    sc = dict(k1=c['kf1']['kps'], d1=c['kf1']['desc'], mp1=c['kf1']['has_mp'], fv1=c['kf1']['fv'], k2=kf2['kps'], d2=kf2['desc'], mp2=kf2['has_mp'],
              fv2=kf2['fv'], sf=c['sf'], sigma2=c['sigma2'])
    return O.search_for_triangulation(sc, c['ep'][k], c['F12'][k], c['coarse'], ori)


def test_tri_shapes_and_boundaries():
    for c in TRI:
        n = sum(_tri(c, k, False)[0] for k in range(len(c['kf2'])))
        assert n >= c['min_matches'], (c['name'], n)
        for e in ('E1', 'N1'):
            if e in c['shape']:
                assert (len(c['kf1']['fv'][0]) if e == 'E1' else len(c['kf1']['kps'])) == c['shape'][e]
    for s in (31, 32, 33, 500):
        for kf2 in BYT['kf2_node_%d' % s]['kf2']:
            assert (np.unique(kf2['fv'][0], return_counts=True)[1] == s).all()
    # equal minimal distances: the last position of the node wins
    c = BYT['lane_ties']
    _, m12 = _tri(c, 0, False)
    (n2, f2) = c['kf2'][0]['fv']
    for g in range(0, len(c['kf1']['fv'][0])):
        i = int(c['kf1']['fv'][1][g])
        fs = list(f2[n2 == c['kf1']['fv'][0][g]])
        cands = [j for j in fs if S.hamming(c['kf1']['desc'][i], c['kf2'][0]['desc'][j]) <= 50]
        assert len(cands) == 2 and m12[i] == max(cands, key=fs.index)
    # 49 / 50 / 51
    c = BYT['th_low_50_51']
    _, m12 = _tri(c, 0, False)
    for i in range(90):
        assert (m12[i] >= 0) == ((49, 50, 51)[i % 3] <= 50)
    # the epipole-distance bar: at the bar kept, one float step inside rejected, for octaves 0 and 3, in both modes
    for name in ('epipole_bar', 'epipole_bar_coarse'):
        c = BYT[name]
        _, m12 = _tri(c, 0, False)
        for e in c['shape']['epipole']:
            kp2 = c['kf2'][0]['kps'][e['j']]
            dx, dy = f32(c['ep'][0][0] - kp2['x']), f32(c['ep'][0][1] - kp2['y'])
            v, bar = f32(np.float64(dx) * dx + np.float64(f32(dy * dy))), f32(f32(100) * f32(c['sf'][e['octave']]))
            assert (v < bar) == e['inside'] and (v == bar or e['inside'] or v > bar)
            assert (m12[e['i']] == e['j']) == (not e['inside'])
        assert {e['octave'] for e in c['shape']['epipole']} == {0, 3}
    bar_hits = sum(1 for e in BYT['epipole_bar']['shape']['epipole'] if not e['inside'] and
                   f32(np.float64(f32(BYT['epipole_bar']['ep'][0][0] - BYT['epipole_bar']['kf2'][0]['kps'][e['j']]['x'])) ** 2) == f32(f32(100) * f32(BYT['epipole_bar']['sf'][e['octave']])))
    assert bar_hits >= 4                                                   # exactly at the bar, not just above it
    # den == 0: nothing in fine mode, matches in coarse mode
    assert sum(_tri(BYT['den0'], k, False)[0] for k in range(2)) == 0 and sum(_tri(BYT['den0_coarse'], k, False)[0] for k in range(2)) > 0
    c = BYT['has_mp_and_empty']
    assert len(c['kf2'][1]['kps']) == 0 and len(c['kf2'][3]['fv'][0]) == 0 < len(c['kf2'][3]['kps'])
    assert c['kf1']['has_mp'].any() and all(k['has_mp'].any() for k in c['kf2'] if len(k['kps']))


def test_fuse_layouts():
    """The Python mirror of frame_smem_bytes / frame_layout puts each keyframe where its case says: 4,496 keypoints is the largest keyframe with
    its descriptors in shared memory, 4,497 the smallest in global memory, 14,008 the largest accepted, 14,009 refused."""
    assert (S.K_SMEM_MAX, S.K_MAX) == (4496, 14008)
    assert [S.fuse_layout(k) for k in (4496, 4497, 14008, 14009)] == ['smem', 'global', 'global', 'refused']
    for c in FUSE + S.sim3_cases():
        if 'layout' in c['shape']:
            K = len(c['kps']) if 'kps' in c else len(c['kf1']['kps'])
            assert K == c['shape']['K'] and S.fuse_layout(K) == c['shape']['layout']
    r = S.refused_keyframe()
    assert len(r['kps']) == 14009 and S.fuse_layout(14009) == 'refused'
    for c in FUSE:
        bi, bd = O.fuse_search(c, c['th'])
        assert (bd <= 50).sum() >= c['min_matches'], c['name']
        if 'M' in c['shape']:
            assert len(c['state']) == c['shape']['M']
    assert sorted({min(16, (M + 127) // 128) for M in (1, 127, 128, 129, 1920, 1921, 2048, 2049, 20000)}) == [1, 2, 15, 16]


def test_fuse_edges_decided_by_the_oracle():
    c = BY['edges']
    mk = c['marks']
    bi, bd = O.fuse_search(c, c['th'])
    si, sd = O.fuse_search_sim3(c, c['Tcw'], c['Ow'], c['th'])
    u = lambda p: S.project(c['cam'], c['xyz'][p])[0]
    assert u(mk['u_min'][0]) == f32(0) and bi[mk['u_min'][0]] == mk['u_min'][1]
    assert u(mk['u_max'][0]) == f32(640) and bi[mk['u_max'][0]] == -1
    for name in ('min_d', 'max_d', 'view', 'zc_neg'):
        a, b, j = mk[name]
        assert bi[a] == j and bi[b] == -1, name
    a, b, j = mk['view']
    d = S.dist3(c['xyz'][a])
    dot = lambda p: f32(f32(f32(c['xyz'][p][0] * c['normal'][p][0]) + f32(c['xyz'][p][1] * c['normal'][p][1])) + f32(c['xyz'][p][2] * c['normal'][p][2]))
    assert np.float64(dot(a)) >= 0.5 * np.float64(d) > np.float64(dot(b)) and np.nextafter(c['normal'][b][2], f32(1)) == c['normal'][a][2]
    for o in (0, 2):
        a, b, ja, jb = mk['chi2_oct%d' % o]
        assert bi[a] == ja and bi[b] == -1 and si[b] == jb             # the gate alone rejects b: Fuse(Scw) has no gate
    s1, s0, s2, s3, j = mk['states']
    assert bi[s1] == j and bi[s0] == bi[s2] == bi[s3] == -1
    for lvl in (0, 7):
        p, j = mk['level_%d' % lvl]
        r = np.log(np.float64(c['max_d'][p]) / np.float64(S.dist3(c['xyz'][p]))) / np.log(1.2)
        assert (r <= 0) if lvl == 0 else (r > 7)
        assert bi[p] == j
    for name in ('tie_rows', 'tie_cols'):
        p, ja, jb = mk[name]
        assert bd[p] == S.hamming(c['mp_desc'][p], c['desc'][ja]) == S.hamming(c['mp_desc'][p], c['desc'][jb]) and ja < jb and bi[p] == jb, name
    p, ja, jb = mk['tie_cell']
    assert S.hamming(c['mp_desc'][p], c['desc'][ja]) == S.hamming(c['mp_desc'][p], c['desc'][jb]) and bi[p] == ja
    inv = f32(64) / f32(640)
    on_border = [j for j in mk['border'] if f32(f32(c['kps'][j]['x']) * inv) % 1 == 0.5]
    assert len(on_border) == len(mk['border'])
    crowd = mk['crowd']
    cells = {(int(np.floor(f32(c['kps'][j]['x'] * inv) + 0.5)), int(np.floor(f32(c['kps'][j]['y'] * f32(48) / f32(480)) + 0.5))) for j in crowd}
    assert len(crowd) > 1000 and len(cells) == 1 and np.isin(bi, crowd).sum() >= 100


def test_new_points_at_the_pair_limit():
    """Exactly 65,535 pairs; the item with the largest KF1 (maxN1) is not the one with the most pairs; every item matches and creates points."""
    items = S.wide_new_points()
    assert sum(len(sc['kf2']) for sc in items) == S.MAX_PAIRS == 65535
    n1 = [len(sc['kf1']['kps']) for sc in items]
    pairs = [len(sc['kf2']) for sc in items]
    assert int(np.argmax(n1)) != int(np.argmax(pairs))
    for sc in items:
        rec, nm, nc, _ = NP.create(sc)
        assert nm.sum() > 0 and nc.sum() > 0 and len(rec) == nc.sum()
