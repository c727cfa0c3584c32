"""Seeded cases for the keyframe matchers: SearchByBoW (both overloads, bow_match_kernel), SearchForTriangulation (tri_match_kernel),
the Fuse searches and SearchBySim3 (fuse_search_kernel) and the batched CreateNewMapPoints, each built for one shape the kernels branch
on.  Every case records that shape in case['shape']; tests/test_keyframe_match_scenes_cpu.py shows from the oracle and the case's own data
that the case reaches it, tests/test_keyframe_match_paths_gpu.py compares the GPU with the oracle on it byte for byte.

Descriptors are random unless planted: a planted descriptor is a copy of another with exactly `d` bits flipped, so its Hamming distance is
d.  Two random descriptors are ~Binomial(256, 1/2) apart (never below ~85 among a few million pairs), far from TH_LOW = 50 and from every
planted distance, so the planted distances alone decide the matches.  FeatureVectors are hand-made (node id, feature index) lists next to
ones the DBoW2 transform makes of real ORB features (tests/new_points_lib.py, oracle_lib.fuse_scene / sim3_scene)."""
import numpy as np

import matcher_scenes as MS
import new_points_lib as NP
import oracle_lib as O
from orb_slam3_modified_b200 import KP_DTYPE

TH_LOW = 50
HISTO_LENGTH = 30
FACTOR = np.float32(1.0) / np.float32(HISTO_LENGTH)
N = 2048                                   # the BoW cases' handle caps (max_keypoints = max_mappoints)
NODE_MAX = 2 ** 31 - 1
BOUNDS = (0.0, 0.0, 640.0, 480.0)
SMEM_LIMIT = 227 * 1024 - 2048             # matcher.cu FRAME_SMEM_LIMIT
_TAB = None


def tables():
    global _TAB
    if _TAB is None:
        _TAB = O.OracleExtractor().tables()
    return _TAB


# ---------------------------------------------------------------------------------------------
# float32 helpers: the kernels' and the oracle's arithmetic, one rounding per operation
# ---------------------------------------------------------------------------------------------
f32 = np.float32


def rot_bin(a1, a2, half_even=False):
    """The rotation-histogram bin of SearchByBoW / SearchForTriangulation: rot = a1 - a2 (+ 360 when negative), round(rot * (1.0f / 30)) with
    round half away from zero (std::round on a float); half_even=True gives rintf's answer instead."""
    rot = f32(f32(a1) - f32(a2))
    if rot < 0:
        rot = f32(rot + f32(360.0))
    x = f32(rot * FACTOR)
    b = int(np.rint(x)) if half_even else int(np.floor(np.float64(x) + 0.5))
    return 0 if b == HISTO_LENGTH else b


def rot_product(a1, a2):
    rot = f32(f32(a1) - f32(a2))
    return f32((f32(rot + f32(360.0)) if rot < 0 else rot) * FACTOR)


def three_maxima(hist):
    """ORBmatcher::ComputeThreeMaxima: the kept bins (ind1, ind2, ind3), -1 where dropped."""
    ind, mx = [-1, -1, -1], [0, 0, 0]
    for b, s in enumerate(hist):
        if s > mx[0]:
            mx = [s, mx[0], mx[1]]; ind = [b, ind[0], ind[1]]
        elif s > mx[1]:
            mx = [mx[0], s, mx[1]]; ind = [ind[0], b, ind[1]]
        elif s > mx[2]:
            mx[2] = s; ind[2] = b
    bar = f32(f32(0.1) * f32(mx[0]))
    if f32(mx[1]) < bar:
        ind[1] = ind[2] = -1
    elif f32(mx[2]) < bar:
        ind[2] = -1
    return tuple(ind)


def _ulps(x, n):
    """The float32 values x - n ulps .. x + n ulps, ascending."""
    out, lo, hi = [f32(x)], f32(x), f32(x)
    for _ in range(n):
        lo, hi = np.nextafter(lo, f32(-np.inf)), np.nextafter(hi, f32(np.inf))
        out = [lo] + out + [hi]
    return out


def straddle(pred, x0, n=4096):
    """Adjacent float32 values (a, b), a < b, near x0 with pred(a) != pred(b), pred monotone in x."""
    xs = _ulps(x0, n)
    vals = [bool(pred(x)) for x in xs]
    for i in range(len(xs) - 1):
        if vals[i] != vals[i + 1]:
            return xs[i], xs[i + 1]
    raise AssertionError('no change of the predicate within %d ulps of %r' % (n, x0))


def flip(d, rng, nbits):
    d = np.array(d, np.uint8, copy=True)
    for bit in rng.choice(256, nbits, replace=False):
        d[bit >> 3] ^= np.uint8(1 << (bit & 7))
    return d


def hamming(a, b):
    return np.unpackbits(np.bitwise_xor(np.asarray(a, np.uint8), np.asarray(b, np.uint8)), axis=-1).sum(-1)


def keypoints(n, rng, x=None, y=None, angle=None, octave=None):
    k = np.zeros(n, KP_DTYPE)
    k['x'] = rng.uniform(5, 635, n) if x is None else x
    k['y'] = rng.uniform(5, 475, n) if y is None else y
    k['size'] = 31.0
    k['angle'] = rng.uniform(0, 360, n).astype(np.float32) if angle is None else angle
    k['response'] = rng.uniform(1e-4, 1e-2, n)
    k['octave'] = 0 if octave is None else octave
    k['class_id'] = -1
    return k


def half_pairs(rng, k, n, wrap):
    """n angle pairs (a1, a2) whose float32 rot * (1.0f / 30) is exactly k + 0.5, found by search: the float32 rot values with that product,
    the differences a1 - a2 that give them, then a2 drawn at random until a1 = a2 + difference subtracts back exactly.  wrap: a1 - a2 is
    negative, so rot comes from the + 360 branch."""
    target = f32(k + 0.5)
    rots = [r for r in _ulps(f32((k + 0.5) * 30), 64) if f32(r * FACTOR) == target]          # rot values with the exact product
    diffs = [q for r in rots for q in _ulps(f32(r - 360), 64) if f32(q + f32(360)) == r] if wrap else rots   # a1 - a2 giving them
    out = []
    for _ in range(100000):
        q = diffs[int(rng.integers(len(diffs)))]
        a2 = f32(rng.uniform(0.5, 40) + (360 - 45 if wrap else 0))
        a1 = f32(q + a2)
        if f32(a1 - a2) == q and 0 <= a1 < 360 and rot_product(a1, a2) == target:
            out.append((a1, a2))
            if len(out) == n:
                return out
    raise AssertionError('no angle pair with rot * (1.0f / 30) == %g found' % target)


def _rot_pair(rng, b, wrap=None):
    """Angles (a1, a2) whose rotation falls in bin b, well inside it; wrap forces (True) or forbids (False) the negative branch."""
    lo, hi = max(30.0 * b - 9, 0.5), min(30.0 * b + 9, 359.0)
    rot = rng.uniform(lo, hi)
    if wrap is None:
        wrap = bool(rng.random() < 0.5)
    a1 = rng.uniform(0, rot) if wrap else rng.uniform(rot, 360)
    a2 = a1 - rot + (360.0 if wrap else 0.0)
    return f32(a1), f32(a2)


# rotation plans: {bin: count}; 'half' entries are (k, count, wrap) of exact k + 0.5 products
ROT_PLANS = {
    'single': {4: 20},
    'tie_max': {3: 12, 8: 12, 1: 3},
    'max2_10v1': {2: 10, 6: 1},
    'max2_11v1': {2: 11, 6: 1},
    'max3_10v1': {2: 10, 6: 5, 9: 1},
    'max3_11v1': {2: 11, 6: 5, 9: 1},
    'four_tied': {1: 10, 4: 10, 7: 10, 11: 10},
    'four_above': {1: 9, 4: 8, 7: 7, 11: 6},
    'wrap_0_12': {0: 8, 12: 8, 6: 3},
    'half_4_5': {5: 2, 4: 4, 7: 6, 9: 6, 'half': (4, 5, False)},        # k + 0.5 has no float32 rot for k = 2 and 9
    'half_0_5': {1: 3, 0: 3, 5: 5, 8: 4, 'half': (0, 4, True)},
}


def rot_angles(rng, plan):
    """The angle pairs of a rotation plan, shuffled: [(a1, a2)]."""
    pairs = []
    for b, c in plan.items():
        if b == 'half':
            pairs += half_pairs(rng, c[0], c[1], c[2])
        else:
            pairs += [_rot_pair(rng, b, True if b in (0, 12) else None) for _ in range(c)]      # bins 0 and 12 through the negative wrap
    return [pairs[i] for i in rng.permutation(len(pairs))]


def plan_hist(plan, half_even=False):
    h = [0] * 13
    for b, c in plan.items():
        if b == 'half':
            h[c[0] + (0 if half_even else 1)] += c[1]
        else:
            h[b] += c
    return h


# ---------------------------------------------------------------------------------------------
# SearchByBoW: one (keyframe, frame) pair, both overloads
# ---------------------------------------------------------------------------------------------
class _Bow:
    """Builder of one BoW case: n_kf / n_f features with random descriptors and angles; nodes, plants and point flags added by the case."""

    def __init__(self, rng, n_kf=N, n_f=N):
        self.rng = rng
        self.dk = rng.integers(0, 256, (n_kf, 32), dtype=np.uint8)
        self.df = rng.integers(0, 256, (n_f, 32), dtype=np.uint8)
        self.kk = keypoints(n_kf, rng)
        self.kf = keypoints(n_f, rng)
        self.kp = np.ones(n_kf, np.uint8)
        self.fp = np.ones(n_f, np.uint8)
        self.nodes_kf, self.nodes_f = [], []         # [(node id, [feature indices in list order])]
        self.plants = []

    def node(self, nid, kf_feats, f_feats):
        if len(kf_feats):
            self.nodes_kf.append((nid, list(kf_feats)))
        if len(f_feats):
            self.nodes_f.append((nid, list(f_feats)))

    def plant(self, i, j, d, angles=None):
        """Frame feature j = keyframe feature i with d bits flipped; angles (a_kf, a_f), default: rotation in bin 0 or 1 (most) or 5 / 9."""
        self.df[j] = flip(self.dk[i], self.rng, d)
        if angles is None:
            angles = _rot_pair(self.rng, int(self.rng.choice([0, 0, 0, 1, 1, 5, 9])), False)
        self.kk['angle'][i], self.kf['angle'][j] = angles
        self.plants.append((i, j, d))

    def case(self, name, shape, nnratio=0.7, min_matches=8):
        def fv(nodes):
            nodes = sorted(nodes, key=lambda t: t[0])
            n = np.array([nid for nid, fs in nodes for _ in fs], np.int32)
            f = np.array([x for _, fs in nodes for x in fs], np.int32)
            return n, f
        return dict(kind='bow', name=name, shape=shape, kk=self.kk, dk=self.dk, kp=self.kp, fvk=fv(self.nodes_kf), kf=self.kf, df=self.df,
                    fp=self.fp, fvf=fv(self.nodes_f), nnratio=f32(nnratio), plants=list(self.plants), min_matches=min_matches)


def _split(rng, idx, g):
    """idx split into g non-empty consecutive runs of random lengths."""
    cuts = np.sort(rng.choice(np.arange(1, len(idx)), g - 1, replace=False)) if g > 1 else []
    return np.split(np.asarray(idx), cuts)


def _groups(g, seed):
    rng = np.random.default_rng(seed)
    B = _Bow(rng)
    ids = np.sort(rng.choice(10 ** 6, g, replace=False)).astype(np.int64) + 1
    ks, fs = _split(rng, rng.permutation(N), g), _split(rng, rng.permutation(N), g)
    for nid, a, b in zip(ids, ks, fs):
        B.node(int(nid), a, b)
        for i in a:
            if rng.random() < 0.7:
                B.plant(int(i), int(rng.choice(b)), int(rng.integers(0, 48)))
    return B.case('groups_%d' % g, dict(groups=g))


def _fnode(s, seed):
    rng = np.random.default_rng(seed)
    B = _Bow(rng)
    G = min(40, N // s)
    kperm, fperm = rng.permutation(N), rng.permutation(N)
    for g in range(G):
        a, b = kperm[6 * g:6 * g + 6], fperm[s * g:s * g + s]
        B.node(100 + 3 * g, a, b)
        for i in a:
            if rng.random() < 0.8:
                B.plant(int(i), int(rng.choice(b)), int(rng.integers(0, 48)))
    return B.case('fnode_%d' % s, dict(f_node_size=s, groups=G))


def bow_cases():
    cs = []
    # eKF = 0
    rng = np.random.default_rng(1)
    B = _Bow(rng)
    for g in range(10):
        B.node(g, [], range(30 * g, 30 * g + 30))
    cs.append(B.case('eKF_0', dict(eKF=0), min_matches=0))
    # one node holds every feature on both sides, N = the handle caps
    rng = np.random.default_rng(2)
    B = _Bow(rng)
    pk, pf = rng.permutation(N), rng.permutation(N)
    B.node(7, range(N), range(N))
    for i in range(1500):
        B.plant(int(pk[i]), int(pf[i]), int(rng.integers(0, 48)))
    cs.append(B.case('one_node_2048', dict(groups=1, node_size=N)))
    cs += [_groups(g, 10 + g) for g in (1, 7, 8, 9, 300)]
    cs += [_fnode(s, 20 + s) for s in (1, 31, 32, 33, 64, 65, 1000)]
    # nodes on one side only, interleaved with shared ones
    rng = np.random.default_rng(3)
    B = _Bow(rng)
    kperm, fperm = rng.permutation(N), rng.permutation(N)
    for g in range(60):
        a, b = kperm[20 * g:20 * g + 20], fperm[20 * g:20 * g + 20]
        side = g % 3                      # 0: both, 1: keyframe only, 2: frame only
        B.node(5 * g + side, a if side != 2 else [], b if side != 1 else [])
        for i in a[:12]:
            B.plant(int(i), int(rng.choice(b)), int(rng.integers(0, 48)))
    cs.append(B.case('one_sided_nodes', dict(one_sided=True)))
    # node ids 0 and 2^31 - 1 at the ends of both vectors, and at the end of one only
    for name, kids, fids in (('node_ids_ends', (0, 9, NODE_MAX), (0, 4, NODE_MAX)), ('node_ids_ends_one_sided', (0, NODE_MAX - 1, NODE_MAX), (1, NODE_MAX - 1))):
        rng = np.random.default_rng(4 + len(name))
        B = _Bow(rng)
        kperm, fperm = rng.permutation(N), rng.permutation(N)
        shared = set(kids) & set(fids)
        for g, nid in enumerate(sorted(set(kids) | set(fids))):
            a, b = kperm[50 * g:50 * g + 50], fperm[50 * g:50 * g + 50]
            B.node(nid, a if nid in kids else [], b if nid in fids else [])
            if nid in shared:
                for i in a[:30]:
                    B.plant(int(i), int(rng.choice(b)), int(rng.integers(0, 48)))
        cs.append(B.case(name, dict(node_ids=sorted(set(kids) | set(fids)))))
    # nEntries < N, and feature lists not in ascending feature order
    for name, order in (('entries_lt_N', 'asc'), ('unsorted_node_lists', 'shuffled')):
        rng = np.random.default_rng(6 + len(name))
        B = _Bow(rng)
        ks = rng.permutation(N)[:1500] if order == 'asc' else rng.permutation(N)
        fs = rng.permutation(N)[:1200] if order == 'asc' else rng.permutation(N)
        for g, (a, b) in enumerate(zip(_split(rng, ks, 40), _split(rng, fs, 40))):
            a, b = (np.sort(a), np.sort(b)) if order == 'asc' else (a[::-1] if g % 2 else a, b)
            B.node(11 * g, a, b)
            for i in a:
                if rng.random() < 0.7:
                    B.plant(int(i), int(rng.choice(b)), int(rng.integers(0, 48)))
        cs.append(B.case(name, dict(eKF=len(ks), eF=len(fs), order=order)))
    # several keyframe features want the same frame feature: later ones take their second choice or fail the ratio test
    rng = np.random.default_rng(7)
    B = _Bow(rng)
    kperm, fperm = rng.permutation(N), rng.permutation(N)
    for g in range(30):
        a, b = kperm[6 * g:6 * g + 6], fperm[40 * g:40 * g + 40]
        B.node(2 * g + 1, a, b)
        for r, i in enumerate(a):
            B.plant(int(i), int(b[0]), 8 + 2 * r)                       # everybody's first choice
            if r % 3 != 2:
                B.plant(int(i), int(b[1 + r]), 16 + 2 * r)              # a second choice clear of the ratio test ...
            if r % 3 == 1:
                B.plant(int(i), int(b[7 + r]), 18 + 2 * r)              # ... or not, once the first choice is gone
    cs.append(B.case('claims', dict(claims=True)))
    # best distances 49 / 50 / 51 (TH_LOW: <= for KeyFrame-Frame, < for KeyFrame-KeyFrame)
    rng = np.random.default_rng(8)
    B = _Bow(rng, 600, 600)
    for g in range(60):
        i, j = 10 * g, 10 * g + 1
        B.node(g, [i], range(10 * g, 10 * g + 10))
        B.plant(i, j, (49, 50, 51)[g % 3])
    cs.append(B.case('th_low_50_51', dict(best=(49, 50, 51))))
    # the ratio test at equality in float32: 30 < 0.75 * 40 is false, 29 < 30 and 30 < 0.75 * 41 are true; no second candidate (256)
    rng = np.random.default_rng(9)
    B = _Bow(rng, 600, 600)
    for g in range(60):
        i = 10 * g
        kind = g % 4
        if kind == 3:
            B.node(g, [i], [10 * g])
            B.plant(i, 10 * g, 20 + g % 7)
            continue
        B.node(g, [i], range(10 * g, 10 * g + 10))
        d1, d2 = ((30, 40), (29, 40), (30, 41))[kind]
        B.plant(i, 10 * g + 3, d1)
        B.plant(i, 10 * g + 7, d2)
    cs.append(B.case('ratio_edge', dict(pairs=((30, 40), (29, 40), (30, 41), 'single')), nnratio=0.75))
    # equal best distances in different lanes and in the same lane: the first position wins (visible only with nnratio > 1)
    rng = np.random.default_rng(10)
    B = _Bow(rng, 1700, 1700)
    for g, (p, q) in enumerate([(0, 1), (0, 32), (3, 35), (5, 40), (31, 32), (1, 69), (40, 5), (64, 2)] * 3):
        i, base = 20 * g, 70 * g
        feats = list(range(base, base + 70))
        B.node(g, [i], feats)
        d = 10 + g % 20
        B.plant(i, feats[p], d)
        B.plant(i, feats[q], d)
    cs.append(B.case('lane_ties', dict(tie_positions=True), nnratio=1.25))
    # kfPoint / fPoint 0, 1, 2
    c = _groups(9, 11)
    rng = np.random.default_rng(12)
    c = dict(c, name='points_012', shape=dict(points=(0, 1, 2)), kp=rng.choice([0, 1, 1, 2], N).astype(np.uint8),
             fp=rng.choice([0, 1, 1, 2], N).astype(np.uint8))
    cs.append(c)
    # rotation histograms
    for pname, plan in ROT_PLANS.items():
        rng = np.random.default_rng(40 + len(cs))
        B = _Bow(rng, 400, 400)
        angles = rot_angles(rng, plan)
        kperm, fperm = rng.permutation(400), rng.permutation(400)
        for g in range(len(angles)):
            a, b = kperm[4 * g:4 * g + 4], fperm[4 * g:4 * g + 4]
            B.node(g, a, b)
            B.plant(int(a[0]), int(b[0]), int(rng.integers(0, 40)), angles[g])
        cs.append(B.case('rot_' + pname, dict(plan=plan), min_matches=len(angles)))
    return cs


# ---------------------------------------------------------------------------------------------
# SearchForTriangulation: one keyframe against several neighbours
# ---------------------------------------------------------------------------------------------
# F12 of a rectified pair (pure x translation): ea = 0, eb = 1, ec = -y1, so the epipolar test passes iff (y2 - y1)^2 < 3.84 sigma2
F_RECT = np.array([0, 0, 0, 0, 0, -1, 0, 1, 0], np.float32)
F_DEN0 = np.array([0, 0, 0, 0, 0, 0, 0, 0, 1], np.float32)      # ea = eb = 0: den == 0
EP_FAR = np.array([-900.0, -900.0], np.float32)


def _tri_kf(rng, n, oct_max=7):
    return dict(kps=keypoints(n, rng, octave=rng.integers(0, oct_max + 1, n)), desc=rng.integers(0, 256, (n, 32), dtype=np.uint8),
                has_mp=np.zeros(n, np.uint8), fv=([], []))


def _fv(nodes):
    nodes = sorted(nodes, key=lambda t: t[0])
    return (np.array([nid for nid, fs in nodes for _ in fs], np.int32), np.array([x for _, fs in nodes for x in fs], np.int32))


def _tri_plant(rng, kf1, kf2, i, j, d, angles=None, dy=None):
    kf2['desc'][j] = flip(kf1['desc'][i], rng, d)
    kf2['kps']['y'][j] = f32(kf1['kps']['y'][i] + (rng.uniform(-0.9, 0.9) if dy is None else dy))
    if angles is None:
        angles = _rot_pair(rng, int(rng.choice([0, 0, 0, 1, 1, 6, 10])), False)
    kf1['kps']['angle'][i], kf2['kps']['angle'][j] = angles


def _tri_case(name, shape, kf1, kf2s, eps=None, F12s=None, coarse=False, min_matches=8):
    n = len(kf2s)
    tab = tables()
    return dict(kind='tri', name=name, shape=shape, kf1=kf1, kf2=kf2s, sf=tab['scale'], sigma2=tab['sigma2'],
                ep=np.array(eps if eps is not None else [EP_FAR] * n, np.float32).reshape(n, 2),
                F12=np.array(F12s if F12s is not None else [F_RECT] * n, np.float32).reshape(n, 9), coarse=coarse, min_matches=min_matches)


def _tri_nodes(rng, n1, e1, n2, g, node2=None, p=0.8, nn=3):
    """KF1 of n1 features, e1 of them in g nodes; nn neighbours of n2 features with node sizes node2 (or spread); plants with probability p."""
    kf1 = _tri_kf(rng, n1)
    feats1 = _split(rng, rng.permutation(n1)[:e1], g)
    ids = np.sort(rng.choice(10 ** 5, g, replace=False))
    kf1['fv'] = _fv(list(zip(ids, feats1)))
    kf2s = []
    for k in range(nn):
        kf2 = _tri_kf(rng, n2)
        perm = rng.permutation(n2)
        if node2 is None:
            feats2 = _split(rng, perm, g)
        else:
            feats2 = [perm[node2 * t:node2 * t + node2] for t in range(g)]
        nodes = []
        for nid, a, b in zip(ids, feats1, feats2):
            if len(b) == 0:
                continue
            nodes.append((nid, b))
            for i in a:
                if rng.random() < p:
                    _tri_plant(rng, kf1, kf2, int(i), int(rng.choice(b)), int(rng.integers(0, 48)))
        kf2['fv'] = _fv(nodes)
        kf2s.append(kf2)
    return kf1, kf2s


def _epipole_bar(seed):
    """KF2 keypoints of octaves 0 and 3 at exactly 100 * scaleFactor squared distance from the epipole (kept: the test is `<`) and one float
    step closer (rejected); each is the only candidate of its own KF1 feature."""
    rng = np.random.default_rng(seed)
    sf = tables()['scale']
    kf1, kf2 = _tri_kf(rng, 64), _tri_kf(rng, 64)
    ep = np.array([300.0, 200.0], np.float32)
    nodes1, nodes2, info = [], [], []
    for t, (oct_, inside) in enumerate([(0, False), (0, True), (3, False), (3, True)] * 4):
        T = f32(f32(100.0) * f32(sf[oct_]))
        dx = next((x for x in _ulps(f32(np.sqrt(np.float64(T))), 64) if f32(np.float64(x) * np.float64(x)) == T), None)
        if dx is None:              # no float32 dx squares to T exactly: take the smallest one at or above it
            dx = min((x for x in _ulps(f32(np.sqrt(np.float64(T))), 64) if f32(np.float64(x) * np.float64(x)) >= T))
        x2 = f32(ep[0] + dx)
        if inside:
            x2 = np.nextafter(x2, f32(-np.inf))
        i, j = 4 * t, 4 * t + 1
        kf1['kps']['y'][i] = ep[1]
        kf2['kps']['x'][j], kf2['kps']['y'][j], kf2['kps']['octave'][j] = x2, ep[1], oct_
        _tri_plant(rng, kf1, kf2, i, j, 10 + t, dy=0.0)
        kf1['kps']['octave'][i] = oct_
        nodes1.append((t, [i])); nodes2.append((t, [j, 4 * t + 2]))
        info.append(dict(i=i, j=j, octave=oct_, inside=inside))
    kf1['fv'], kf2['fv'] = _fv(nodes1), _fv(nodes2)
    return kf1, kf2, ep, info


def tri_cases():
    cs = []
    for e1 in (1, 7, 8, 9):
        rng = np.random.default_rng(100 + e1)
        kf1, kf2s = _tri_nodes(rng, 40, e1, 60, e1, p=1.0, nn=4)
        cs.append(_tri_case('E1_%d' % e1, dict(E1=e1, N1=40), kf1, kf2s, min_matches=min(e1 * 4, 8)))
    for n1 in (255, 256, 257, 2048):
        rng = np.random.default_rng(110 + n1)
        kf1, kf2s = _tri_nodes(rng, n1, n1 - 5, min(n1, 1000), max(1, n1 // 8), nn=3)
        cs.append(_tri_case('N1_%d' % n1, dict(N1=n1, E1=n1 - 5), kf1, kf2s))
    for s in (31, 32, 33, 500):
        rng = np.random.default_rng(120 + s)
        kf1, kf2s = _tri_nodes(rng, 60, 40, max(10 * s, 600), 10, node2=s, nn=3)
        cs.append(_tri_case('kf2_node_%d' % s, dict(kf2_node_size=s), kf1, kf2s))
    # equal minimal distances: the last position wins
    rng = np.random.default_rng(130)
    kf1, kf2 = _tri_kf(rng, 64), _tri_kf(rng, 1700)
    n1, n2 = [], []
    for g, (p, q) in enumerate([(0, 1), (0, 32), (3, 35), (5, 40), (31, 32), (1, 69), (40, 5), (64, 2)] * 3):
        i, feats = 2 * g, list(range(70 * g, 70 * g + 70))
        d = 5 + g % 30
        _tri_plant(rng, kf1, kf2, i, feats[p], d)
        _tri_plant(rng, kf1, kf2, i, feats[q], d)
        kf2['kps']['octave'][feats[p]] = kf2['kps']['octave'][feats[q]] = 0
        n1.append((g, [i])); n2.append((g, feats))
    kf1['fv'], kf2['fv'] = _fv(n1), _fv(n2)
    cs.append(_tri_case('lane_ties', dict(tie_positions=True), kf1, [kf2]))
    # distances 49 / 50 / 51 (<= TH_LOW)
    rng = np.random.default_rng(131)
    kf1, kf2 = _tri_kf(rng, 90), _tri_kf(rng, 900)
    n1, n2 = [], []
    for g in range(90):
        _tri_plant(rng, kf1, kf2, g, 10 * g, (49, 50, 51)[g % 3])
        n1.append((g, [g])); n2.append((g, range(10 * g, 10 * g + 10)))
    kf1['fv'], kf2['fv'] = _fv(n1), _fv(n2)
    cs.append(_tri_case('th_low_50_51', dict(best=(49, 50, 51)), kf1, [kf2]))
    # the epipole-distance test at its bar
    kf1, kf2, ep, info = _epipole_bar(132)
    c = _tri_case('epipole_bar', dict(epipole=info), kf1, [kf2], eps=[ep])
    cs.append(c)
    cs.append(dict(c, name='epipole_bar_coarse', coarse=True))
    # den == 0: every non-coarse candidate rejected, coarse mode still matches
    rng = np.random.default_rng(133)
    kf1, kf2s = _tri_nodes(rng, 300, 280, 300, 30, nn=2)
    cs.append(_tri_case('den0', dict(den0=True), kf1, kf2s, F12s=[F_DEN0] * 2, min_matches=0))
    cs.append(_tri_case('den0_coarse', dict(den0=True), kf1, kf2s, F12s=[F_DEN0] * 2, coarse=True))
    # hasMapPoint on either side; a neighbour without features and one without FeatureVector entries among normal ones
    rng = np.random.default_rng(134)
    kf1, kf2s = _tri_nodes(rng, 500, 480, 500, 60, nn=4)
    kf1['has_mp'] = (rng.random(500) < 0.3).astype(np.uint8)
    for k in kf2s:
        k['has_mp'] = (rng.random(500) < 0.3).astype(np.uint8)
    empty = dict(kps=kf2s[0]['kps'][:0], desc=kf2s[0]['desc'][:0], has_mp=kf2s[0]['has_mp'][:0], fv=(np.zeros(0, np.int32), np.zeros(0, np.int32)))
    no_fv = dict(kf2s[1], fv=(np.zeros(0, np.int32), np.zeros(0, np.int32)))
    cs.append(_tri_case('has_mp_and_empty', dict(has_mp=True, N2=0, E2=0), kf1, [kf2s[0], empty, kf2s[1], no_fv, kf2s[2], kf2s[3]]))
    # rotation plans
    for pname, plan in ROT_PLANS.items():
        rng = np.random.default_rng(140 + len(cs))
        angles = rot_angles(rng, plan)
        kf1, kf2 = _tri_kf(rng, 4 * len(angles)), _tri_kf(rng, 4 * len(angles))
        n1, n2 = [], []
        for g, a in enumerate(angles):
            _tri_plant(rng, kf1, kf2, 4 * g, 4 * g + 1, int(rng.integers(0, 40)), a)
            n1.append((g, [4 * g, 4 * g + 2])); n2.append((g, [4 * g + 1, 4 * g + 3]))
        kf1['fv'], kf2['fv'] = _fv(n1), _fv(n2)
        cs.append(_tri_case('rot_' + pname, dict(plan=plan), kf1, [kf2], min_matches=len(angles)))
    return cs


# ---------------------------------------------------------------------------------------------
# Fuse / SearchBySim3
# ---------------------------------------------------------------------------------------------
def frame_smem_bytes(ks, ms, desc):
    """matcher.cu's frame_smem_bytes: the dynamic shared memory of a CTA for ks keypoints and ms map points."""
    al = lambda v: (v + 15) & ~15
    b = al(4 * 64 * 48) + al(2 * (64 * 48 + 1)) + al(2 * ks) + 2 * al(4 * ks) + al(ks) + al(4 * ((ks + 31) // 32)) + al(4 * ks)
    b += 2 * al(2 * ms) + al(ms)
    return b + (al(32 * ks) if desc else 0)


def fuse_layout(K):
    """fuse_search_run's frame_layout for a keyframe of K keypoints: 'smem' (descriptors in shared memory), 'global' or 'refused'."""
    if frame_smem_bytes(K, 1, True) <= SMEM_LIMIT:
        return 'smem'
    return 'global' if frame_smem_bytes(K, 1, False) <= SMEM_LIMIT else 'refused'


K_SMEM_MAX = max(k for k in range(4000, 5000) if fuse_layout(k) == 'smem')                 # 4496
K_MAX = max(k for k in range(13000, 15000) if fuse_layout(k) != 'refused')                 # 14008
IDENTITY = np.array([1, 0, 0, 0, 0, 0, 0], np.float32)


def project(cam, p):
    """Fuse's projection of a camera-frame point in float32: u = fx * x / z + cx."""
    fx, fy, cx, cy = (f32(c) for c in cam)
    return f32(f32(f32(fx * f32(p[0])) / f32(p[2])) + cx), f32(f32(f32(fy * f32(p[1])) / f32(p[2])) + cy)


def dist3(p):
    p = [f32(c) for c in p]
    return f32(np.sqrt(f32(f32(f32(p[0] * p[0]) + f32(p[1] * p[1])) + f32(p[2] * p[2]))))


class _Fuse:
    """A keyframe with the identity pose (camera = world frame) and map points planted on its keypoints."""

    def __init__(self, rng):
        tab = tables()
        self.rng = rng
        self.cam = np.array([458.0, 458.0, 320.0, 240.0], np.float32)
        self.kps, self.desc = [], []
        self.pts = dict(state=[], xyz=[], normal=[], min_d=[], max_d=[], mp_desc=[])
        self.sf, self.isg, self.log_sf = tab['scale'], tab['inv_sigma2'], f32(np.log(f32(1.2)))
        self.marks = {}

    def kp(self, x, y, octave, desc=None):
        self.kps.append((f32(x), f32(y), octave))
        self.desc.append(self.rng.integers(0, 256, 32, dtype=np.uint8) if desc is None else desc)
        return len(self.kps) - 1

    def point(self, xyz, desc, level=None, state=1, normal=None, min_d=None, max_d=None):
        xyz = np.asarray(xyz, np.float32)
        d = float(dist3(xyz))
        if max_d is None:
            max_d = f32(d * 1.2 ** ((level if level is not None else 1) - 0.5))
        if min_d is None:
            min_d = f32(max_d / 1.2 ** 7)
        if normal is None:
            normal = (xyz / np.linalg.norm(xyz.astype(np.float64))).astype(np.float32)
        for k, v in (('state', state), ('xyz', xyz), ('normal', normal), ('min_d', f32(min_d)), ('max_d', f32(max_d)), ('mp_desc', desc)):
            self.pts[k].append(v)
        return len(self.pts['state']) - 1

    def at(self, u, v, z):
        """A camera-frame point projecting to about (u, v) at depth z."""
        fx, fy, cx, cy = (float(c) for c in self.cam)
        return np.array([(u - cx) / fx * z, (v - cy) / fy * z, z], np.float32)

    def planted(self, j, d, level=None, z=None):
        """A map point on keypoint j with descriptor distance d, predicted level = its octave unless given."""
        x, y, o = self.kps[j]
        p = self.at(float(x), float(y), z or self.rng.uniform(2, 9))
        return self.point(p, flip(self.desc[j], self.rng, d), level=o if level is None else level)

    def case(self, name, shape, min_matches=8, th=3.0):
        k = np.zeros(len(self.kps), KP_DTYPE)
        if len(self.kps):
            k['x'], k['y'], k['octave'] = zip(*self.kps)
        k['size'], k['class_id'] = 31.0, -1
        k['angle'] = self.rng.uniform(0, 360, len(k))
        k['response'] = self.rng.uniform(1e-4, 1e-2, len(k))
        M = len(self.pts['state'])
        pts = dict(state=np.array(self.pts['state'], np.uint8), xyz=np.array(self.pts['xyz'], np.float32).reshape(M, 3),
                   normal=np.array(self.pts['normal'], np.float32).reshape(M, 3), min_d=np.array(self.pts['min_d'], np.float32),
                   max_d=np.array(self.pts['max_d'], np.float32), mp_desc=np.array(self.pts['mp_desc'], np.uint8).reshape(M, 32))
        return dict(kind='fuse', name=name, shape=shape, kps=k, desc=np.array(self.desc, np.uint8).reshape(len(k), 32), bounds=BOUNDS, sf=self.sf,
                    isg=self.isg, log_sf=self.log_sf, Tcw=IDENTITY.copy(), Ow=np.zeros(3, np.float32), cam=self.cam, th=th, marks=dict(self.marks),
                    min_matches=min_matches, **pts)


def _fuse_random(K, M, seed, frac=0.6):
    """K random keypoints (octaves 0..7), M map points: a fraction planted on keypoints at distances 0..59, the rest anywhere; states 0 / 1 / 2 / 3."""
    rng = np.random.default_rng(seed)
    F = _Fuse(rng)
    xs, ys, os_ = rng.uniform(0, 640, K), rng.uniform(0, 480, K), rng.integers(0, 8, K)
    for x, y, o in zip(xs, ys, os_):
        F.kp(x, y, int(o))
    for m in range(M):
        if rng.random() < frac:
            F.planted(int(rng.integers(0, K)), int(rng.integers(0, 60)))
        else:
            F.point(F.at(rng.uniform(-20, 660), rng.uniform(-20, 500), rng.uniform(1, 12)), rng.integers(0, 256, 32, dtype=np.uint8), int(rng.integers(0, 8)))
        F.pts['state'][-1] = int(rng.choice([0, 1, 1, 1, 1, 1, 1, 2, 3]))
    return F


def _fuse_real(t, M, seed):
    """oracle_lib.fuse_scene(t) with its map points resampled (with noise) to M."""
    sc = O.fuse_scene(t)
    rng = np.random.default_rng(seed)
    sel = rng.integers(0, len(sc['state']), M) if M > len(sc['state']) else rng.permutation(len(sc['state']))[:M]
    out = dict(sc, **{k: np.ascontiguousarray(sc[k][sel]) for k in ('state', 'xyz', 'normal', 'min_d', 'max_d', 'mp_desc')})
    if M > len(sc['state']):
        out['xyz'] = (out['xyz'] + rng.normal(0, 0.002, out['xyz'].shape)).astype(np.float32)
    return dict(out, kind='fuse', name='real_M_%d' % M, shape=dict(M=M, ctas=min(16, (M + 127) // 128)), th=3.0, marks={},
                min_matches=1 if M < 128 else 8)


def _fuse_edges(seed):
    """Each test of the search with a pair of map points on either side of it, at spots 40 px apart with only the planted keypoints; cell-border
    keypoints; a cell with more than 1000 keypoints; predicted levels 0 and nlevels - 1; equal distances in GetFeaturesInArea order."""
    rng = np.random.default_rng(seed)
    F = _Fuse(rng)
    spots = iter([(60.0 + 40 * a, 60.0 + 40 * b) for b in range(9) for a in range(13)])
    marks = F.marks
    # image bounds: u == minX is in, u == maxX is out (x solved so that the projection is exactly the bound)
    for name, target in (('u_min', 0.0), ('u_max', 640.0)):
        y = 120.0 + 60 * len(marks)
        j = F.kp(target + (0.6 if target == 0 else -0.6), y, 0)
        z = f32(4.0)
        x0 = f32((target - 320.0) / 458.0 * 4.0)
        px = next(x for x in _ulps(x0, 4096) if project(F.cam, (x, f32((y - 240.0) / 458.0 * 4.0), z))[0] == f32(target))
        p = np.array([px, (y - 240.0) / 458.0 * 4.0, z], np.float32)
        marks[name] = F.point(p, flip(F.desc[j], rng, 5), level=0), j
    # the other tests at free spots: (in, out) map points and the keypoint each should find
    def spot_kp(o=0):
        x, y = next(spots)
        return F.kp(x + 0.4, y - 0.3, o), x, y
    # 0.8 * minD and 1.2 * maxD
    j, x, y = spot_kp(1)
    p = F.at(x, y, 5.0); d = dist3(p)
    lo, hi = straddle(lambda m: d < f32(f32(0.8) * f32(m)), f32(d / 0.8))
    marks['min_d'] = (F.point(p, flip(F.desc[j], rng, 4), level=1, min_d=lo), F.point(p, flip(F.desc[j], rng, 4), level=1, min_d=hi), j)
    j, x, y = spot_kp(0)
    p = F.at(x, y, 5.0); d = dist3(p)
    lo, hi = straddle(lambda m: d > f32(f32(1.2) * f32(m)), f32(d / 1.2))
    marks['max_d'] = (F.point(p, flip(F.desc[j], rng, 4), max_d=hi), F.point(p, flip(F.desc[j], rng, 4), max_d=lo), j)
    # the viewing angle: dot < 0.5 * dist3D
    j, x, y = spot_kp(1)
    p = F.at(x, y, 6.0); d = dist3(p)
    nx, ny = f32(0.3), f32(-0.2)
    dot = lambda nz: f32(f32(f32(p[0] * nx) + f32(p[1] * ny)) + f32(p[2] * f32(nz)))
    lo, hi = straddle(lambda nz: np.float64(dot(nz)) < 0.5 * np.float64(d), f32((0.5 * d - p[0] * nx - p[1] * ny) / p[2]))
    marks['view'] = (F.point(p, flip(F.desc[j], rng, 4), level=1, normal=np.array([nx, ny, hi], np.float32)),
                     F.point(p, flip(F.desc[j], rng, 4), level=1, normal=np.array([nx, ny, lo], np.float32)), j)
    # the chi-square gate at 5.99 (octave 0: invSigma2 = 1), e2 = ex^2 with ey = 0
    for o in (0, 2):
        x, y = next(spots)
        p = F.at(x, y, 3.0)
        u, v = project(F.cam, p)
        isg = f32(F.isg[o])
        gate = lambda kx: np.float64(f32(f32(np.float64(f32(u - f32(kx))) ** 2) * isg)) > 5.99
        inside, outside = straddle(gate, f32(u - np.sqrt(5.99 / isg)))[::-1]
        ja = F.kp(inside, v, o)
        x2, y2 = next(spots)
        p2 = F.at(x2, y2, 3.0)
        u2, v2 = project(F.cam, p2)
        jb = F.kp(f32(u2 - f32(u - outside)), v2, o)
        assert f32(u2 - F.kps[jb][0]) == f32(u - outside)
        marks['chi2_oct%d' % o] = (F.point(p, flip(F.desc[ja], rng, 3), level=o), F.point(p2, flip(F.desc[jb], rng, 3), level=o), ja, jb)
    # zc < 0 (projects onto its keypoint all the same), states 0 / 2 / 3 next to state 1
    j, x, y = spot_kp(1)
    p = F.at(x, y, 4.0)
    marks['zc_neg'] = (F.point(p, flip(F.desc[j], rng, 4), level=1), F.point(-p, flip(F.desc[j], rng, 4), level=1), j)
    j, x, y = spot_kp(1)
    p = F.at(x, y, 4.0)
    marks['states'] = tuple(F.point(p, flip(F.desc[j], rng, 4), level=1, state=s) for s in (1, 0, 2, 3)) + (j,)
    # predicted level 0 (window [-1, 0]) and nlevels - 1 = 7 (maxD far above: the prediction clamps)
    for lvl in (0, 7):
        j, x, y = spot_kp(lvl)
        p = F.at(x, y, 4.0)
        marks['level_%d' % lvl] = (F.point(p, flip(F.desc[j], rng, 6), max_d=f32(dist3(p) * 1.2 ** (lvl + 3.0 if lvl else -0.5)), min_d=f32(dist3(p) / 2)), j)
    # equal distances: the first keypoint in GetFeaturesInArea order (cell column, cell row, position in the cell) wins, not the lowest index
    for name, (ax, ay, bx, by) in (('tie_rows', (0, 1.2, 0, -1.2)), ('tie_cols', (1.2, -1.0, -1.2, 1.0)), ('tie_cell', (0.6, 0.3, -0.6, -0.3))):
        x, y = next(spots)
        # a cell corner (PosInGrid rounds, so cells are centred on multiples of 10), or a cell centre for the tie inside one cell
        cx_, cy_ = (f32(x), f32(y)) if name == 'tie_cell' else (f32(x + 5.0), f32(y + 5.0))
        base = rng.integers(0, 256, 32, dtype=np.uint8)
        ja = F.kp(cx_ + ax, cy_ + ay, 1, flip(base, rng, 7))         # lower index, later in enumeration order (except in one cell)
        jb = F.kp(cx_ + bx, cy_ + by, 1, flip(base, rng, 7))
        marks[name] = (F.point(F.at(float(cx_), float(cy_), 5.0), base, level=1), ja, jb)
    # keypoints exactly on cell borders (PosInGrid's (p - min) * inv == k + 0.5) and map points around them
    border = []
    for c in range(10):
        bx, by = MS.cell_coord(BOUNDS, 20.5 + c, 0), MS.cell_coord(BOUNDS, 30.5 + (c % 4), 1)
        border.append(F.kp(bx, by, int(rng.integers(0, 3))))
        border.append(F.kp(bx, MS.cell_coord(BOUNDS, 40.0 + (c % 5), 1), int(rng.integers(0, 3))))
    for j in border:
        F.planted(j, int(rng.integers(0, 40)))
        F.point(F.at(float(F.kps[j][0]) + rng.uniform(-3, 3), float(F.kps[j][1]) + rng.uniform(-3, 3), rng.uniform(2, 6)),
                flip(F.desc[j], rng, int(rng.integers(0, 40))), level=F.kps[j][2])
    marks['border'] = border
    # one cell with 1100 keypoints, searched by 150 map points
    crowd = [F.kp(rng.uniform(595.6, 604.4), rng.uniform(435.6, 444.4), int(rng.integers(0, 3))) for _ in range(1100)]
    for j in rng.choice(crowd, 150, replace=False):
        F.planted(int(j), int(rng.integers(0, 50)))
    marks['crowd'] = crowd
    return F.case('edges', dict(tests=sorted(marks)), min_matches=20)


def fuse_cases():
    cs = []
    for K in (K_SMEM_MAX, K_SMEM_MAX + 1, K_MAX):
        c = _fuse_random(K, 2500, 200 + K % 97).case('K_%d' % K, dict(K=K, layout=fuse_layout(K)))
        cs.append(c)
    cs += [_fuse_real(7 + i % 5, M, 300 + M) for i, M in enumerate((1, 127, 128, 129, 1920, 1921, 2048, 2049, 20000))]
    cs.append(_fuse_edges(400))
    return cs


def refused_keyframe():
    """A keyframe of K_MAX + 1 keypoints (no layout fits) with a few map points."""
    return _fuse_random(K_MAX + 1, 50, 500).case('K_%d' % (K_MAX + 1), dict(K=K_MAX + 1, layout='refused'), min_matches=0)


def sim3_cases():
    """SearchBySim3: oracle_lib.sim3_scene (real features), and keyframes of K_SMEM_MAX + 1 and K_MAX features seen with the identity Sim3:
    KF2 = KF1's keypoints with descriptors a few bits apart, each feature's map point on its keypoint."""
    out = []
    sc = O.sim3_scene(9)
    p21, p12 = O.sim3_camera_points(sc)
    side = lambda k, pc: dict(kps=sc['k%d' % k], desc=sc['d%d' % k], state=sc['state%d' % k], pcam=pc, min_d=sc['min%d' % k], max_d=sc['max%d' % k],
                              mp_desc=sc['mpd%d' % k])
    out.append(dict(kind='sim3', name='sim3_real', shape=dict(K=len(sc['k1'])), kf1=side(1, p21), kf2=side(2, p12), sf=sc['sf'], log_sf=sc['log_sf'],
                    cam=sc['cam'], pre12=sc['pre12'], th=7.5, min_matches=8))
    for K in (K_SMEM_MAX + 1, K_MAX):
        F = _fuse_random(K, 0, 600 + K % 89)
        rng = F.rng
        base = F.case('x', {})
        kfs = []
        for s in range(2):
            pc, mpd = [], []
            for j, (x, y, o) in enumerate(F.kps):
                pc.append(F.at(float(x), float(y), rng.uniform(2, 9)))
            pc = np.array(pc, np.float32)
            dist = np.linalg.norm(pc.astype(np.float64), axis=1)
            max_d = (dist * 1.2 ** (base['kps']['octave'] - 0.5)).astype(np.float32)
            desc = base['desc'] if s == 0 else np.array([flip(dd, rng, int(rng.integers(0, 6))) for dd in base['desc']], np.uint8)
            kfs.append(dict(kps=base['kps'], desc=desc, state=rng.choice([0, 1, 1, 1, 1, 2], K).astype(np.uint8), pcam=pc, min_d=(max_d / f32(1.2 ** 7)).astype(np.float32),
                            max_d=max_d, mp_desc=np.array([flip(dd, rng, int(rng.integers(0, 30))) for dd in desc], np.uint8)))
        pre = np.full(K, -1, np.int32)
        good2 = np.flatnonzero(kfs[1]['state'] == 1)
        pre[np.flatnonzero(kfs[0]['state'] == 1)[:40:4]] = rng.choice(good2, 10, replace=False)
        out.append(dict(kind='sim3', name='sim3_K_%d' % K, shape=dict(K=K, layout=fuse_layout(K)), kf1=kfs[0], kf2=kfs[1], sf=F.sf, log_sf=F.log_sf,
                        cam=F.cam, pre12=pre, th=7.5, min_matches=8))
    return out


# ---------------------------------------------------------------------------------------------
# CreateNewMapPoints: 65,535 (keyframe, neighbour) pairs in one call
# ---------------------------------------------------------------------------------------------
MAX_PAIRS = 65535


def wide_new_points():
    """Three items of orbm_create_new_map_points_batch with MAX_PAIRS pairs in all: item 0 has the largest KF1 (it sets maxN1) and one
    neighbour; item 1 a 6-feature KF1 with MAX_PAIRS - 2 one-feature neighbours (the most pairs), each holding the match of one KF1
    feature in the real neighbour it is cut from; item 2, whose pair is the call's last, a real scene with a smaller KF1."""
    n1 = {t: len(MS.extract(t)[0]) for t in range(16, 24)}
    big = NP.scene(max(n1, key=n1.get), (3,))
    last = NP.scene(min(n1, key=n1.get), (2,))
    src = NP.scene(18, (3,))
    n_wide = MAX_PAIRS - 2
    kf1 = src['kf1']
    rec = NP.create(src)[0]                                          # KF1's new points with the neighbour: each tiny neighbour holds one
    m12 = np.full(len(kf1['kps']), -1, np.int32)
    m12[rec['idx1']] = rec['idx2']
    keep = np.sort(rec['idx1'][:6])
    remap = {int(f): i for i, f in enumerate(keep)}
    sel = np.isin(kf1['fv'][1], keep)
    small1 = dict(kps=kf1['kps'][keep], desc=kf1['desc'][keep], has_mp=np.zeros(6, np.uint8),
                  fv=(kf1['fv'][0][sel], np.array([remap[int(f)] for f in kf1['fv'][1][sel]], np.int32)))
    nb = src['kf2'][0]
    nodes = {int(f): int(n) for n, f in zip(*nb['fv'])}
    tiny = []
    for k in range(n_wide):
        f = int(m12[keep[k % len(keep)]])
        tiny.append(dict(kps=nb['kps'][f:f + 1], desc=nb['desc'][f:f + 1], has_mp=np.zeros(1, np.uint8),
                         fv=(np.array([nodes[f]], np.int32), np.zeros(1, np.int32))))
    wide = dict(src, kf1=small1, kf2=tiny, ep=np.tile(src['ep'], (n_wide, 1)), F12=np.tile(src['F12'], (n_wide, 1)),
                Tcw=np.concatenate([src['Tcw'][:1], np.tile(src['Tcw'][1:], (n_wide, 1, 1))]), Ow=np.concatenate([src['Ow'][:1], np.tile(src['Ow'][1:], (n_wide, 1))]),
                cam=np.tile(src['cam'][:1], (n_wide + 1, 1)))
    assert len(big['kf1']['kps']) > len(last['kf1']['kps']) > len(small1['kps'])
    return [big, wide, last]
