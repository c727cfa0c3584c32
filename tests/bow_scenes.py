"""Vocabularies and frames for the DBoW2 transform's tests (CPU only, seeded), and a numpy restatement of the transform written from
DBoW2's text (TemplatedVocabulary::transform, Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1127-1259; BowVector::addWeight /
addIfNotExist / normalize, BowVector.cpp:35-88; FeatureVector::addFeature, FeatureVector.cpp:30-45) without the oracle's or the
kernels' code.

A vocabulary is a dict in the flat OrbVocabulary layout of include/orb_b200.h (L, child_start, children, desc, weight, word_id) plus
parent [nNodes] (-1 for the root) and depth [nNodes], from which the checks find a feature's ancestors without any descent, and ties:
the (node, p, q) sibling pairs whose descriptors are identical, p and q being positions in the node's child list."""
import functools
import math
from fractions import Fraction

import numpy as np

#: the trees of the tests: name -> keyword arguments of random_tree.  Child counts are drawn from 1..k (the root takes k, plus one leaf),
#: so k = 16, 17, 32, 33 and 64 give nodes whose children a half-warp of 16 lanes walks in 2, 3 or 5 strides.
TREES = {
    'k1_chain': dict(k=1, L=6, seed=1),
    'k10_L5': dict(k=10, L=5, seed=2),
    'k16_L4': dict(k=16, L=4, seed=3),
    'k17_L4': dict(k=17, L=4, seed=4),
    'k32_L3': dict(k=32, L=3, seed=5),
    'k33_L3': dict(k=33, L=3, seed=6),
    'k64_L3': dict(k=64, L=3, seed=7),
    'k17_stop0': dict(k=17, L=3, seed=8, stop=0.0),
    'k17_stop_half': dict(k=17, L=3, seed=9, stop=0.5),
    'k10_stop_all': dict(k=10, L=4, seed=10, stop=1.0),
    'k33_id_order': dict(k=33, L=3, seed=11, shuffle=False, relabel=False, permute_words=False),
}
#: list positions of the planted sibling ties; 'last' = the last two children of a node
TIE_POSITIONS = ((0, 1), (15, 16), (16, 32), 'last')

POPCOUNT = np.array([bin(i).count('1') for i in range(256)], np.uint8)


def _flip(rng, d, nbits):
    """d with nbits random bits flipped (a bit may be drawn twice)."""
    d = d.copy()
    b = rng.integers(0, 256, nbits)
    np.bitwise_xor.at(d, b >> 3, (1 << (b & 7)).astype(np.uint8))
    return d


def _finish(rng, parent, desc, L, stop, shuffle, permute_words, ties=()):
    """The flat layout of a tree given by its parent array (node 0 the root): child lists in node-id order or shuffled, word ids over
    the leaves in node-id order or permuted, idf-like weights with a fraction `stop` of the leaves stopped (weight 0), and the ties
    planted: for each entry of `ties` a node with enough children, the child at position q given the descriptor of the one at p."""
    parent = np.asarray(parent, np.int64)
    n = len(parent)
    kids = [[] for _ in range(n)]
    for i in range(1, n):
        kids[parent[i]].append(i)
    if shuffle:
        for lst in kids:
            rng.shuffle(lst)
    child_start = np.zeros(n + 1, np.int32)
    child_start[1:] = np.cumsum([len(c) for c in kids])
    children = np.array([c for lst in kids for c in lst], np.int32)
    depth = np.zeros(n, np.int32)
    for i in _bfs(child_start, children)[1:]:     # a parent before its children, whatever the node ids

        depth[i] = depth[parent[i]] + 1
    leaves = np.flatnonzero(np.diff(child_start) == 0)
    word_id = np.full(n, -1, np.int32)
    word_id[leaves] = rng.permutation(len(leaves)) if permute_words else np.arange(len(leaves))
    weight = np.zeros(n)
    weight[leaves] = rng.uniform(0.5, 9.0, len(leaves))
    weight[rng.choice(leaves, int(round(stop * len(leaves))), replace=False)] = 0.0
    desc = np.array(desc, np.uint8)
    planted, shadowed = [], set()          # shadowed: the q children, which the descent never enters
    count = np.diff(child_start)

    def line(i):                           # i and its ancestors
        return [i] + line(int(parent[i])) if i > 0 else [0]

    need_of = lambda pq: 2 if pq == 'last' else pq[1] + 1                # noqa: E731
    for pq in sorted(ties, key=need_of, reverse=True):                   # the rarest nodes first
        need = need_of(pq)
        cand = []
        for node in np.flatnonzero(count >= need):
            p, q = (count[node] - 2, count[node] - 1) if pq == 'last' else pq
            qc = int(children[child_start[node] + q])
            # every tie stays reachable: none below a shadowed child, and no shadowed child above an earlier tie
            if node not in {t for t, _, _ in planted} and not shadowed & set(line(int(node))) and \
                    not any(qc in line(t) for t, _, _ in planted):
                cand.append((int(node), int(p), int(q), qc))
        if not cand:
            continue
        node, p, q, qc = cand[rng.integers(0, len(cand))]
        a = child_start[node]
        desc[qc] = desc[children[a + p]]
        shadowed.add(qc)
        planted.append((node, p, q))
    return dict(L=L, parent=parent, depth=depth, desc=desc, weight=weight, child_start=child_start, children=children, word_id=word_id,
                n_words=len(leaves), ties=planted)


def _bfs(child_start, children):
    order, head = [0], 0
    while head < len(order):
        i = order[head]
        head += 1
        order.extend(children[child_start[i]:child_start[i + 1]].tolist())
    return order


def random_tree(k, L, seed, stop=0.02, leaf_p=0.15, shuffle=True, relabel=True, permute_words=True):
    """A DBoW2-like tree of depth L: the root has k children plus one leaf, every other inner node 1..k (what k-means gives a node with
    few descriptors); below the root a node above depth L is a leaf with probability leaf_p.  A child's descriptor is its parent's
    with a few bits flipped.  relabel: node ids 1.. permuted against the construction (BFS) order; shuffle: child lists not in id order;
    permute_words: word ids not in node order.  Ties are planted at TIE_POSITIONS where a node has the children for them."""
    rng = np.random.default_rng(seed)
    parent, desc = [-1], [rng.integers(0, 256, 32).astype(np.uint8)]
    frontier = [0]
    for lv in range(1, L + 1):
        nxt = []
        for p in frontier:
            cnt = k + 1 if p == 0 else int(rng.integers(1, k + 1))
            for c in range(cnt):
                parent.append(p)
                desc.append(rng.integers(0, 256, 32).astype(np.uint8) if lv == 1 else _flip(rng, desc[p], 60 // lv))
                root_leaf = p == 0 and c == cnt - 1
                if lv < L and not root_leaf and rng.random() >= leaf_p:
                    nxt.append(len(parent) - 1)
        frontier = nxt
    n = len(parent)
    parent, desc = np.array(parent), np.stack(desc)
    if relabel:
        new = np.concatenate([[0], 1 + rng.permutation(n - 1)])        # new[old]
        p2 = np.empty(n, np.int64); d2 = np.empty_like(desc)
        p2[new] = np.where(parent >= 0, new[np.maximum(parent, 0)], -1)
        d2[new] = desc
        parent, desc = p2, d2
    return _finish(rng, parent, desc, L, stop, shuffle, permute_words, TIE_POSITIONS)


def orbvoc_tree(seed=0, k=10, L=6, stop=0.02):
    """The shape of ORB-SLAM3's ORBvoc.txt: a full k-ary tree of depth L (k = 10, L = 6: 1,111,111 nodes, 10^6 words), built level by
    level with numpy.  Node ids in BFS order, each child list shuffled, word ids permuted; children's descriptors are their parent's
    with about 32, 16 or 8 bits flipped (levels 2, 3-4, 5-6)."""
    rng = np.random.default_rng(seed)
    sizes = [k ** lv for lv in range(L + 1)]
    start = np.concatenate([[0], np.cumsum(sizes)])
    n, n_inner = int(start[-1]), int(start[L])
    desc = np.zeros((n, 32), np.uint8)
    desc[1:start[2]] = rng.integers(0, 256, (k, 32), dtype=np.uint8)
    for lv in range(2, L + 1):
        mask = rng.integers(0, 256, (sizes[lv], 32), dtype=np.uint8)
        for _ in range(2 if lv == 2 else 3 if lv <= 4 else 4):
            mask &= rng.integers(0, 256, (sizes[lv], 32), dtype=np.uint8)
        desc[start[lv]:start[lv + 1]] = np.repeat(desc[start[lv - 1]:start[lv]], k, axis=0) ^ mask
    parent = np.concatenate([[-1], (np.arange(1, n) - 1) // k])
    child_start = np.concatenate([np.arange(n_inner + 1) * k, np.full(n - n_inner, n_inner * k)]).astype(np.int32)
    children = rng.permuted(np.arange(1, n, dtype=np.int32).reshape(n_inner, k), axis=1).reshape(-1)
    leaves = np.arange(n_inner, n)
    word_id = np.full(n, -1, np.int32)
    word_id[leaves] = rng.permutation(len(leaves))
    weight = np.zeros(n)
    weight[leaves] = rng.uniform(0.5, 9.0, len(leaves))
    weight[rng.choice(leaves, int(stop * len(leaves)), replace=False)] = 0.0
    depth = np.repeat(np.arange(L + 1), sizes).astype(np.int32)
    return dict(L=L, parent=parent, depth=depth, desc=desc, weight=weight, child_start=child_start, children=children, word_id=word_id,
                n_words=len(leaves), ties=[])


@functools.lru_cache(maxsize=None)
def vocabulary(name):
    """The tree TREES[name], or 'orbvoc' = orbvoc_tree(), built once per process."""
    return orbvoc_tree() if name == 'orbvoc' else random_tree(**TREES[name])


def near(voc, nodes, n, seed, max_flips=4):
    """n descriptors, each a node of `nodes` (drawn in turn) with 0..max_flips bits flipped: features that descend towards them."""
    rng = np.random.default_rng(seed)
    nodes = np.asarray(nodes)
    out = voc['desc'][nodes[np.arange(n) % len(nodes)]].copy()
    for i in range(n):
        out[i] = _flip(rng, out[i], int(rng.integers(0, max_flips + 1)))
    return out


def tie_targets(voc):
    """The child at position p of every planted tie: features near it meet the tie at its parent."""
    cs, ch = voc['child_start'], voc['children']
    return [int(ch[cs[node] + p]) for node, p, _ in voc['ties']]


def tie_hits(voc, feats):
    """Per planted tie (node, p, q): how many features descend through the child at p and through the one at q (equal descriptors, so
    the first-minimum rule sends every feature that reaches the tie to p)."""
    leaf, _ = descend(voc, feats, 0)
    cs, ch = voc['child_start'], voc['children']
    out = []
    for node, p, q in voc['ties']:
        cp, cq = ch[cs[node] + p], ch[cs[node] + q]
        d = voc['depth'][cp]
        up = ancestor(voc, leaf, d)
        deep = voc['depth'][leaf] >= d
        out.append((int(((up == cp) & deep).sum()), int(((up == cq) & deep).sum())))
    return out


def frames(voc, seed, n_near=600, n_random=300):
    """The test frames of a vocabulary: features near the planted ties and near random nodes, uniformly random descriptors, and both
    mixed in one frame."""
    rng = np.random.default_rng(seed)
    nodes = rng.choice(np.arange(1, len(voc['parent'])), 64)
    ties = near(voc, tie_targets(voc), n_near, seed + 1) if voc['ties'] else np.zeros((0, 32), np.uint8)
    nodes_f = near(voc, nodes, n_near, seed + 2)
    rand = rng.integers(0, 256, (n_random, 32)).astype(np.uint8)
    mixed = np.concatenate([ties, nodes_f, rand])[rng.permutation(len(ties) + n_near + n_random)]
    return [f for f in (ties, nodes_f, rand, mixed) if len(f)]


def one_word_frame(voc, n, seed):
    """n copies of one descriptor whose leaf is a kept word: one word receives all n features."""
    rng = np.random.default_rng(seed)
    while True:
        d = rng.integers(0, 256, (1, 32)).astype(np.uint8)
        if voc['weight'][descend(voc, d, 0)[0][0]] > 0:
            return np.repeat(d, n, axis=0)


def stopped_frame(voc, n, seed):
    """n features that all land on stopped words (weight 0): near the stopped leaves, kept where the descent ends on one."""
    stopped = np.flatnonzero((np.diff(voc['child_start']) == 0) & (voc['weight'] == 0))
    stopped = stopped[stopped > 0]
    cand = near(voc, stopped, 8 * n, seed, max_flips=1)
    cand = cand[voc['weight'][descend(voc, cand, 0)[0]] == 0]
    assert len(cand) >= n, 'too few features reach a stopped word'
    return cand[:n]


# ---------------------------------------------------------------------------------------------
# transform, restated
# ---------------------------------------------------------------------------------------------
def descend(voc, feats, levelsup, chunk=4096):
    """TemplatedVocabulary::transform(feature, word_id, weight, nid, levelsup) for every feature: at each level the child with the least
    Hamming distance, the first of equal ones in list order (np.argmin returns the first minimum).  Returns (leaf, nid) [N]: nid is the
    node reached at depth L - levelsup, 0 where the descent never passes that depth."""
    cs, ch, D = voc['child_start'].astype(np.int64), voc['children'].astype(np.int64), voc['desc']
    feats = np.asarray(feats, np.uint8).reshape(-1, 32)
    N = len(feats)
    leaf, nid = np.zeros(N, np.int64), np.zeros(N, np.int64)
    nid_level = voc['L'] - levelsup
    active, level = np.arange(N), 0
    while active.size:
        level += 1
        for s in range(0, active.size, chunk):
            act = active[s:s + chunk]
            cur = leaf[act]
            a, b = cs[cur], cs[cur + 1]
            pos = a[:, None] + np.arange((b - a).max())
            ok = pos < b[:, None]
            cid = ch[np.where(ok, pos, a[:, None])]
            dist = POPCOUNT[feats[act][:, None, :] ^ D[cid]].sum(-1, dtype=np.int32)
            dist[~ok] = 1 << 20
            leaf[act] = cid[np.arange(len(act)), dist.argmin(1)]
        if level == nid_level:
            nid[active] = leaf[active]
        active = active[cs[leaf[active] + 1] > cs[leaf[active]]]
    return leaf, nid


def fma(a, b, c):
    """a * b + c rounded once (math.fma arrives in Python 3.13): the exact rational rounded to the nearest double."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def transform(voc, feats, levelsup=4, weighting=0, norm=1):
    """TemplatedVocabulary::transform(features, BowVector, FeatureVector, levelsup).  Returns (word ids ascending, values, fv nodes,
    fv features) like oracle_lib.bow_transform.  weighting 0 TF_IDF, 1 TF, 2 IDF, 3 BINARY; norm 0 none, 1 L1, 2 L2."""
    leaf, nid = descend(voc, feats, levelsup)
    w = voc['weight'][leaf]
    wid = voc['word_id'][leaf]
    v = {}
    for i in range(len(leaf)):                   # feature order: the order std::map::operator+= sees the weights
        if w[i] > 0:
            key, x = int(wid[i]), float(w[i])
            if weighting in (0, 1):
                v[key] = v.get(key, 0.0) + x     # addWeight
            elif key not in v:
                v[key] = x                       # addIfNotExist
    words = sorted(v)
    vals = [v[key] for key in words]
    if weighting in (0, 1) and vals and norm == 0:     # the !must branch: divide by the number of words
        nd = float(len(vals))
        vals = [x / nd for x in vals]
    if norm:
        nrm = 0.0
        if norm == 1:
            for x in vals:
                nrm += abs(x)
        else:
            for x in vals:
                nrm = fma(x, x, nrm)             # one rounding per term, as the reference's build contracts it
            nrm = math.sqrt(nrm)
        if nrm > 0.0:
            vals = [x / nrm for x in vals]
    kept = np.flatnonzero(w > 0)
    order = np.lexsort((kept, nid[kept]))
    return (np.array(words, np.int32), np.array(vals, np.float64), nid[kept][order].astype(np.int32), kept[order].astype(np.int32))


def ancestor(voc, nodes, depth):
    """The ancestor of each node at `depth` (<= the node's depth), from the parent array."""
    a = np.asarray(nodes, np.int64).copy()
    for _ in range(int(voc['depth'][a].max(initial=0))):
        up = voc['depth'][a] > depth
        a[up] = voc['parent'][a[up]]
    return a
