"""Seeded matcher scenarios built from real extractor output of consecutive synthetic frames, and variants with keypoints and map
points placed on purpose: image borders, grid-cell ties, one crowded cell, equal-distance candidates and claim staircases."""
import numpy as np

import oracle_lib as O
from orb_slam3_modified_b200 import synth

_CACHE = {}
UNDISTORTED = (-12.613, -9.271, 651.384, 487.906)   # bounds as Frame::ComputeImageBounds gives them for a distorted 640x480 camera


def extract(t, seed=0, w=640, h=480, nf=1000):
    key = (t, seed, w, h, nf)
    if key not in _CACHE:
        _CACHE[key] = O.OracleExtractor(nf, 1.2, 8, 20, 7)(synth.frame(t, w, h, seed), (0, 1000))[1:]
    return _CACHE[key]


def last_frame_scene(t, seed=0, rng=None, pose_noise=0.004, frac_invalid=0.1, frac_noobs=0.1, w=640, h=480, nf=1000, bounds=None, prev=(1,)):
    """Current frame = frame t, last frame = the keypoints of frames t - d (d in prev) as map points on the plane z=0."""
    rng = rng or np.random.default_rng(t * 31 + seed)
    kps, desc = extract(t, seed, w, h, nf)
    xyz, octv, ang, ld = [], [], [], []
    for d in prev:
        lk, dd = extract(t - d, seed, w, h, nf)
        xyz.append(synth.backproject(np.stack([lk['x'], lk['y']], 1), t - d, seed, w, h).astype(np.float32))
        octv.append(lk['octave']); ang.append(lk['angle']); ld.append(dd)
    xyz, octv, ang, ld = (np.concatenate(a) for a in (xyz, octv, ang, ld))
    M = len(xyz)
    last = dict(valid=(rng.random(M) > frac_invalid).astype(np.uint8), xyz=xyz, octave=octv.astype(np.int32),
                angle=ang.astype(np.float32), hasObs=(rng.random(M) > frac_noobs).astype(np.uint8), descriptors=ld)
    T = synth.pose(t, seed)
    T[4:] += rng.normal(0, pose_noise, 3)
    q = T[:4] + rng.normal(0, pose_noise * 0.2, 4)
    T[:4] = q / np.linalg.norm(q)
    sf = O.OracleExtractor().tables()['scale']
    return dict(kps=kps, desc=desc, bounds=bounds or (0.0, 0.0, float(w), float(h)), sf=sf, Tcw=T.astype(np.float32), cam=synth.camera(w, h), last=last)


def local_map_scene(t, seed=0, rng=None, M=2500, w=640, h=480, nf=1000, bounds=None, dts=(-3, -2, -1, 1, 2)):
    """Local map = keypoints of several neighbouring frames projected into frame t (fields as Frame::isInFrustum writes them)."""
    rng = rng or np.random.default_rng(t * 17 + seed + 5)
    bounds = bounds or (0.0, 0.0, float(w), float(h))
    kps, desc = extract(t, seed, w, h, nf)
    T = synth.pose(t, seed)
    w_, x, y, z = T[:4]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w_), 2 * (x * z + y * w_)], [2 * (x * y + z * w_), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w_)],
                  [2 * (x * z - y * w_), 2 * (y * z + x * w_), 1 - 2 * (x * x + y * y)]])
    cam = synth.camera(w, h)
    px, py, lv, dd, dep = [], [], [], [], []
    for dt in dts:
        lk, ld = extract(t + dt, seed, w, h, nf)
        P = synth.backproject(np.stack([lk['x'], lk['y']], 1), t + dt, seed, w, h)
        Pc = (R @ P.T).T + T[4:]
        u = cam[0] * Pc[:, 0] / Pc[:, 2] + cam[2] + rng.normal(0, 1.5, len(lk))
        v = cam[1] * Pc[:, 1] / Pc[:, 2] + cam[3] + rng.normal(0, 1.5, len(lk))
        px.append(u); py.append(v); lv.append(np.clip(lk['octave'] + rng.integers(-1, 2, len(lk)), 0, 7)); dd.append(ld); dep.append(Pc[:, 2])
    px, py, lv, dd, dep = (np.concatenate(a) for a in (px, py, lv, dd, dep))
    sel = rng.permutation(len(px))[:M]
    px, py, lv, dd, dep = px[sel], py[sel], lv[sel], dd[sel], dep[sel]
    inb = (px >= bounds[0]) & (px <= bounds[2]) & (py >= bounds[1]) & (py <= bounds[3])
    n = len(px)
    pts = dict(inView=(inb & (rng.random(n) > 0.05)).astype(np.uint8), bad=(rng.random(n) < 0.03).astype(np.uint8), depth=dep.astype(np.float32),
               projX=px.astype(np.float32), projY=py.astype(np.float32), level=lv.astype(np.int32),
               viewCos=np.where(rng.random(n) < 0.5, 0.9995, 0.9).astype(np.float32), hasObs=(rng.random(n) > 0.1).astype(np.uint8), descriptors=dd)
    sf = O.OracleExtractor().tables()['scale']
    return dict(kps=kps, desc=desc, bounds=bounds, sf=sf, pts=pts)


# ---- keypoints and map points placed on purpose ----

def cell_coord(bounds, c, axis):
    """The float32 image coordinate p nearest to minX + c / gridWInv (axis 0; y for axis 1) for which Frame::PosInGrid's
    (p - min) * inv evaluates to exactly c in float32, when one exists within 64 ulps; else the nearest one."""
    lo = np.float32(bounds[axis])
    inv = np.float32(64 if axis == 0 else 48) / (np.float32(bounds[2 + axis]) - lo)
    p = np.float32(lo + np.float32(c) / inv)
    up = down = p
    for _ in range(64):
        for q in (up, down):
            if np.float32(np.float32(q - lo) * inv) == np.float32(c):
                return q
        up, down = np.nextafter(up, np.float32(np.inf)), np.nextafter(down, np.float32(-np.inf))
    return p


def _flip(d, rng, nbits):
    d = d.copy()
    for bit in rng.choice(256, nbits, replace=False):
        d[bit >> 3] ^= np.uint8(1 << (bit & 7))
    return d


def _world(s, u, v, z=3.0):
    """World point that scene s's (noisy) Tcw projects to (u, v) at depth z, for the last-frame search."""
    qw, qx, qy, qz = (float(a) for a in s['Tcw'][:4])
    R = np.array([[1 - 2 * (qy * qy + qz * qz), 2 * (qx * qy - qz * qw), 2 * (qx * qz + qy * qw)], [2 * (qx * qy + qz * qw), 1 - 2 * (qx * qx + qz * qz), 2 * (qy * qz - qx * qw)],
                  [2 * (qx * qz - qy * qw), 2 * (qy * qz + qx * qw), 1 - 2 * (qx * qx + qy * qy)]])
    fx, fy, cx, cy = (float(c) for c in s['cam'])
    Pc = np.array([(u - cx) / fx * z, (v - cy) / fy * z, z])
    return (R.T @ (Pc - s['Tcw'][4:].astype(np.float64))).astype(np.float32)


def _plant(s, mode, rng, u, v, desc, level, angle, hasObs=None, shuffle=True):
    """Appends map points whose queries are centred on (u, v) to a copy of scene s: mode 0 = local map (projX / projY are exactly u, v),
    1 = last frame (xyz projects to within a few 1e-4 px of u, v).  shuffle: spread the planted points over the map-point order."""
    n = len(u)
    hasObs = np.ones(n, np.uint8) if hasObs is None else hasObs
    s = dict(s)
    if mode == 0:
        p = s['pts']
        add = dict(inView=np.ones(n, np.uint8), bad=np.zeros(n, np.uint8), depth=np.full(n, 3.0, np.float32), projX=np.asarray(u, np.float32),
                   projY=np.asarray(v, np.float32), level=np.asarray(level, np.int32), viewCos=np.where(rng.random(n) < 0.5, 0.9995, 0.9).astype(np.float32),
                   hasObs=hasObs, descriptors=np.asarray(desc, np.uint8))
        key = 'pts'
    else:
        p = s['last']
        add = dict(valid=np.ones(n, np.uint8), xyz=np.array([_world(s, a, b) for a, b in zip(u, v)], np.float32).reshape(n, 3),
                   octave=np.asarray(level, np.int32), angle=np.asarray(angle, np.float32), hasObs=hasObs, descriptors=np.asarray(desc, np.uint8))
        key = 'last'
    merged = {k: np.concatenate([p[k], add[k]]) for k in p}
    if shuffle:
        perm = rng.permutation(len(merged[next(iter(merged))]))
        merged = {k: v_[perm] for k, v_ in merged.items()}
    s[key] = merged
    return s


def _with_kps(s, kps, desc):
    s = dict(s)
    s['kps'], s['desc'] = kps, desc
    return s


def edges_scene(base, mode, seed=0):
    """Keypoints moved just outside the image bounds, on both sides of the -0.5 cell tie and of the 63.5 / 47.5 ties, and onto k + 0.5
    ties; map points searched next to them, and map points whose queries sit exactly on (maxX, y), (x, maxY) and (maxX, maxY)."""
    rng = np.random.default_rng(seed + 101)
    kps, desc = base['kps'].copy(), base['desc'].copy()
    b = base['bounds']
    offs = (-0.6, -0.51, -0.5, -0.49, -0.2, 0.5, 62.5, 63.49, 63.5, 63.51, 64.2)
    sel = rng.choice(len(kps), 240, replace=False)
    for j, i in enumerate(sel):
        axis = j % 2
        c = offs[(j // 2) % len(offs)]
        c = c if axis == 0 else {62.5: 46.5, 63.49: 47.49, 63.5: 47.5, 63.51: 47.51, 64.2: 48.2}.get(c, c)
        kps['xy'[axis]][i] = cell_coord(b, c, axis)
    s = _with_kps(base, kps, desc)
    u = np.clip(kps['x'][sel] + rng.uniform(-1, 1, len(sel)), b[0], b[2]).astype(np.float32)
    v = np.clip(kps['y'][sel] + rng.uniform(-1, 1, len(sel)), b[1], b[3]).astype(np.float32)
    d = np.array([_flip(desc[i], rng, 6) for i in sel])
    lvl = kps['octave'][sel]
    # queries exactly on the right / bottom bounds, aimed at the keypoints nearest to them
    near = np.argsort(np.minimum(b[2] - kps['x'], b[3] - kps['y']))[:60]
    ue = np.where(np.arange(60) % 3 == 1, kps['x'][near], np.float32(b[2])).astype(np.float32)
    ve = np.where(np.arange(60) % 3 == 0, kps['y'][near], np.float32(b[3])).astype(np.float32)
    u, v = np.concatenate([u, ue]), np.concatenate([v, ve])
    d = np.concatenate([d, [_flip(desc[i], rng, 4) for i in near]])
    lvl = np.concatenate([lvl, kps['octave'][near]])
    return _plant(s, mode, rng, u, v, d, lvl, kps['angle'][np.concatenate([sel, near])])


def ties_scene(base, mode, seed=0):
    """Pairs of keypoints with one descriptor: A exactly on a cell tie k + 0.5 (cell k + 1 under round-half-away-from-zero, cell k
    under round-half-to-even when k is even), B in cell k with a higher index, and a map point equally far from both.  Only the
    enumeration order of Frame::GetFeaturesInArea decides which of them wins.  In the local-map search A and B sit on different
    levels so that the ratio test lets the equal pair through."""
    rng = np.random.default_rng(seed + 202)
    kps, desc = base['kps'].copy(), base['desc'].copy()
    b = base['bounds']
    idx = rng.choice(len(kps), 2 * 120, replace=False).reshape(120, 2)
    idx.sort(1)
    u, v, d, lvl, ang = [], [], [], [], []
    for g, (a, bb) in enumerate(idx):
        axis = g % 2
        k = 2 * int(rng.integers(1, 30 if axis == 0 else 22))       # even k: the two roundings disagree
        other = rng.uniform(30, (b[3] - b[1] if axis == 0 else b[2] - b[0]) - 30) + (b[1] if axis == 0 else b[0])
        tie = cell_coord(b, k + 0.5, axis)
        step = np.float32((b[2 + axis] - b[axis]) / (64 if axis == 0 else 48))
        xa, xb = tie, np.float32(tie - np.float32(0.3) * step)
        for i, p in ((a, xa), (bb, xb)):
            kps['xy'[axis]][i] = p
            kps['yx'[axis]][i] = np.float32(other)
        D = desc[a].copy()
        desc[bb] = D
        kps['octave'][a] = 1
        kps['octave'][bb] = 1 if mode == 1 else 0
        kps['angle'][bb] = kps['angle'][a]
        c = np.float32((float(xa) + float(xb)) / 2 + rng.uniform(-0.5, 0.5))
        u.append(c if axis == 0 else np.float32(other)); v.append(np.float32(other) if axis == 0 else c)
        d.append(_flip(D, rng, 5)); lvl.append(1); ang.append(kps['angle'][a])
    return _plant(_with_kps(base, kps, desc), mode, rng, u, v, d, lvl, ang)


def crowd_scene(base, mode, seed=0, n=420):
    """n keypoints moved into one grid cell (distinct positions), and map points aimed at most of them."""
    rng = np.random.default_rng(seed + 303)
    kps, desc = base['kps'].copy(), base['desc'].copy()
    b = base['bounds']
    cx, cy = cell_coord(b, 30, 0), cell_coord(b, 20, 1)
    wx, wy = (b[2] - b[0]) / 64, (b[3] - b[1]) / 48
    sel = rng.choice(len(kps), n, replace=False)
    kps['x'][sel] = (cx + rng.uniform(-0.45, 0.45, n) * wx).astype(np.float32)
    kps['y'][sel] = (cy + rng.uniform(-0.45, 0.45, n) * wy).astype(np.float32)
    tgt = sel[rng.permutation(n)[:300]]
    u = (kps['x'][tgt] + rng.uniform(-1, 1, 300)).astype(np.float32)
    v = (kps['y'][tgt] + rng.uniform(-1, 1, 300)).astype(np.float32)
    d = np.array([_flip(desc[i], rng, int(rng.integers(0, 30))) for i in tgt])
    return _plant(_with_kps(base, kps, desc), mode, rng, u, v, d, kps['octave'][tgt], kps['angle'][tgt])


def stairs_scene(base, mode, seed=0, clusters=10, steps=28):
    """Claim staircases: in each cluster, keypoints k_0..k_n sit within 3 px of one another with descriptors B ^ e_j (e_j: byte j set),
    and map point i (all with observations) is 4 bits from k_{i-1} and 12 from k_i (20 from the rest).  Map point i then takes k_i
    only once i - 1 has taken k_{i-1}, so the fixed-point pass needs a sweep per step.  In every second cluster each map point is
    repeated four times in a row, so later copies find all four pass-1 candidates taken and go to the rescan queue."""
    rng = np.random.default_rng(seed + 404)
    kps, desc = base['kps'].copy(), base['desc'].copy()
    b = base['bounds']
    sel = rng.choice(len(kps), clusters * steps, replace=False).reshape(clusters, steps)
    u, v, d, lvl, ang = [], [], [], [], []
    for c in range(clusters):
        x0 = np.float32(b[0] + (c + 1) * (b[2] - b[0]) / (clusters + 1))
        y0 = np.float32(b[1] + (0.3 + 0.4 * (c % 2)) * (b[3] - b[1]))
        B = rng.integers(0, 256, 32).astype(np.uint8)
        for j, i in enumerate(sel[c]):
            kps['x'][i] = x0 + np.float32(j % 6 - 2.5)
            kps['y'][i] = y0 + np.float32(j // 6 - 2.0)
            kps['octave'][i] = 0; kps['angle'][i] = np.float32(10.0)
            e = np.zeros(32, np.uint8); e[j] = 0xFF
            desc[i] = B ^ e
        rep = 4 if c % 2 else 1
        for j in range(steps):
            x = np.zeros(32, np.uint8)
            x[j] = 0x0F                                   # h_j: half of e_j
            if j:
                x[j - 1] = 0xFF                           # e_{j-1}
            for _ in range(rep):
                u.append(x0 + np.float32(rng.uniform(-0.4, 0.4))); v.append(y0 + np.float32(rng.uniform(-0.4, 0.4)))
                d.append(B ^ x); lvl.append(0); ang.append(10.0)
    s = _plant(_with_kps(base, kps, desc), mode, rng, u, v, d, lvl, ang, shuffle=False)
    return s


PLACED = dict(edges=edges_scene, ties=ties_scene, crowd=crowd_scene, stairs=stairs_scene)


def special_scene(name, mode):
    """The named scene for the local-map (mode 0) or last-frame (mode 1) search: geometries 'kitti' (1241x376, 2000 features), 'hd'
    (1280x720, 3000 features), 'undistorted' (640x480 with UNDISTORTED bounds), the placed scenes of PLACED (edges on UNDISTORTED
    bounds, the others on (0, 0, 640, 480)), and 'big' (8192 map points merged from neighbouring frames)."""
    key = ('special', name, mode)
    if key in _CACHE:
        return _CACHE[key]
    geo = dict(kitti=dict(w=1241, h=376, nf=2000), hd=dict(w=1280, h=720, nf=3000), undistorted=dict(bounds=UNDISTORTED), edges=dict(bounds=UNDISTORTED))
    kw = geo.get(name, {})
    t = 5 + sorted(['kitti', 'hd', 'undistorted', 'big'] + list(PLACED)).index(name)
    if name == 'big':
        s = local_map_scene(t, M=8192, dts=(-5, -4, -3, -2, -1, 1, 2, 3, 4, 5)) if mode == 0 else last_frame_scene(t, prev=tuple(range(1, 10)))
        if mode == 1:
            s['last'] = {k: v[:8192] for k, v in s['last'].items()}
    else:
        s = local_map_scene(t, **kw) if mode == 0 else last_frame_scene(t, **kw)
        if name in PLACED:
            s = PLACED[name](s, mode, seed=t)
    _CACHE[key] = s
    return s


SPECIAL = ('kitti', 'hd', 'undistorted', 'edges', 'ties', 'crowd', 'stairs', 'big')


def pos_in_grid(p, lo, inv):
    """Frame::PosInGrid's cell: C `round` of (p - lo) * inv evaluated in float32, which rounds halves away from zero (np.round would
    round them to even, and the exact ties k + 0.5 are common: level-0 keypoints have integer coordinates)."""
    a = (np.float32(p) - np.float32(lo)) * np.float32(inv)
    a = np.asarray(a, np.float32).astype(np.float64)
    return np.trunc(a + np.copysign(0.5, a)).astype(int)


class Cands:
    """Frame::GetFeaturesInArea without grid lists: every keypoint is tested (cell by pos_in_grid, cell range of the query by
    floor / ceil, level filter, window test) and the result is ordered by (cell x, cell y, keypoint index), the order the reference's
    walk over its cell lists produces (src/Frame.cc:657-723)."""
    def __init__(self, kps, bounds):
        self.k = kps
        self.minX, self.minY, maxX, maxY = (np.float32(b) for b in bounds)
        self.wi = np.float32(64) / (maxX - self.minX)
        self.hi = np.float32(48) / (maxY - self.minY)
        self.cx = pos_in_grid(kps['x'], self.minX, self.wi)
        self.cy = pos_in_grid(kps['y'], self.minY, self.hi)
        self.order = np.lexsort((np.arange(len(kps)), self.cy, self.cx))
        self.ingrid = (self.cx >= 0) & (self.cx < 64) & (self.cy >= 0) & (self.cy < 48)

    def query(self, x, y, r, lo, hi):
        x, y, r = np.float32(x), np.float32(y), np.float32(r)
        x0 = max(0, int(np.floor((x - self.minX - r) * self.wi)))
        x1 = min(63, int(np.ceil((x - self.minX + r) * self.wi)))
        y0 = max(0, int(np.floor((y - self.minY - r) * self.hi)))
        y1 = min(47, int(np.ceil((y - self.minY + r) * self.hi)))
        if x0 >= 64 or x1 < 0 or y0 >= 48 or y1 < 0:
            return []
        k = self.k
        ok = self.ingrid & (self.cx >= x0) & (self.cx <= x1) & (self.cy >= y0) & (self.cy <= y1)
        if lo > 0 or hi >= 0:
            ok &= k['octave'] >= lo
            if hi >= 0:
                ok &= k['octave'] <= hi
        ok &= (np.abs(k['x'] - x) < r) & (np.abs(k['y'] - y) < r)
        return [i for i in self.order if ok[i]]
