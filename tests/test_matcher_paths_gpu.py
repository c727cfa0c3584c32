"""SearchByProjection's frame matcher (match_frame_kernel) at every launch shape Matcher::run can choose, against the CPU oracle.

Matcher::run makes four decisions from a call's shape: the cluster size C (1..8, the largest with batch x C <= 2 x SMs whose clusters
are all resident; the handle reports it through last_cluster_size()), the pass-1 split of the map points over C x 16 warps, whether
the descriptors are staged in shared memory (frame_smem_bytes(ks, ms, true) <= 100 KB), and how many CTAs fit on an SM.  Every case
here compares every frame's match, claimed and nmatches with the oracle byte for byte; the oracle's answer depends only on the frame,
so it is computed once per scene."""
import numpy as np
import pytest

import matcher_scenes as S
import oracle_lib as O

pytestmark = pytest.mark.gpu
TH = 15.0
FRAMES = tuple(range(5, 41, 3))          # twelve distinct 640x480 last-frame scenes, cycled to fill a batch
BATCHES = (1, 33, 34, 37, 38, 44, 45, 52, 53, 66, 67, 88, 89, 132, 133, 264)
SMEM_LIMIT = 227 * 1024 - 2048           # Matcher::run: the opt-in maximum minus the kernel's static shared memory


def frame_smem_bytes(ks, ms, desc):
    """matcher.cu's frame_smem_bytes: the dynamic shared memory of one CTA for ks keypoints and ms map points."""
    al = lambda v: (v + 15) & ~15
    b = al(4 * 64 * 48) + al(2 * (64 * 48 + 1)) + al(2 * ks) + 2 * al(4 * ks) + al(ks) + al(4 * ((ks + 31) // 32)) + al(4 * ks)
    b += 2 * al(2 * ms) + al(ms)
    return b + (al(32 * ks) if desc else 0)


def desc_in_smem(kcap, mcap):
    return frame_smem_bytes(kcap, mcap, True) <= 100 * 1024


# the largest kcap = mcap whose descriptors are still staged in shared memory, and the next one (read from global memory)
SMEM_EDGE = max(n for n in range(1000, 2000) if desc_in_smem(n, n))


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


_SCENES, _ORACLE = {}, {}


def scene(key):
    """('f', t): last_frame_scene(t); ('m', t, M): the first M map points of frames t-1..t-5 merged; ('nokp', t): frame t without
    keypoints; ('special', name): matcher_scenes.special_scene(name, 1)."""
    if key not in _SCENES:
        if key[0] == 'f':
            s = S.last_frame_scene(key[1])
        elif key[0] == 'm':
            s = S.last_frame_scene(key[1], prev=(1, 2, 3, 4, 5))
            assert len(s['last']['valid']) >= key[2]
            s = dict(s, last={k: v[:key[2]] for k, v in s['last'].items()})
        elif key[0] == 'nokp':
            s = S.last_frame_scene(key[1])
            s = dict(s, kps=s['kps'][:0], desc=s['desc'][:0])
        else:
            s = S.special_scene(key[1], 1)
        _SCENES[key] = s
    return _SCENES[key]


def oracle(key):
    if key not in _ORACLE:
        s = scene(key)
        om = np.full(len(s['kps']), -1, np.int32); oc = np.zeros(len(s['kps']), np.uint8)
        on = O.search_last_frame(s['kps'], s['desc'], s['bounds'], s['sf'], s['Tcw'], s['cam'], s['last'], TH, True, om, oc)
        _ORACLE[key] = (om, oc, on)
    return _ORACLE[key]


def pack(orb, keys, kcap, mcap):
    """The batch dict of search_last_frame_batch (numpy) for the scenes `keys`, one per stream, in [batch][kcap] / [batch][mcap] slabs."""
    B, s0 = len(keys), scene(keys[0])
    d = dict(batch=B, kcap=kcap, mcap=mcap, nlevels=8, bounds=tuple(float(b) for b in s0['bounds']), cam=[float(c) for c in s0['cam']],
             kps=np.zeros((B, kcap), orb.KP_DTYPE), desc=np.zeros((B, kcap, 32), np.uint8), nK=np.zeros(B, np.int32),
             scaleFactors=np.ascontiguousarray(s0['sf'], np.float32), nM=np.zeros(B, np.int32), valid=np.zeros((B, mcap), np.uint8),
             xyz=np.zeros((B, mcap, 3), np.float32), octave=np.zeros((B, mcap), np.int32), angle=np.zeros((B, mcap), np.float32),
             hasObs=np.zeros((B, mcap), np.uint8), mpDesc=np.zeros((B, mcap, 32), np.uint8), Tcw7=np.zeros((B, 7), np.float32))
    for b, key in enumerate(keys):
        s = scene(key)
        L = s['last']
        k, m = len(s['kps']), len(L['valid'])
        d['nK'][b], d['nM'][b] = k, m
        d['kps'][b, :k], d['desc'][b, :k] = s['kps'], s['desc']
        for src, dst in (('valid', 'valid'), ('xyz', 'xyz'), ('octave', 'octave'), ('angle', 'angle'), ('hasObs', 'hasObs'), ('descriptors', 'mpDesc')):
            d[dst][b, :m] = L[src]
        d['Tcw7'][b] = s['Tcw']
    return d


def run_host(m, d, match=None, claimed=None):
    B, K = d['batch'], d['kcap']
    match = np.full((B, K), -1, np.int32) if match is None else match.copy()
    claimed = np.zeros((B, K), np.uint8) if claimed is None else claimed.copy()
    nm = np.full(B, -7, np.int32)
    m.mbCheckOrientation = True
    m.search_last_frame_batch(d, TH, match, claimed, nm)
    return match, claimed, nm


def run_device(m, d, match=None, claimed=None):
    import torch
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype.fields else np.ascontiguousarray(a)).cuda()
    dd = {k: (dev(v) if isinstance(v, np.ndarray) else v) for k, v in d.items()}
    B, K = d['batch'], d['kcap']
    dm = dev(np.full((B, K), -1, np.int32) if match is None else match)
    dc = dev(np.zeros((B, K), np.uint8) if claimed is None else claimed)
    dn = torch.full((B,), -7, dtype=torch.int32, device='cuda')
    m.mbCheckOrientation = True
    st = torch.cuda.current_stream()
    m.search_last_frame_batch_device(dd, TH, dm, dc, dn, st.cuda_stream)
    st.synchronize()
    return dm.cpu().numpy(), dc.cpu().numpy(), dn.cpu().numpy()


def check(keys, out, what, expect=None):
    """Every stream equals its oracle answer (or expect[b] = (match, claimed, n)); the slab tail [K, kcap) is -1 / 0."""
    match, claimed, nm = out
    for b, key in enumerate(keys):
        om, oc, on = expect[b] if expect is not None else oracle(key)
        K = len(om)
        assert nm[b] == on, (what, b, key, int(nm[b]), on)
        assert match[b, :K].tobytes() == om.tobytes(), (what, b, key, int((match[b, :K] != om).sum()))
        assert claimed[b, :K].tobytes() == oc.tobytes(), (what, b, key)
        assert (match[b, K:] == -1).all() and (claimed[b, K:] == 0).all(), (what, b, key)


def cycle(B, base=FRAMES):
    return [('f', base[b % len(base)]) for b in range(B)]


def test_cluster_size_by_batch(orb, sms):
    """a. Host and device batch forms at batch sizes around every threshold 2 x SMs / C; the cluster size each one ran with."""
    m = orb.ORBmatcher(0.8, True, max_batch=max(BATCHES), max_keypoints=1100, max_mappoints=1100)
    sizes = {}
    for B in BATCHES:
        keys = cycle(B)
        d = pack(orb, keys, 1100, 1100)
        check(keys, run_host(m, d), ('host', B))
        c = m.last_cluster_size()
        assert m.last_launch_count() == 1
        check(keys, run_device(m, d), ('device', B))
        assert m.last_cluster_size() == c
        sizes[B] = c
    print('\nmatch_frame_kernel cluster size by batch (kcap = mcap = 1100, %d SMs): %s' % (sms, sizes))
    for B, c in sizes.items():
        assert 1 <= c <= 8 and B * c <= 2 * sms, (B, c)
    cs = [sizes[B] for B in BATCHES]
    assert all(a >= b for a, b in zip(cs, cs[1:])), sizes
    assert {1, 2, 8} <= set(cs) and len(set(cs) & {3, 4, 5, 6, 7}) >= 2, sizes


# b. (kcap, mcap) -> descriptors in shared memory?, CTAs per SM.  The frames have about 1,005 keypoints, so the smallest caps are
# 1100 rather than 1000.  SMEM_EDGE (1608) is the largest square cap whose descriptors fit the 100 KB budget; SMEM_EDGE + 1 reads them
# from global memory.  4000 / 8000 needs 116 KB without descriptors, more than half of an SM: one CTA per SM.
REGIMES = ((1100, 1100, True, 2), (SMEM_EDGE, SMEM_EDGE, True, 2), (SMEM_EDGE + 1, SMEM_EDGE + 1, False, 2), (1700, 1700, False, 2),
           (2048, 2048, False, 2), (4000, 8000, False, 1))


def test_shared_memory_regimes(orb, sms):
    B = 60
    keys = cycle(B)
    sizes = {}
    for kcap, mcap, smem, ctas in REGIMES:
        assert desc_in_smem(kcap, mcap) == smem
        sm = frame_smem_bytes(kcap, mcap, smem)
        assert sm <= SMEM_LIMIT and (sm > 113 * 1024) == (ctas == 1), (kcap, mcap, sm)
        m = orb.ORBmatcher(0.8, True, max_batch=B, max_keypoints=kcap, max_mappoints=mcap)
        d = pack(orb, keys, kcap, mcap)
        check(keys, run_host(m, d), ('host', kcap, mcap))
        sizes[(kcap, mcap)] = m.last_cluster_size()
        if ctas == 1 or not smem:
            check(keys, run_device(m, d), ('device', kcap, mcap))
        m.close()
    print('\nmatch_frame_kernel cluster size at batch %d by (kcap, mcap): %s' % (B, sizes))
    two = [sizes[(k, mm)] for k, mm, _, c in REGIMES if c == 2]
    assert len(set(two)) == 1 and sizes[(4000, 8000)] < two[0] and B * two[0] <= 2 * sms and B * sizes[(4000, 8000)] <= sms, sizes


@pytest.mark.parametrize('B', [8, 66, 133])
def test_pass1_tails(orb, sms, B):
    """c. Map-point counts on both sides of every multiple of the pass-1 stride (16 C warps) and of its 32-point groups (512 C), at the
    cluster size the batch runs with; a frame without keypoints next to one with exactly kcap."""
    bases = (11, 23, 35)
    kcap = max(len(scene(('f', t))['kps']) for t in bases)
    mcap = 4100
    m = orb.ORBmatcher(0.8, True, max_batch=B, max_keypoints=kcap, max_mappoints=mcap)
    probe = [('m', bases[b % 3], 4097) for b in range(B)]
    run_host(m, pack(orb, probe, kcap, mcap))
    C = m.last_cluster_size()
    Ms = (0, 1, 16 * C - 1, 16 * C, 16 * C + 1, 512 * C - 1, 512 * C, 512 * C + 1)
    keys = [('m', bases[b % 3], Ms[b % len(Ms)]) for b in range(B)]
    big = max(bases, key=lambda t: len(scene(('f', t))['kps']))
    keys[0] = ('nokp', bases[0])
    keys[1] = ('m', big, 700)                                   # nK == kcap
    assert len(scene(keys[1])['kps']) == kcap
    d = pack(orb, keys, kcap, mcap)
    check(keys, run_host(m, d), ('host', B, C))
    assert m.last_cluster_size() == C and B * C <= 2 * sms
    check(keys, run_device(m, d), ('device', B, C))
    print('\nbatch %d: cluster size %d, map-point counts %s' % (B, C, Ms))


def test_entry_claims_and_reset(orb):
    """d. With resetState = 0 the claims at entry are honoured; with resetState = 1 garbage in match / claimed is ignored and the slab
    tail [K, kcap) is cleared."""
    B, kcap, mcap = 7, 1100, 1100
    keys = cycle(B)
    m = orb.ORBmatcher(0.8, True, max_batch=B, max_keypoints=kcap, max_mappoints=mcap)
    d = pack(orb, keys, kcap, mcap)
    rng = np.random.default_rng(5)
    match = np.where(rng.random((B, kcap)) < 0.2, rng.integers(0, 900, (B, kcap)), -1).astype(np.int32)
    claimed = (rng.random((B, kcap)) < 0.5).astype(np.uint8)
    expect = []
    for b, key in enumerate(keys):
        s = scene(key)
        K = len(s['kps'])
        match[b, K:], claimed[b, K:] = -1, 0
        om, oc = match[b, :K].copy(), claimed[b, :K].copy()
        on = O.search_last_frame(s['kps'], s['desc'], s['bounds'], s['sf'], s['Tcw'], s['cam'], s['last'], TH, True, om, oc)
        expect.append((om, oc, on))
    check(keys, run_host(m, d, match, claimed), 'host, claims at entry', expect)
    check(keys, run_device(m, d, match, claimed), 'device, claims at entry', expect)
    junk_m = rng.integers(-5, 70000, (B, kcap)).astype(np.int32)
    junk_c = rng.integers(0, 256, (B, kcap)).astype(np.uint8)
    d['reset'] = 1
    check(keys, run_host(m, d, junk_m, junk_c), 'host, reset')
    check(keys, run_device(m, d, junk_m, junk_c), 'device, reset')


def test_alternating_shapes_on_one_handle(orb):
    """d. One handle alternates (batch, caps) A, B, A: every call equals the oracle and runs with the cluster size a fresh handle picks."""
    shapes = ((8, 1100, 1100), (66, 4000, 8000), (8, 1100, 1100), (66, 4000, 8000))
    fresh = {}
    for B, kcap, mcap in set(shapes):
        f = orb.ORBmatcher(0.8, True, max_batch=B, max_keypoints=kcap, max_mappoints=mcap)
        keys = cycle(B)
        check(keys, run_host(f, pack(orb, keys, kcap, mcap)), ('fresh', B))
        fresh[(B, kcap, mcap)] = f.last_cluster_size()
        f.close()
    m = orb.ORBmatcher(0.8, True, max_batch=66, max_keypoints=4000, max_mappoints=8000)
    for B, kcap, mcap in shapes:
        keys = cycle(B, FRAMES[::-1])
        check(keys, run_host(m, pack(orb, keys, kcap, mcap)), ('shared', B, kcap))
        assert m.last_cluster_size() == fresh[(B, kcap, mcap)], (B, kcap, mcap)
    assert fresh[(66, 4000, 8000)] < fresh[(8, 1100, 1100)]


def _local(orb, m, s, th):
    F = orb.Frame(s['kps'], s['desc'], s['bounds'], s['sf'])
    m.mfNNratio = 0.8
    n = m.SearchByProjection(F, s['pts'], th)
    om = np.full(len(s['kps']), -1, np.int32); oc = np.zeros(len(s['kps']), np.uint8)
    on = O.search_local_map(s['kps'], s['desc'], s['bounds'], s['sf'], s['pts'], th, 0.8, False, 50.0, om, oc)
    assert n == on and F.match.tobytes() == om.tobytes() and F.claimed.tobytes() == oc.tobytes(), (n, on, int((F.match != om).sum()))
    return n


def _last(orb, m, s):
    F = orb.Frame(s['kps'], s['desc'], s['bounds'], s['sf'])
    m.mbCheckOrientation = True
    n = m.SearchByProjection(F, s['last'], TH, True, Tcw=s['Tcw'], cam=s['cam'])
    om = np.full(len(s['kps']), -1, np.int32); oc = np.zeros(len(s['kps']), np.uint8)
    on = O.search_last_frame(s['kps'], s['desc'], s['bounds'], s['sf'], s['Tcw'], s['cam'], s['last'], TH, True, om, oc)
    assert n == on and F.match.tobytes() == om.tobytes() and F.claimed.tobytes() == oc.tobytes(), (n, on, int((F.match != om).sum()))
    return n


def test_local_map_single_frame_regimes(orb):
    """e. The single-frame local-map search sizes shared memory from the frame's own K and M: K ~ 2000 with 2500 points reads the
    descriptors from global memory (2 CTAs per SM), K ~ 4000 with 8192 points needs one CTA per SM, K ~ 1000 with 8192 points
    reads them from global memory too."""
    m = orb.ORBmatcher(0.8, True, max_batch=1, max_keypoints=4096, max_mappoints=8192)
    cases = ((S.local_map_scene(7, nf=2000, M=2500), False, 2), (S.local_map_scene(8, nf=4000, M=8192, dts=(-5, -4, -3, -2, -1, 1, 2, 3, 4, 5)), False, 1),
             (S.special_scene('big', 0), False, 2))
    for s, smem, ctas in cases:
        K, M = len(s['kps']), len(s['pts']['projX'])
        assert desc_in_smem(K, M) == smem and (frame_smem_bytes(K, M, smem) > 113 * 1024) == (ctas == 1), (K, M)
        for th in (1.0, 3.0):
            assert _local(orb, m, s, th) > 100
            assert m.last_launch_count() == 1 and m.last_cluster_size() == 8


@pytest.mark.parametrize('name', S.SPECIAL)
def test_special_scenes(orb, name):
    """f. Other geometries and bounds, keypoints on cell ties and outside the bounds, one crowded cell, claim staircases and 8192 map
    points: both single-frame searches, and the last-frame batch form with the scene in every stream."""
    m = orb.ORBmatcher(0.8, True, max_batch=3, max_keypoints=3100, max_mappoints=8192)
    s0 = S.special_scene(name, 0)
    _local(orb, m, s0, 1.0)
    _local(orb, m, s0, 3.0)
    _last(orb, m, scene(('special', name)))
    keys = [('special', name)] * 3
    s = scene(keys[0])
    d = pack(orb, keys, len(s['kps']), len(s['last']['valid']))
    check(keys, run_host(m, d), ('host', name))
    check(keys, run_device(m, d), ('device', name))


def test_capacity_refusal(orb):
    """g. A frame above the shared-memory limit, or more than 65535 map points, is refused on the host with ORB_ERR_CAPACITY before any
    launch: last_launch_count() is then 0, and the next call on the handle is still exact."""
    m = orb.ORBmatcher(0.8, True, max_batch=1, max_keypoints=14000, max_mappoints=70000)
    assert frame_smem_bytes(14000, 1100, False) > SMEM_LIMIT
    keys = [('f', 5)]
    good = pack(orb, keys, 1100, 1100)
    s = scene(keys[0])

    def refused(call):
        with pytest.raises(orb.OrbError) as ei:
            call()
        assert ei.value.code == orb.ORB_ERR_CAPACITY
        assert m.last_launch_count() == 0
        check(keys, run_host(m, good), 'after a refusal')
        assert m.last_launch_count() == 1

    check(keys, run_host(m, good), 'first')
    refused(lambda: run_host(m, pack(orb, keys, 14000, 1100)))
    refused(lambda: run_host(m, pack(orb, keys, 1100, 70000)))
    refused(lambda: run_device(m, pack(orb, keys, 14000, 1100)))
    reps = -(-14000 // len(s['kps']))
    wide = dict(s, kps=np.tile(s['kps'], reps)[:14000], desc=np.tile(s['desc'], (reps, 1))[:14000])
    refused(lambda: _last(orb, m, wide))
    reps = -(-70000 // len(s['last']['valid']))
    many = dict(s, last={k: np.concatenate([v] * reps)[:70000] for k, v in s['last'].items()})
    refused(lambda: _last(orb, m, many))
