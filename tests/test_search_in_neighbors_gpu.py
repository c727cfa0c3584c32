"""GPU tests of orbm_fuse_search_batch: every round of the lockstep SearchInNeighbors driver (tests/search_in_neighbors_lib.py) equals
orbm_fuse_search item by item, byte for byte, with empty items mixed in; the batched lockstep run equals the per-call GPU chain and the
oracle chain in final map state; one launch per call; the argument errors; the C++ mirror's digest equals the Python binding's."""
import os
import subprocess

import numpy as np
import pytest

import search_in_neighbors_lib as SN

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def g():
    return SN.globals_()


def _empty_items(items):
    """An item without points and one whose keyframe has no keypoints, shaped like the first real one."""
    it = items[0]
    no_pts = dict(it, **{k: it[k][:0] for k in ('state', 'xyz', 'normal', 'min_d', 'max_d', 'mp_desc')})
    no_kps = dict(it, kps=it['kps'][:0], desc=it['desc'][:0])
    return [no_pts, no_kps]


class CheckedBatch(SN.GpuBatchBackend):
    """Every batch call with two empty items mixed in, compared with orbm_fuse_search of each item."""
    def __init__(self, matcher, single):
        super().__init__(matcher)
        self.single, self.rounds = single, 0

    def fuse(self, items):
        if not items:
            return []
        mixed = [items[0]] + _empty_items(items) + items[1:]
        out = self.m.fuse_search_batch(mixed)
        assert self.m.last_launch_count() == 1
        for it, (bi, bd) in zip(mixed, out):
            sbi, sbd = self.single.FuseSearch(*[it[k] for k in SN.FUSE_KEYS], it['th'])
            assert bi.tobytes() == sbi.tobytes() and bd.tobytes() == sbd.tobytes()
        assert (out[2][0] == -1).all() and (out[2][1] == 256).all() and len(out[1][0]) == 0
        self.rounds += 1
        return [out[0]] + out[3:]


@pytest.mark.parametrize('B', [1, 7, 24])
def test_batch_equals_single_calls_every_round(orb, g, B):
    nt = [1 + (s * 5) % 6 for s in range(B)]
    if B > 1:
        nt[1] = 0
    jobs = SN.make_jobs(g, B, 10 + B, nt, no_points=(3,) if B > 3 else ())
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=2048, max_mappoints=64)
    single = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=2048, max_mappoints=64)
    be = CheckedBatch(m, single)
    SN.lockstep(be, jobs)
    assert be.rounds == max(nt) + 1


def test_lockstep_equals_gpu_chain_and_oracle(orb, g):
    args = (7, 4, [3, 0, 5, 2, 6, 1, 4], (5,), (2,))
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=2048, max_mappoints=64)
    runs = []
    for driver, be in ((SN.lockstep, SN.GpuBatchBackend(m)), (SN.sequential, SN.GpuChainBackend(m)), (SN.sequential, SN.OracleBackend())):
        jobs = SN.make_jobs(g, *args)
        ev = driver(be, jobs)
        runs.append(([j['map'].state() for j in jobs], ev, getattr(be, 'calls', None)))
    assert runs[0][0] == runs[1][0] == runs[2][0]
    assert runs[0][1] == runs[1][1] == runs[2][1] and runs[0][1]['replace_from_kf'] > 0 and runs[0][1]['add'] > 0
    assert runs[0][2] == max(args[2]) + 1 and runs[1][2] == sum(args[2]) + 6


def _item_array(orb, items):
    """The ctypes items of fuse_search_batch over copies of the items' arrays, for hand-made bad arguments."""
    keep = []
    arr = (orb._OrbmFuseItem * len(items))()
    for j, it in enumerate(items):
        k = [np.array(it['kps'], orb.KP_DTYPE), np.array(it['desc'], np.uint8), np.array(it['sf'], np.float32), np.array(it['isg'], np.float32)]
        p = [np.array(it[n], dt) for n, dt in (('state', np.uint8), ('xyz', np.float32), ('normal', np.float32), ('min_d', np.float32),
                                                            ('max_d', np.float32), ('mp_desc', np.uint8))]
        o = [np.zeros(len(p[0]), np.int32), np.zeros(len(p[0]), np.int32)]
        keep += k + p + o
        s = arr[j]
        s.KF = orb._OrbmFrame(len(k[0]), k[0].ctypes.data, k[1].ctypes.data, *it['bounds'], k[2].ctypes.data, len(k[2]))
        s.invLevelSigma2 = k[3].ctypes.data
        s.logScaleFactor = float(it['log_sf'])
        s.Tcw7[:] = [float(v) for v in it['Tcw']]; s.Ow[:] = [float(v) for v in it['Ow']]; s.cam[:] = [float(v) for v in it['cam']]
        s.th = 3.0
        s.pts = orb._OrbmFusePoints(len(p[0]), *[a.ctypes.data for a in p])
        s.bestIdx, s.bestDist = o[0].ctypes.data, o[1].ctypes.data
    return arr, keep


def test_bad_arguments_and_capacity(orb, g):
    jobs = SN.make_jobs(g, 2, 31, [1, 1])
    items = [j['map'].fuse_item(j['map'].kfs[j['targets'][0]], [int(p) for p in j['map'].kfs[j['cur']].mp if p >= 0]) for j in jobs]
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=2048, max_mappoints=64)
    L = orb.lib()
    m.fuse_search_batch(items)
    assert m.last_launch_count() == 1
    m.fuse_search_batch([_empty_items(items)[0]])
    assert m.last_launch_count() == 0                                  # nothing to search: no launch
    m.fuse_search_batch(items)

    def expect(code, edit, handle=m):
        arr, keep = _item_array(orb, items)
        edit(arr, keep)
        assert L.orbm_fuse_search_batch(handle._h, len(items), arr) == code, edit
        assert handle.last_launch_count() == (1 if handle is m else 0)     # rejected before any launch

    def octave(a, k): k[0]['octave'][5] = 8
    def neg_octave(a, k): k[12]['octave'][0] = -1
    def bounds(a, k): a[1].KF.maxX = a[1].KF.minX
    def null_state(a, k): a[0].pts.state = None
    def null_desc(a, k): a[1].pts.descriptors = None
    def null_out(a, k): a[1].bestDist = None
    def null_isg(a, k): a[0].invLevelSigma2 = None
    def null_kps(a, k): a[1].KF.keypoints = None
    def nlevels(a, k): a[0].KF.nlevels = 0
    for f in (octave, neg_octave, bounds, null_state, null_desc, null_out, null_isg, null_kps, nlevels):
        expect(orb.ORB_ERR_ARG, f)
    assert L.orbm_fuse_search_batch(m._h, -1, None) == orb.ORB_ERR_ARG
    narrow = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=500, max_mappoints=64)
    expect(orb.ORB_ERR_CAPACITY, lambda a, k: None, narrow)
    # a keyframe whose grid does not fit in shared memory even without its descriptors
    rng = np.random.default_rng(0)
    K = 16000
    kps = np.zeros(K, orb.KP_DTYPE)
    kps['x'], kps['y'], kps['octave'] = rng.uniform(0, 640, K), rng.uniform(0, 480, K), rng.integers(0, 8, K)
    big = dict(items[0], kps=kps, desc=rng.integers(0, 256, (K, 32)).astype(np.uint8))
    wide = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=K, max_mappoints=64)
    with pytest.raises(orb.OrbError) as ei:
        wide.fuse_search_batch([items[1], big])
    assert ei.value.code == orb.ORB_ERR_CAPACITY and wide.last_launch_count() == 0
    with pytest.raises(orb.OrbError) as ei:
        wide.FuseSearch(*[big[k] for k in SN.FUSE_KEYS], 3.0)
    assert ei.value.code == orb.ORB_ERR_CAPACITY


def _digest(out):
    h = 14695981039346656037
    for bi, bd in out:
        for b in bi.tobytes() + bd.tobytes():
            h = ((h ^ b) * 1099511628211) & 0xFFFFFFFFFFFFFFFF
    return h


def test_cpp_fuse_batch_equals_python(orb, g, tmp_path):
    """ORBmatcher::FuseBatch (include/orb_b200/orb_slam3.hpp) from a g++-built caller: the first lockstep round of five keyframes and
    an empty item give the Python binding's digest."""
    jobs = SN.make_jobs(g, 5, 41, [2, 3, 1, 2, 4])
    items = [j['map'].fuse_item(j['map'].kfs[j['targets'][0]], [int(p) for p in j['map'].kfs[j['cur']].mp if p >= 0]) for j in jobs]
    items.insert(2, _empty_items(items)[0])
    lines = [str(len(items))]
    for j, it in enumerate(items):
        vals = [len(it['kps']), len(it['state']), len(it['sf'])] + [repr(float(v)) for v in it['bounds']] + \
               [repr(float(v)) for v in [it['log_sf'], it['th']] + list(it['Tcw']) + list(it['Ow']) + list(it['cam'])]
        lines.append(' '.join(str(v) for v in vals))
        for k, dt in (('kps', orb.KP_DTYPE), ('desc', np.uint8), ('sf', np.float32), ('isg', np.float32), ('state', np.uint8), ('xyz', np.float32),
                      ('normal', np.float32), ('min_d', np.float32), ('max_d', np.float32), ('mp_desc', np.uint8)):
            (tmp_path / ('item%d_%s.raw' % (j, k))).write_bytes(np.ascontiguousarray(it[k], dt).tobytes())
    (tmp_path / 'dims.txt').write_text('\n'.join(lines) + '\n')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, 'orb_slam3_modified_b200')
    exe = tmp_path / 'search_in_neighbors_example'
    subprocess.check_call(['g++', '-std=c++14', '-O2', '-Wall', '-I', os.path.join(root, 'include'), os.path.join(root, 'tests', 'search_in_neighbors_example.cpp'),
                           '-o', str(exe), '-L', lib, '-l:liborb_b200.so', '-Wl,-rpath,' + lib, '-lpthread'])
    out = dict(l.split() for l in subprocess.check_output([str(exe), str(tmp_path)]).decode().splitlines())
    m = orb.ORBmatcher(0.6, True, max_batch=1, max_keypoints=2048, max_mappoints=64)
    res = m.fuse_search_batch(items)
    assert out['digest'] == '%016x' % _digest(res)
    assert int(out['fused']) == sum(int((bd <= 50).sum()) for _, bd in res) > 100
    assert out['launches'] == '1'
