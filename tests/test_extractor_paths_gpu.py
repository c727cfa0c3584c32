"""GPU parity of the extractor paths the host picks from the caller's layout, the image size, the scale factor and the thresholds: every
level plane, blurred plane, FAST candidate list, monoIndex, keypoint and descriptor against the CPU oracle, frame by frame.

- device layouts whose level 0 is read in place by TMA (16-byte aligned base, pitch and frame stride) or copied first (anything else),
  with the copy visible in the launch count (nlevels + 4 kernels without it, nlevels + 5 with it);
- one handle alternating layouts, and one handle reconfigured for other image sizes (and refusing bad ones) between calls;
- the bilinear branch of pyr_resize_kernel (a level that is not an exact 2x decimation and whose source box is wider than TMA allows);
- FAST thresholds other than 20 / 7, a 4095-px wide image, a single level, lapping areas inside the image;
- the host form's per-frame upload and copy-out branches and both forms' capacity overflow;
- the device form of ComputeStereoMatches on planes read in place and copied."""
import ctypes as C

import numpy as np
import pytest

import oracle_lib as O
from orb_slam3_modified_b200 import synth
from test_extractor_gpu import _check_frame

pytestmark = pytest.mark.gpu

LAP = (0, 1000)
SENTINEL = 0xAB


@pytest.fixture(scope='module')
def orb():
    import orb_slam3_modified_b200 as m
    m.lib()
    return m


@pytest.fixture(scope='module')
def torch():
    import torch as t
    return t


def _frames(B, w, h, t0=0):
    return np.stack([synth.frame(t0 + 7 * b, w, h, seed=b % 3) for b in range(B)])


def _on_device(torch, frames, layout):
    """frames [B, h, w] as a CUDA view of the given layout: 'packed' (contiguous), 'crop' (big[:, 3:3+h, 5:5+w] of a buffer 60 px
    wider: unaligned base and pitch) or 'padded' (pitch a multiple of 16 other than w, 3 padding rows between frames)."""
    B, h, w = frames.shape
    src = torch.from_numpy(frames)
    if layout == 'packed':
        return src.cuda()
    if layout == 'crop':
        big = torch.zeros((B, h + 10, w + 60), dtype=torch.uint8)
        big[:, 3:3 + h, 5:5 + w] = src
        return big.cuda()[:, 3:3 + h, 5:5 + w]
    assert layout == 'padded'
    buf = torch.zeros((B, h + 3, (w + 15) // 16 * 16 + 16), dtype=torch.uint8)
    buf[:, :h, :w] = src
    return buf.cuda()[:, :h, :w]


def _reads_in_place(d):
    return d.data_ptr() % 16 == 0 and d.stride(1) % 16 == 0 and d.stride(0) % 16 == 0


def _extract_device(orb, torch, ex, d_images, lap=LAP, cap=None):
    """extract_batch_device into slabs prefilled with SENTINEL bytes; returns (n, mono, kps [B, cap], desc [B, cap, 32]) on the host."""
    B = d_images.shape[0]
    cap = cap or ex.max_keypoints
    d_kps = torch.full((B, cap, 28), SENTINEL, dtype=torch.uint8, device='cuda')
    d_desc = torch.full((B, cap, 32), SENTINEL, dtype=torch.uint8, device='cuda')
    d_n = torch.zeros(B, dtype=torch.int32, device='cuda')
    d_mono = torch.zeros(B, dtype=torch.int32, device='cuda')
    ex.extract_batch_device(d_images, d_kps, d_desc, d_n, d_mono, lap)
    torch.cuda.synchronize()
    return (d_n.cpu().numpy(), d_mono.cpu().numpy(), d_kps.cpu().numpy().view(orb.KP_DTYPE).reshape(B, cap), d_desc.cpu().numpy())


def _results(n, mono, kps, desc):
    return [(int(mono[f]), kps[f, :n[f]], desc[f, :n[f]]) for f in range(len(n))]


def _check_all(ex, oe, frames, results, lap, tag):
    for f in range(len(frames)):
        _check_frame(ex, f, results[f], oe, oe(frames[f], lap), '%s frame %d' % (tag, f))


def _check_device(orb, torch, ex, oe, frames, layout, lap=LAP, tag=''):
    d = _on_device(torch, frames, layout)
    n, mono, kps, desc = _extract_device(orb, torch, ex, d, lap)
    _check_all(ex, oe, frames, _results(n, mono, kps, desc), lap, '%s %s' % (tag, layout))
    for f in range(len(frames)):      # the level-0 tap of a device call shows the frames that call read
        assert np.array_equal(ex.level(0, f), frames[f]), (tag, layout, 'level 0 tap', f)
    assert ex.last_launch_count() == ex.nlevels + (4 if _reads_in_place(d) else 5), (tag, layout, ex.last_launch_count())
    return d


def _host_call(orb, ex, buf, B, rows, cols, step, frame_stride, cap, lap=LAP):
    """orbx_extract_batch on a raw host buffer (step / frame_stride in bytes) into sentinel-filled slabs of capacity `cap`."""
    kps = np.full((B, cap, 28), SENTINEL, np.uint8)
    desc = np.full((B, cap, 32), SENTINEL, np.uint8)
    n = np.zeros(B, np.int32)
    mono = np.zeros(B, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = orb.lib().orbx_extract_batch(ex._h, p(buf), B, rows, cols, step, frame_stride, lap[0], lap[1], p(kps), p(desc), cap, p(n), p(mono))
    return rc, n, mono, kps.view(orb.KP_DTYPE).reshape(B, cap), desc


# ---------------------------------------------------------------------------------------------------------------------------------
# device layouts
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('layout,w,h,B,max_batch', [('packed', 640, 480, 3, 3), ('crop', 640, 480, 3, 3), ('packed', 1241, 376, 3, 3),
                                                    ('padded', 640, 480, 3, 3), ('packed', 640, 480, 1, 4), ('crop', 640, 480, 2, 4)])
def test_device_layouts(orb, torch, layout, w, h, B, max_batch):
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, w, h, max_batch)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    d = _check_device(orb, torch, ex, oe, _frames(B, w, h, t0=B), layout, tag='%dx%d B=%d' % (w, h, B))
    assert _reads_in_place(d) == (layout == 'padded' or (layout == 'packed' and w % 16 == 0))


def test_one_handle_alternating_layouts(orb, torch):
    """Level 0's TMA descriptors are built per call from the caller's frames: a descriptor left over from the previous call would read
    that call's frames."""
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 3)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    for k, layout in enumerate(('packed', 'crop', 'packed')):
        _check_device(orb, torch, ex, oe, _frames(3, 640, 480, t0=40 * k + 1), layout, tag='call %d' % k)


def test_size_changes_on_one_handle(orb, torch):
    """One handle sized for 1280x720 runs smaller and larger images in turn through both forms, refuses sizes it cannot take and then
    runs a valid size again: the cell / block tables, the resize tables and every TMA descriptor are rebuilt on each change."""
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 1280, 720, 2)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    steps = [(1280, 720, 'host'), (640, 480, 'device'), (517, 389, 'host'), (1280, 720, 'device'), (640, 480, 'host'), (517, 389, 'device'),
             (1280, 720, 'host')]
    for k, (w, h, form) in enumerate(steps):
        frames = _frames(2, w, h, t0=5 * k)
        tag = 'step %d %dx%d %s' % (k, w, h, form)
        if form == 'host':
            _check_all(ex, oe, frames, list(zip(*ex.extract_batch(frames, LAP))), LAP, tag)
        else:
            _check_device(orb, torch, ex, oe, frames, 'crop' if k % 4 == 1 else 'packed', tag=tag)
    with pytest.raises(orb.OrbError) as e:
        ex.extract_batch(np.zeros((1, 721, 1280), np.uint8), LAP)         # taller than the handle
    assert e.value.code == orb.ORB_ERR_ARG
    u8 = lambda *shape: torch.zeros(shape, dtype=torch.uint8, device='cuda')
    i32 = lambda: torch.zeros(1, dtype=torch.int32, device='cuda')
    with pytest.raises(orb.OrbError) as e:
        ex.extract_batch_device(u8(1, 480, 1281), u8(1, 8, 28), u8(1, 8, 32), i32(), i32(), LAP)   # wider than the handle
    assert e.value.code == orb.ORB_ERR_ARG
    with pytest.raises(orb.OrbError) as e:
        ex.extract_batch(np.zeros((1, 700, 300), np.uint8), LAP)          # aspect < 0.5: the reference divides by zero
    assert e.value.code == orb.ORB_ERR_ASPECT
    frames = _frames(2, 640, 480, t0=99)
    _check_device(orb, torch, ex, oe, frames, 'packed', tag='after refusals')
    _check_all(ex, oe, frames, list(zip(*ex.extract_batch(frames, LAP))), LAP, 'after refusals host')


# ---------------------------------------------------------------------------------------------------------------------------------
# bilinear branch of pyr_resize_kernel
# ---------------------------------------------------------------------------------------------------------------------------------
def _level1_resize(w, h, scale, nlevels):
    """Level 1's size, whether it is an exact 2x decimation, and the TMA source box configure() computes for it (csrc/extractor.cu:
    the resize coefficient tables and the box covering the sources of any 128 x 8 destination tile)."""
    inv = O.OracleExtractor(1000, scale, nlevels, 20, 7).tables()['inv_scale']
    dw, dh = int(np.rint(np.float32(w) * inv[1])), int(np.rint(np.float32(h) * inv[1]))

    def tab(S, D):   # (first source, second source) per destination index, as the x / y tables clamp them
        s = np.floor(((np.arange(D) + 0.5) * (S / D) - 0.5).astype(np.float32).astype(np.float64)).astype(int)
        return np.clip(s, 0, S - 1), np.minimum(np.maximum(s + 1, 0), S - 1)
    x0, x1 = tab(w, dw)
    y0, y1 = tab(h, dh)
    bw = max([16] + [x1[min(d + 127, dw - 1)] - (x0[d] & ~15) + 1 for d in range(0, dw, 128)])
    bh = max([2] + [y1[min(d + 7, dh - 1)] - y0[d] + 1 for d in range(0, dh, 8)])
    return (dw, dh), (w == 2 * dw and h == 2 * dh), ((bw + 15) // 16 * 16, bh)


@pytest.mark.parametrize('w,h,scale,nlevels,size1,box_w', [(517, 389, 2.0, 3, (258, 194), 272), (1241, 376, 2.0, 3, (620, 188), 272),
                                                           (640, 480, 2.5, 3, (256, 192), 320), (640, 480, 3.0, 2, (213, 160), 384)])
def test_bilinear_pyramid_branch(orb, torch, w, h, scale, nlevels, size1, box_w):
    size, area2x, box = _level1_resize(w, h, scale, nlevels)
    # level 1 takes the bilinear branch of pyr_resize_kernel: not an exact 2x decimation, and a source box wider than TMA's 256
    assert size == size1 and not area2x and box[0] == box_w > 256, (size, area2x, box)
    ex = orb.ORBextractor(1000, scale, nlevels, 20, 7, w, h, 2)
    oe = O.OracleExtractor(1000, scale, nlevels, 20, 7)
    frames = _frames(2, w, h, t0=3)
    _check_all(ex, oe, frames, list(zip(*ex.extract_batch(frames, LAP))), LAP, 'host')
    _check_device(orb, torch, ex, oe, _frames(2, w, h, t0=21), 'crop')


# ---------------------------------------------------------------------------------------------------------------------------------
# FAST thresholds, geometry extremes, lapping areas
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('ini,mn', [(12, 5), (40, 7), (20, 20), (60, 12), (3, 1)])
def test_fast_thresholds(orb, ini, mn):
    rng = np.random.default_rng(ini * 100 + mn)
    frames = np.stack([synth.frame(4), (128 + rng.integers(-6, 7, (480, 640))).astype(np.uint8), rng.integers(0, 256, (480, 640)).astype(np.uint8)])
    ex = orb.ORBextractor(1000, 1.2, 8, ini, mn, 640, 480, 3)
    oe = O.OracleExtractor(1000, 1.2, 8, ini, mn)
    _check_all(ex, oe, frames, list(zip(*ex.extract_batch(frames, LAP))), LAP, 'th %d/%d' % (ini, mn))


def test_4095_px_wide(orb, torch):
    """The widest image the 12-bit candidate packing takes (level-0 x up to 4094)."""
    w, h = 4095, 300
    ex = orb.ORBextractor(2000, 1.2, 8, 20, 7, w, h, 1)
    oe = O.OracleExtractor(2000, 1.2, 8, 20, 7)
    wide = lambda t: np.tile(synth.frame(t, 1365, h), 3)[None]     # texture across the whole width
    frames = wide(2)
    _check_all(ex, oe, frames, list(zip(*ex.extract_batch(frames, LAP))), LAP, '4095 host')
    assert ex.candidates(0)[:, 0].max() > 4000
    _check_device(orb, torch, ex, oe, wide(9), 'packed', tag='4095')
    with pytest.raises(orb.OrbError):
        orb.ORBextractor(2000, 1.2, 8, 20, 7, 4096, 300, 1)


def test_single_level(orb, torch):
    """nlevels = 1: no pyramid launch."""
    ex = orb.ORBextractor(1000, 1.2, 1, 20, 7, 640, 480, 2)
    oe = O.OracleExtractor(1000, 1.2, 1, 20, 7)
    frames = _frames(2, 640, 480, t0=6)
    _check_all(ex, oe, frames, list(zip(*ex.extract_batch(frames, LAP))), LAP, 'host')
    _check_device(orb, torch, ex, oe, _frames(2, 640, 480, t0=13), 'packed', tag='nlevels=1')
    assert ex.last_launch_count() == 5


def test_lapping_areas(orb, torch):
    """Areas inside the image, an empty one, and bounds equal to the x of level-0 keypoints (both bounds are inclusive)."""
    frames = _frames(3, 640, 480, t0=17)
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    _, k0, _ = oe(frames[0], (0, 0))
    xs = np.unique(k0['x'][k0['octave'] == 0])
    lo, hi = int(xs[(xs > 100) & (xs < 300)][0]), int(xs[(xs > 400) & (xs < 600)][-1])
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 3)
    for lap in [(200, 440), (0, 0), (lo, hi)]:
        d = _on_device(torch, frames, 'packed')
        n, mono, kps, desc = _extract_device(orb, torch, ex, d, lap)
        _check_all(ex, oe, frames, _results(n, mono, kps, desc), lap, 'lap %s' % (lap,))
        if lap == (lo, hi):   # a keypoint on each bound: its row and monoIndex depend on whether the bound is inclusive
            assert (kps[0, :n[0]]['x'] == lo).any() and (kps[0, :n[0]]['x'] == hi).any()
    _check_all(ex, oe, frames, list(zip(*ex.extract_batch(frames, (lo, hi)))), (lo, hi), 'host lap')


# ---------------------------------------------------------------------------------------------------------------------------------
# host-form branches and capacity
# ---------------------------------------------------------------------------------------------------------------------------------
def _flat_sparse_dense():
    flat = np.full((480, 640), 90, np.uint8)
    sparse = flat.copy()
    sparse[200:209, 300:309] = 200        # one bright square: a handful of corners over the levels
    return np.stack([flat, sparse, synth.frame(12)])


def test_host_padded_frame_stride(orb):
    B, w, h = 3, 640, 480
    frames = _frames(B, w, h, t0=8)
    buf = np.zeros((B, h + 2, w), np.uint8)
    buf[:, :h] = frames
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, w, h, B)
    rc, n, mono, kps, desc = _host_call(orb, ex, buf, B, h, w, w, (h + 2) * w, ex.max_keypoints)
    assert rc == orb.ORB_OK
    _check_all(ex, O.OracleExtractor(1000, 1.2, 8, 20, 7), frames, _results(n, mono, kps, desc), LAP, 'padded stride')


def test_host_capacity_other_than_max_keypoints(orb):
    B = 3
    frames = _frames(B, 640, 480, t0=30)
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, B)
    cap = ex.max_keypoints - 7
    rc, n, mono, kps, desc = _host_call(orb, ex, frames, B, 480, 640, 640, 480 * 640, cap)
    assert rc == orb.ORB_OK and n.max() <= cap
    _check_all(ex, O.OracleExtractor(1000, 1.2, 8, 20, 7), frames, _results(n, mono, kps, desc), LAP, 'cap %d' % cap)
    for f in range(B):   # per-frame copies: nothing past n[f]
        assert (kps[f, n[f]:].view(np.uint8) == SENTINEL).all() and (desc[f, n[f]:] == SENTINEL).all(), f


def _oracle_counts(frames):
    oe = O.OracleExtractor(1000, 1.2, 8, 20, 7)
    return [oe(f, LAP) for f in frames]


def test_host_capacity_error(orb):
    """cap below one frame's count: ORB_ERR_CAPACITY, every n[f] / mono[f] reported, the frames that fit copied, the others untouched."""
    frames = _flat_sparse_dense()
    want = _oracle_counts(frames)
    assert len(want[0][1]) == 0 and 0 < len(want[1][1]) <= 64 < len(want[2][1])
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 3)
    rc, n, mono, kps, desc = _host_call(orb, ex, frames, 3, 480, 640, 640, 480 * 640, 64)
    assert rc == orb.ORB_ERR_CAPACITY
    for f, (om, ok, od) in enumerate(want):
        assert n[f] == len(ok) and mono[f] == om, (f, n[f], len(ok), mono[f], om)
        if n[f] <= 64:
            assert kps[f, :n[f]].tobytes() == ok.tobytes() and np.array_equal(desc[f, :n[f]], od), f
        else:
            assert (kps[f].view(np.uint8) == SENTINEL).all() and (desc[f] == SENTINEL).all(), f


def test_device_capacity_overflow(orb, torch):
    """Device form with cap = 64: the frames that fit are written, the dense frame reports d_n > cap and its slab rows keep the sentinel."""
    frames = _flat_sparse_dense()
    want = _oracle_counts(frames)
    ex = orb.ORBextractor(1000, 1.2, 8, 20, 7, 640, 480, 3)
    n, mono, kps, desc = _extract_device(orb, torch, ex, _on_device(torch, frames, 'packed'), LAP, cap=64)
    for f, (om, ok, od) in enumerate(want):
        assert n[f] == len(ok) and mono[f] == om, (f, n[f], len(ok), mono[f], om)
        k = n[f] if n[f] <= 64 else 0
        assert kps[f, :k].tobytes() == ok[:k].tobytes() and np.array_equal(desc[f, :k], od[:k]), f
        assert (kps[f, k:].view(np.uint8) == SENTINEL).all() and (desc[f, k:] == SENTINEL).all(), f
    assert n[2] > 64


# ---------------------------------------------------------------------------------------------------------------------------------
# device form of ComputeStereoMatches
# ---------------------------------------------------------------------------------------------------------------------------------
def test_stereo_matches_device(orb, torch):
    """Left frames read in place, right frames copied first: the stereo kernel reads both handles' level planes through the last call."""
    B, w, h, nf = 3, 640, 480, 1200
    pairs = [synth.stereo_pair(4 + 3 * b, w, h, seed=b) for b in range(B)]
    left, right = np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
    exl, exr = orb.ORBextractor(nf, 1.2, 8, 20, 7, w, h, B), orb.ORBextractor(nf, 1.2, 8, 20, 7, w, h, B)
    cap = exl.max_keypoints
    slabs = []
    for ex, frames, layout in ((exl, left, 'packed'), (exr, right, 'crop')):
        d = _on_device(torch, frames, layout)
        s = dict(img=d, kps=torch.zeros((B, cap, 28), dtype=torch.uint8, device='cuda'), desc=torch.zeros((B, cap, 32), dtype=torch.uint8, device='cuda'),
                 n=torch.zeros(B, dtype=torch.int32, device='cuda'), mono=torch.zeros(B, dtype=torch.int32, device='cuda'))
        ex.extract_batch_device(d, s['kps'], s['desc'], s['n'], s['mono'], (0, 0))
        slabs.append(s)
    L, R = slabs
    ur = torch.full((B, cap), -7.0, dtype=torch.float32, device='cuda')
    dep = torch.full((B, cap), -7.0, dtype=torch.float32, device='cuda')
    mbf = 22.0 * 8.0
    mb = mbf / 458.0
    exl.ComputeStereoMatchesDevice(exr, L['kps'], L['desc'], L['n'], R['kps'], R['desc'], R['n'], mb, mbf, ur, dep)
    torch.cuda.synchronize()
    ur, dep = ur.cpu().numpy(), dep.cpu().numpy()
    ol, orr = O.OracleExtractor(nf, 1.2, 8, 20, 7), O.OracleExtractor(nf, 1.2, 8, 20, 7)
    tb = ol.tables()
    for s in (L, R):
        n = s['n'].cpu().numpy()
        kps = s['kps'].cpu().numpy().view(orb.KP_DTYPE).reshape(B, cap)
        desc = s['desc'].cpu().numpy()
        s['host'] = [(kps[f, :n[f]], desc[f, :n[f]]) for f in range(B)]
    for b in range(B):
        _, okl, odl = ol(left[b], (0, 0))
        _, okr, odr = orr(right[b], (0, 0))
        assert L['host'][b][0].tobytes() == okl.tobytes() and R['host'][b][0].tobytes() == okr.tobytes(), b
        assert np.array_equal(L['host'][b][1], odl) and np.array_equal(R['host'][b][1], odr), b
        our, odep = O.stereo_matches([ol.level(l) for l in range(8)], [orr.level(l) for l in range(8)], okl, odl, okr, odr, tb['scale'], tb['inv_scale'],
                                     mb, mbf)
        n = len(okl)
        assert ur[b, :n].tobytes() == our.tobytes() and dep[b, :n].tobytes() == odep.tobytes(), (b, int((ur[b, :n] != our).sum()))
        assert (our >= 0).sum() > 300
