"""Time Frame::UndistortKeyPoints on the GPU against what a caller of the device tracking chain has to do without it, in the same run.

(a) orbx_undistort_keypoints_device inside the chain extract_batch_device -> undistort -> search_last_frame_batch_device: CUDA events
    bracket the undistortion launch alone on the chain's stream, median over --reps chains after warm-up.
(b) the round trip it replaces: synchronise after extraction, download the keypoint slab and the counts, cv2.undistortPoints per frame on
    the host (as Frame::UndistortKeyPoints calls it), upload the [batch][cap] slab again.  Host clock from the synchronise to the end of
    the upload, median over --reps.
Frames: the synthetic trajectory rendered through EuRoC cam0's distortion (752 x 480, tests/undistort_lib.py), 6 distinct frames tiled to
the batch; nfeatures 1000 and 1650 give about 1000 and 1650 keypoints per frame.  Both results are checked against each other before timing.
Prints the GPU's name, power limit and max SM clock with the numbers, and one JSON line.  Without a GPU it fails at the first CUDA call.
Usage: python tools/undistort_time.py [--reps 50] [--sizes 1,24,240] [--features 1000,1650]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]

import orb_slam3_modified_b200 as orb  # noqa: E402
import undistort_lib as U  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
    except FileNotFoundError:
        return None
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None


def host_round_trip(d_kps, d_n, K, D, out):
    """(b): download, cv2.undistortPoints per frame, upload into ``out``."""
    import torch
    torch.cuda.synchronize()
    kps = d_kps.cpu().numpy().view(np.uint8).reshape(d_kps.shape[0], d_kps.shape[1], 28).view(U.O.KP_DTYPE)[..., 0]
    n = d_n.cpu().numpy()
    un = kps.copy()
    for f in range(len(n)):
        k = int(n[f])
        if 0 < k <= kps.shape[1]:
            xy = U.cv2_undistort(np.stack([kps[f, :k]['x'], kps[f, :k]['y']], 1), K, D)
            un[f, :k]['x'] = xy[:, 0]; un[f, :k]['y'] = xy[:, 1]
    out.copy_(torch.from_numpy(un.view(np.uint8).reshape(out.shape[0], out.shape[1], 28).view(np.float32)))
    torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--sizes', default='1,24,240')
    ap.add_argument('--features', default='1000,1650')
    a = ap.parse_args()
    import torch
    K, D, W, H = U.CALIBRATIONS['euroc']
    base = np.stack([U.distorted_frame(t, W, H, K, D) for t in range(6)])
    info = gpu_info()
    print('GPU:', info)
    rows = []
    st = torch.cuda.Stream()
    for nf in [int(x) for x in a.features.split(',')]:
        for B in [int(x) for x in a.sizes.split(',')]:
            ex = orb.ORBextractor(nf, 1.2, 8, 20, 7, W, H, B)
            cap = ex.max_keypoints
            d_img = torch.from_numpy(np.ascontiguousarray(base[np.arange(B) % 6])).cuda()
            d_kps = torch.zeros((B, cap, 7), dtype=torch.float32, device='cuda'); d_desc = torch.zeros((B, cap, 32), dtype=torch.uint8, device='cuda')
            d_n = torch.zeros(B, dtype=torch.int32, device='cuda'); d_mono = torch.zeros(B, dtype=torch.int32, device='cuda')
            d_un = torch.zeros_like(d_kps); d_host = torch.zeros_like(d_kps)
            mcap = cap
            m = orb.ORBmatcher(0.9, True, max_batch=B, max_keypoints=cap, max_mappoints=mcap)
            # last frame: the current frame's own keypoints, back-projected at 3 m, so the search does real work
            bounds = orb.image_bounds(K, D, W, H)
            z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device='cuda')
            d = dict(batch=B, kcap=cap, mcap=mcap, nlevels=8, kps=d_un, desc=d_desc, nK=d_n,
                     scaleFactors=torch.from_numpy((1.2 ** np.arange(8)).astype(np.float32)).cuda(), nM=d_n, valid=z(B, mcap, dt=torch.uint8) + 1,
                     xyz=z(B, mcap, 3), octave=z(B, mcap, dt=torch.int32), angle=z(B, mcap), hasObs=z(B, mcap, dt=torch.uint8) + 1, mpDesc=d_desc,
                     Tcw7=torch.tensor([[1, 0, 0, 0, 0, 0, 0]] * B, dtype=torch.float32, device='cuda'), cam=[float(c) for c in K], bounds=bounds, reset=1)
            match = z(B, cap, dt=torch.int32); claimed = z(B, cap, dt=torch.uint8); nm = z(B, dt=torch.int32)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s = st.cuda_stream

            def chain(timed):
                ex.extract_batch_device(d_img, d_kps, d_desc, d_n, d_mono, (0, 1000), s)
                if timed:
                    e0.record(st)
                ex.undistort_keypoints_device(K, D, d_kps, d_n, d_un, s)
                if timed:
                    e1.record(st)
                u = d_un.view(torch.uint8).view(B, cap, 28)
                with torch.cuda.stream(st):
                    xy = d_un[:, :, :2].double()
                    d['xyz'] = torch.stack([(xy[..., 0] - K[2]) / K[0] * 3.0, (xy[..., 1] - K[3]) / K[1] * 3.0, torch.full_like(xy[..., 0], 3.0)], 2).float().contiguous()
                    d['octave'] = u[:, :, 20:24].contiguous().view(torch.int32).view(B, cap).contiguous()
                    d['angle'] = d_un[:, :, 3].contiguous()
                m.search_last_frame_batch_device(d, 15.0, match, claimed, nm, s)

            chain(False)
            torch.cuda.synchronize()
            host_round_trip(d_kps, d_n, K, D, d_host)
            n = d_n.cpu().numpy()
            a_ = d_un.cpu().numpy().view(np.uint8).reshape(B, cap, 28); b_ = d_host.cpu().numpy().view(np.uint8).reshape(B, cap, 28)
            assert all(a_[f, :n[f]].tobytes() == b_[f, :n[f]].tobytes() for f in range(B)), 'device and cv2 undistortion differ'
            assert int(nm.cpu().numpy().min()) > 0, 'the chain found no matches'
            dev_ms, host_ms = [], []
            for _ in range(a.reps):
                chain(True)
                torch.cuda.synchronize()
                dev_ms.append(e0.elapsed_time(e1))
            for _ in range(a.reps):
                ex.extract_batch_device(d_img, d_kps, d_desc, d_n, d_mono, (0, 1000), s)
                t0 = time.perf_counter()
                host_round_trip(d_kps, d_n, K, D, d_host)
                host_ms.append(1e3 * (time.perf_counter() - t0))
            row = dict(frames=B, nfeatures=nf, mean_keypoints=float(n.mean()), device_ms=statistics.median(dev_ms), host_round_trip_ms=statistics.median(host_ms))
            rows.append(row)
            print('%4d frames, %5.0f keypoints/frame: device %.4f ms, host round trip %.3f ms' % (B, row['mean_keypoints'], row['device_ms'], row['host_round_trip_ms']))
            del ex, m
    print(json.dumps(dict(gpu=info, calibration='euroc cam0 752x480', rows=rows)))


if __name__ == '__main__':
    main()
