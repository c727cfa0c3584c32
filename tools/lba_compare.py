"""LocalBundleAdjustment on bench.py's batch of 48 problems (one launch, as the device-resident loop runs it), for checking that a
kernel change leaves the results where they were.

  ORB_B200_LIB=<lib> python tools/lba_compare.py save OUT.npz     runs the batch twice, checks that the two runs are byte-identical
                                                                  and saves the results of the library ORB_B200_LIB selects
  python tools/lba_compare.py compare A.npz B.npz                 iteration and trial counts, largest pose, point and edge-chi2
                                                                  differences, largest final-chi2 difference"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
KEYS = ('poses', 'points', 'chi2')


def save(path):
    import orb_slam3_modified_b200 as orb
    from bench import LBA_CFG, lba_problems
    probs = lba_problems(48)
    opt = orb.Optimizer(max_poses=LBA_CFG['n_kf'], max_points=LBA_CFG['n_pts'], max_edges=LBA_CFG['n_pts'] * LBA_CFG['obs_per_pt'],
                        max_batch=len(probs))
    runs = []
    for _ in range(2):
        opt.upload(probs)
        opt.run_device()
        runs.append(opt.download())
    for a, b in zip(*runs):
        assert all(a[k].tobytes() == b[k].tobytes() for k in KEYS) and (a['iters'], a['trials'], a['final_chi2']) == \
            (b['iters'], b['trials'], b['final_chi2']), 'two runs of one build differ'
    out = runs[0]
    np.savez(path, **{k: np.stack([o[k] for o in out]) for k in KEYS},
             iters=np.array([o['iters'] for o in out]), trials=np.array([o['trials'] for o in out]),
             final_chi2=np.array([o['final_chi2'] for o in out]), cluster=opt.last_cluster_size())
    print('%s: %d problems, cluster %d, repeats byte-identical' % (path, len(out), opt.last_cluster_size()))


def compare(pa, pb):
    a, b = np.load(pa), np.load(pb)
    print('iterations identical: %s, trials identical: %s' % (np.array_equal(a['iters'], b['iters']), np.array_equal(a['trials'], b['trials'])))
    for k in KEYS:
        print('largest %-6s difference %.3g' % (k, np.abs(a[k] - b[k]).max()))
    print('largest final chi2 difference %.3g (relative %.3g)' % (np.abs(a['final_chi2'] - b['final_chi2']).max(),
                                                                 (np.abs(a['final_chi2'] - b['final_chi2']) / np.abs(a['final_chi2'])).max()))


if __name__ == '__main__':
    if sys.argv[1:2] == ['save']:
        save(sys.argv[2])
    elif sys.argv[1:2] == ['compare']:
        compare(sys.argv[2], sys.argv[3])
    else:
        sys.exit(__doc__)
