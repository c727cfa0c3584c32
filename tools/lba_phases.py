import sys, ctypes as C; sys.path.insert(0,'.'); sys.path.insert(0,'tests')
import numpy as np, time
import orb_slam3_modified_b200 as orb
from orb_slam3_modified_b200 import synth
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1
opt = orb.Optimizer(20, 5000, 40000, max_batch=n)
p = synth.lba_problem()
import torch
opt.upload([p]*n)
if len(sys.argv) > 2: opt.set_cluster_size(int(sys.argv[2]))
if len(sys.argv) > 3: opt.set_helpers(int(sys.argv[3]))
for _ in range(2): opt.run_device()
torch.cuda.synchronize()
e0,e1=torch.cuda.Event(enable_timing=True),torch.cuda.Event(enable_timing=True)
e0.record(); opt.run_device(torch.cuda.current_stream().cuda_stream); e1.record(); torch.cuda.synchronize()
out = opt.download()
ns = np.zeros(10)
L = orb.lib()
L.lba_get_phase_ns(opt._h, 0, ns.ctypes.data_as(C.c_void_p))
names=['errors(it0)','build','poses_combine','point_prep','schur_partial','ldlt','schur_combine','pose_trial','points_trial']
print('batch',n,'cluster',opt.last_cluster_size(),'helper clusters',opt.last_helpers(),'kernel ms',e0.elapsed_time(e1),'iters',out[0]['iters'],'trials',out[0]['trials'])
for k,v in zip(names,ns): print('  %-14s %8.1f us total  %7.1f us/trial'%(k,v/1e3,v/1e3/max(out[0]['trials'],1)))
helped, per = [], []
for i in range(n):
    L.lba_get_phase_ns(opt._h, i, ns.ctypes.data_as(C.c_void_p)); helped.append(int(ns[9])); per.append(ns[:9] / 1e3 / max(out[i]['trials'], 1))
per = np.array(per)
print('  over all %d problems, us/trial:  %s' % (n, '  '.join('%s mean %.1f max %.1f' % (k, per[:, j].mean(), per[:, j].max())
                                                           for j, k in enumerate(names) if k in ('build', 'schur_partial', 'points_trial'))))
print('chunks served by helpers per problem: min %d  mean %.1f  max %d  (problem 0: %d)' % (min(helped), sum(helped) / n, max(helped), helped[0]))
