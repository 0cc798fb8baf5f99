import os, sys, torch, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import bench
from serl_b200 import rollout, refsig
dev = torch.device('cuda:0')
pop = int(sys.argv[1]) if len(sys.argv) > 1 else 512
w = torch.from_numpy(bench.population(pop)).to(dev)
lv, st = refsig.make_ref_params(128)
md = torch.zeros(128, dtype=torch.int32, device=dev)
r = rollout.population_rollout(w, rollout.actor_shape(72), torch.as_tensor(lv, device=dev), torch.as_tensor(st, device=dev), md, actions=True)
for i in range(3):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); sm = rollout.smoothness(r.actions, r.steps); e1.record(); torch.cuda.synchronize()
    print('K6: %.2f ms for %d trajectories' % (e0.elapsed_time(e1), r.steps.numel()))
print('mean smoothness', float(sm.mean()))
