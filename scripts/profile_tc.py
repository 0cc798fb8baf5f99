import os, sys, torch, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
from serl_b200 import rollout, refsig
from oracle import actor as A
dev = torch.device('cuda:0')
widths = [int(x) for x in sys.argv[1].split(',')] if len(sys.argv) > 1 else [400, 300]
pop, n_envs, horizon = 132, 256, int(sys.argv[2]) if len(sys.argv) > 2 else 60
torch.manual_seed(7)
g = np.stack([A.flatten(A.WideActor(widths)) for _ in range(4)])
w = torch.from_numpy(np.tile(g, (pop // 4, 1)).astype(np.float32)).to(dev)
lv, st = refsig.make_ref_params(n_envs)
md = torch.zeros(n_envs, dtype=torch.int32, device=dev)
for i in range(2):
    r = rollout.population_rollout(w, rollout.actor_shape(72), torch.as_tensor(lv, device=dev), torch.as_tensor(st, device=dev), md, horizon=horizon, widths=widths)
    torch.cuda.synchronize()
print('ok', int(r.steps.sum()))
