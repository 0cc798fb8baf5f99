"""Time K7 with prioritized replay (serl_td3_learn with a tree) against K7's uniform sampler (serl_td3_learn without): h = 72, L = 3,
batch 86, CAPS on, 800,000 replay rows from K1 flights, the tree's priorities made uneven by PER steps before the timing.
Per cluster size, the two alternate three times over `--steps` steps each (CUDA events after warm-up).  Also times the
insert of one SERL10 generation's rows into the tree (serl_per_insert: the max reduction and the rebuild).  Prints one
JSON line with the card's name, power limit and SM clock.

    python scripts/time_td3_per.py [--steps 3000]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from serl_b200.core.replay_memory import DevicePrioritizedReplayMemory  # noqa: E402
from serl_b200.td3_fused import FusedTD3  # noqa: E402
from time_td3 import SERL10_STEPS, fill_replay, learner_args, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3000)
    ap.add_argument('--warmup', type=int, default=300)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_td3_per.py measures on the GPU; no CUDA device found')
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    mem = fill_replay(dev)
    per = DevicePrioritizedReplayMemory(mem.capacity, dev, seed=7, beta_frames=800_000)
    per.add_rows(mem.data[:len(mem)])
    assert torch.equal(per.data, mem.data)
    args = learner_args(dev)
    torch.manual_seed(7)
    fused = FusedTD3(args)

    def k7(n, cs, p):
        if p:
            fused.run(per.data, len(per), n, fused.critic_steps + 1, False, cluster_size=cs, per=per)
        else:
            fused.run(mem.data, len(mem), n, fused.critic_steps + 1, False, cluster_size=cs)

    sizes = (1, 2, 4, 8)
    k7(5000, 8, True)                                   # uneven priorities: 5000 steps of re-prioritising
    for cs in sizes:
        k7(a.warmup, cs, False)
        k7(a.warmup, cs, True)
    res = {cs: {'uniform': [], 'per': []} for cs in sizes}
    for _ in range(3):
        for cs in sizes:
            res[cs]['uniform'].append(timed(lambda: k7(a.steps, cs, False)) / a.steps)
            res[cs]['per'].append(timed(lambda: k7(a.steps, cs, True)) / a.steps)
    rows = mem.data[:SERL10_STEPS].clone()
    per.add_rows(rows)
    insert = [timed(lambda: per.add_rows(rows)) for _ in range(5)]
    fused.status.zero_()
    st = fused.run(per.data, len(per), 10, fused.critic_steps + 1, False, per=per)
    st.check()
    leaves = per.leaves()
    out = {'card': q, 'replay_rows': len(per), 'steps': a.steps, 'batch': args.batch_size, 'hidden': 72, 'num_layers': 3,
           'us_per_step': {str(cs): {k: [round(x, 2) for x in v] for k, v in r.items()} for cs, r in res.items()},
           'per_over_uniform': {str(cs): round(min(r['per']) / min(r['uniform']), 4) for cs, r in res.items()},
           'insert_%d_rows_us' % SERL10_STEPS: [round(x, 1) for x in insert],
           'priority_min_max': [float(leaves.min()), float(leaves.max())]}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
