"""Time K7's group launch of prioritized learners (serl_td3_learn) against what it replaces and against uniform
replay in a group.  h = 72, L = 3, batch 86, CAPS on, cluster size 8, 800,000 replay rows from K1 flights in every tree,
the trees' priorities made uneven by 5,000 PER steps before the timing (each learner gets its own copy of that tree).

(a) S prioritized learners in ONE serl_td3_learn launch, against S solo prioritized launches back to back.
(b) The same S learners uniform in ONE serl_td3_learn launch, against prioritized in one launch.
    For S = 1, 4, 16, 64: the three arms alternate three times over `--steps` steps each (CUDA events after warm-up);
    us per step of the group (every learner takes one step).
(c) Two Sweeps of S SERL10-sized runs (pop 10, 3 envs, h = 72, fused_td3), one with every run prioritized (Sweep(...,
    per=True)), one with every run uniform: seconds per sweep generation (synchronised host clock), generations 2 and 3
    of each, the two sweeps alternated.  Includes each prioritized run's tree inserts.
Prints one JSON line with the card's name, power limit and max SM clock.

    python scripts/time_td3_group_per.py [--steps 2000] [--sweep 8]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from serl_b200 import td3_fused  # noqa: E402
from serl_b200.core.replay_memory import DevicePrioritizedReplayMemory  # noqa: E402
from serl_b200.td3_fused import FusedTD3  # noqa: E402
from time_td3 import fill_replay, learner_args, timed  # noqa: E402
from time_td3_group import serl10_params  # noqa: E402

SIZES = (1, 4, 16, 64)
CS = 8


def time_groups(dev, steps, warmup):
    mem = fill_replay(dev)
    base = DevicePrioritizedReplayMemory(mem.capacity, dev, seed=7, beta_frames=800_000)
    base.add_rows(mem.data[:len(mem)])
    torch.manual_seed(7)
    f0 = FusedTD3(learner_args(dev), cluster_size=CS)
    f0.run(base.data, len(base), 5000, 1, False, per=base).check()      # uneven priorities
    leaves = base.leaves()
    spread = [float(leaves.min()), float(leaves.max())]
    S_max = max(SIZES)
    fs = []
    for g in range(S_max):
        torch.manual_seed(7 + g)
        fs.append(FusedTD3(learner_args(dev), cluster_size=CS, seed=7 + g))
    trees = []
    for g in range(S_max):        # the rows are shared; each learner re-prioritises its own copy of the tree
        b = copy.copy(base)
        b.tree = base.tree.clone()
        trees.append(b)

    def group_per(S, n):
        td3_fused.train_group(fs[:S], trees[:S], [n] * S, [f.critic_steps + 1 for f in fs[:S]], [False] * S, prioritized=True)

    def solo_per(S, n):
        for f, b in zip(fs[:S], trees[:S]):
            f.run(b.data, len(b), n, f.critic_steps + 1, False, per=b)

    def group_uniform(S, n):
        td3_fused.train_group(fs[:S], [mem] * S, [n] * S, [f.critic_steps + 1 for f in fs[:S]], [False] * S)

    arms = {'group_per': group_per, 'solo_per': solo_per, 'group_uniform': group_uniform}
    for S in SIZES:
        for fn in arms.values():
            fn(S, warmup)
    res = {S: {k: [] for k in arms} for S in SIZES}
    for _ in range(3):
        for S in SIZES:
            for name, fn in arms.items():
                res[S][name].append(timed(lambda: fn(S, steps)) / steps)
    for f, b in zip(fs, trees):
        f.status.zero_()
        f.run(b.data, len(b), 5, f.critic_steps + 1, False, per=b).check()
    out = {}
    for S in SIZES:
        r = res[S]
        out[str(S)] = {'us_per_group_step': {k: [round(x, 1) for x in v] for k, v in r.items()},
                       'solo_per_over_group_per': round(min(r['solo_per']) / min(r['group_per']), 3),
                       'group_per_over_group_uniform': round(min(r['group_per']) / min(r['group_uniform']), 4)}
    return out, len(mem), spread


def time_sweeps(S):
    from serl_b200.envs import config
    from serl_b200.sweep import Sweep
    out = {'runs': S, 'per': [], 'uniform': []}
    with tempfile.TemporaryDirectory() as tmp:
        sweeps = {}
        for arm in ('per', 'uniform'):
            ps = [serl10_params(7 + i, tmp) for i in range(S)]
            for p in ps:
                p.per = arm == 'per'
            sweeps[arm] = Sweep([(p, config.select_env('PHlab_attitude_nominal')) for p in ps], per=True)
            sweeps[arm].train()                   # generation 1: warm-up
        for _ in range(2):                        # generations 2 and 3, the arms alternated
            for arm, sw in sweeps.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                stats = sw.train()
                torch.cuda.synchronize()
                out[arm].append(round(time.perf_counter() - t0, 3))
                assert all(s is not None for s in stats)
        out['rl_steps_per_run'] = sweeps['per'].runs[0].agent.rl_iteration
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=2000)
    ap.add_argument('--warmup', type=int, default=200)
    ap.add_argument('--sweep', type=int, default=8, help='runs per sweep in (c) (0 to skip)')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_td3_group_per.py measures on the GPU; no CUDA device found')
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    groups, rows, spread = time_groups(dev, a.steps, a.warmup)
    out = {'card': q, 'replay_rows': rows, 'steps': a.steps, 'batch': 86, 'hidden': 72, 'num_layers': 3, 'cluster_size': CS,
           'priority_min_max': spread, 'groups': groups}
    torch.cuda.empty_cache()
    if a.sweep:
        out['sweep'] = time_sweeps(a.sweep)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
