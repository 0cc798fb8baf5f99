"""Time K7's group launch (serl_td3_learn with one learner per run) and the sweep driver.

(a) G learners at h = 72, L = 3, batch 86, CAPS on, on a replay of 800,000 K1 flight rows, cluster size 8 (and G = 32 at
    cluster size 4), three arms alternated twice: ONE grouped launch of G clusters, G solo launches in sequence (the only
    option in one process before), G solo launches on G streams.  Reports us per step of the group (every learner takes
    one step) and learner-steps per second.
(b) A Sweep of S SERL10-shaped runs (pop 10, 3 envs, h = 72, fused_td3): seconds per sweep generation, against S x the
    seconds of one run's generation.  The first generation of every S is a warm-up (it also fills the replay past
    learn_start); the second is timed.
CUDA events / a synchronised host clock after warm-up.  Prints one JSON line with the card's name and power limit.

    python scripts/time_td3_group.py [--steps 300] [--sweep 1,4,8,16]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from serl_b200 import td3_fused  # noqa: E402
from serl_b200.td3_fused import FusedTD3  # noqa: E402
from time_td3 import fill_replay, learner_args, timed  # noqa: E402

GROUPS = [(1, 8), (2, 8), (4, 8), (8, 8), (12, 8), (16, 8), (32, 8), (32, 4)]


def learners(dev, G, cs):
    out = []
    for g in range(G):
        torch.manual_seed(7 + g)
        out.append(FusedTD3(learner_args(dev), cluster_size=cs, seed=7 + g))
    return out


def time_groups(dev, mem, steps, warmup):
    pool = {key: learners(dev, *key) for key in GROUPS}
    streams = [torch.cuda.Stream(dev) for _ in range(max(G for G, _ in GROUPS))]

    def grouped(fs, n):
        td3_fused.train_group(fs, [mem] * len(fs), [n] * len(fs), [f.critic_steps + 1 for f in fs], [False] * len(fs))

    def sequential(fs, n):
        for f in fs:
            f.run(mem.data, len(mem), n, f.critic_steps + 1, False)

    def streamed(fs, n):
        cur = torch.cuda.current_stream(dev)
        for f, s in zip(fs, streams):
            s.wait_stream(cur)
            with torch.cuda.stream(s):
                f.run(mem.data, len(mem), n, f.critic_steps + 1, False)
        for s in streams[:len(fs)]:
            cur.wait_stream(s)

    arms = {'group': grouped, 'sequential': sequential, 'streams': streamed}
    for fs in pool.values():
        for fn in arms.values():
            fn(fs, warmup)
    res = {'%d@cs%d' % key: {k: [] for k in arms} for key in GROUPS}
    for _ in range(2):
        for key, fs in pool.items():
            for name, fn in arms.items():
                res['%d@cs%d' % key][name].append(timed(lambda: fn(fs, steps)) / steps)
    for fs in pool.values():
        for f in fs:
            f.status.zero_()
            f.run(mem.data, len(mem), 5, f.critic_steps + 1, False).check()
    out = {}
    for (G, cs) in GROUPS:
        r = res['%d@cs%d' % (G, cs)]
        out['%d@cs%d' % (G, cs)] = {
            'us_per_group_step': {k: [round(x, 1) for x in v] for k, v in r.items()},
            'learner_steps_per_s': {k: round(G * 1e6 / min(v)) for k, v in r.items()},
        }
    return out


def serl10_params(seed, tmpdir):
    from serl_b200.parameters import Parameters
    cwd = os.getcwd()
    os.chdir(tmpdir)
    try:
        p = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=seed, pop_size=10, mut_type='normal', test_ea=False,
                                             fused_td3=True))
    finally:
        os.chdir(cwd)
    p.state_dim, p.action_dim = 7, 3
    return p


def time_sweeps(sizes):
    import tempfile
    from serl_b200.envs import config
    from serl_b200.sweep import Sweep
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for S in sizes:
            sw = Sweep([(serl10_params(7 + i, tmp), config.select_env('PHlab_attitude_nominal')) for i in range(S)])
            sw.train()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            stats = sw.train()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            steps = [r.agent.rl_iteration for r in sw.runs]
            assert all(s is not None for s in stats) and min(steps) > 0
            out[S] = {'s_per_generation': round(dt, 3), 'rl_steps_per_run': steps[0]}
            del sw, stats
            torch.cuda.empty_cache()
    one = out[min(sizes)]['s_per_generation'] / min(sizes)
    for S in sizes:
        out[S]['s_x_one_run'] = round(S * one, 3)
    return {str(k): v for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--sweep', type=str, default='1,4,8,16', help='sweep sizes S ("" to skip)')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_td3_group.py measures on the GPU; no CUDA device found')
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    mem = fill_replay(dev)
    out = {'card': q, 'replay_rows': len(mem), 'steps': a.steps, 'batch': 86, 'hidden': 72, 'num_layers': 3,
           'sms': torch.cuda.get_device_properties(dev).multi_processor_count,
           'groups': time_groups(dev, mem, a.steps, a.warmup)}
    del mem
    torch.cuda.empty_cache()
    if a.sweep:
        out['sweep'] = time_sweeps([int(s) for s in a.sweep.split(',')])
    print(json.dumps(out))


if __name__ == '__main__':
    main()
