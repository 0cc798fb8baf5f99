"""Time the population evaluation suite against the per-(actor, condition) validate_agent loop it replaces.

Populations: SERL10 (10 actors, h = 72, tanh) and the 8 SERL50 actors (h = 32, tanh) of tests/golden/actors.npz, on every
condition (evaluation.CONDITIONS) with num_trails = 2 (three 80 s trials per actor and condition).
  suite     evaluation.evaluate_population: one rollout launch per sensor-noise group + one K6 launch (host clock around the
            call, which ends in a device synchronise); the K6 launch is timed with CUDA events inside the same calls
  per-call  evaluation.validate_agent for each actor and condition, one traced launch each (host clock)
One warm-up call of each arm first; the suite is timed --reps times.  Prints one JSON line with the card's name and power
limit.

    python scripts/time_eval_suite.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from serl_b200 import evaluation, rollout  # noqa: E402

POPS = {'serl10_h72': ('serl10_pop_h72_tanh', 72), 'serl50_h32': ('serl50_pop8_h32_tanh', 32)}


def timed_k6():
    """wrap rollout.smoothness (the module function evaluate_population calls) to time each call with CUDA events"""
    inner, times = rollout.smoothness, []

    def wrapper(actions, steps, dt=0.01):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out = inner(actions, steps, dt)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
        return out
    rollout.smoothness = wrapper
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--num_trails', type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_eval_suite.py measures on the GPU; no CUDA device found')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    acts = np.load(os.path.join(ROOT, 'tests', 'golden', 'actors.npz'))
    conds = list(evaluation.CONDITIONS)
    k6 = timed_k6()
    out = {'card': q, 'conditions': len(conds), 'trials': a.num_trails + 1, 'episode_steps': 8001, 'pops': {}}
    for name, (key, h) in POPS.items():
        g = acts[key]
        shape = rollout.actor_shape(h)
        np.random.seed(7)
        refs = evaluation.eval_refs(a.num_trails)
        evaluation.evaluate_population(g, shape, conds, refs, a.num_trails)          # warm-up
        evaluation.validate_agent(g[0], shape, evaluation.condition_env('nominal'), refs, a.num_trails)
        suite = []
        del k6[:]
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            evaluation.evaluate_population(g, shape, conds, refs, a.num_trails)
            suite.append(time.perf_counter() - t0)
        k6_s = list(k6)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for c in conds:
            env = evaluation.condition_env(c)
            for i in range(g.shape[0]):
                evaluation.validate_agent(g[i], shape, env, refs, a.num_trails)
        loop = time.perf_counter() - t0
        out['pops'][name] = {'actors': int(g.shape[0]), 'trajectories': int(g.shape[0]) * len(conds) * (a.num_trails + 1),
                             'suite_s': suite, 'k6_s': k6_s, 'k6_share': float(np.median(k6_s) / np.median(suite)),
                             'per_call_loop_s': loop, 'per_call_calls': int(g.shape[0]) * len(conds),
                             'speedup': float(loop / np.median(suite))}
        print(json.dumps({name: out['pops'][name]}), flush=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
