"""Time the mutation-operator study (serl_b200.operators) against the same study flown as a direct port of
base/core/operator_runner.py would fly it.

Populations: SERL10 (10 actors, h = 72, tanh) and the 8 SERL50 actors (h = 32, tanh) of tests/golden/actors.npz, nominal
condition, 20 s episodes, num_trails 0 and 3, one magnitude (the run default 0.05) and five (0.01, 0.02, 0.05, 0.1, 0.2).
  study   OperatorRunner.test_mutation: one per-actor-block parent launch, the mutations, one tracking launch for every
          child (host clock around the call, which ends in device synchronises)
  port    the study's flights as one evaluation.validate_agent launch per (model, variant, trial): the parent and the
          3 x |mags| children of every model (host clock; flights only, the mutations are not included)
One warm-up call of each arm per configuration; the study is timed --reps times, the port once.  Prints one JSON line with
the card's name and power limit.

    python scripts/time_operators.py [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from serl_b200 import evaluation, operators  # noqa: E402

POPS = {'serl10_h72': ('serl10_pop_h72_tanh', 72), 'serl50_h32': ('serl50_pop8_h32_tanh', 32)}
MAGS = {1: None, 5: [0.01, 0.02, 0.05, 0.1, 0.2]}


def port(runner, genomes, children, refs):
    env = runner.env
    n = 0
    for g in list(genomes) + list(children):
        for t in range(runner.num_trails + 1):
            evaluation.validate_agent(g, runner.shape, env, [refs[t]], 0)
            n += 1
    torch.cuda.synchronize()
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_operators.py measures on the GPU; no CUDA device found')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    acts = np.load(os.path.join(ROOT, 'tests', 'golden', 'actors.npz'))
    out = {'card': q, 'episode_steps': 2001, 'runs': []}
    for name, (key, h) in POPS.items():
        g = acts[key]
        args = types.SimpleNamespace(hidden_size=h, num_layers=3, activation_actor='tanh', individual_bs=10_000,
                                     mutation_batch_size=64, mutation_mag=0.05, seed=7)
        for num_trails in (0, 3):
            np.random.seed(7)
            refs = operators.study_refs(num_trails)
            runner = operators.OperatorRunner(args, 'nominal', num_trails=num_trails)
            for n_mags, mags in MAGS.items():
                runner.test_mutation(g, refs, mags)            # warm-up
                times = []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    study = runner.test_mutation(g, refs, mags)
                    torch.cuda.synchronize()
                    times.append(time.perf_counter() - t0)
                kids = study.child_genomes.reshape(-1, study.child_genomes.shape[-1])
                port(runner, g[:1], [], refs)                  # warm-up
                t0 = time.perf_counter()
                n = port(runner, g, kids, refs)
                tp = time.perf_counter() - t0
                rec = {'pop': name, 'actors': int(g.shape[0]), 'num_trails': num_trails, 'mags': n_mags,
                       'episodes': int(n), 'study_s': [round(x, 4) for x in times], 'port_s': round(tp, 3),
                       'speedup': round(tp / min(times), 1)}
                print(json.dumps(rec), flush=True)
                out['runs'].append(rec)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
