"""The evaluation suite's tracking launch (track=True, cost=True) of incremental and symmetric control (suite=True) against its
attitude twin, on a SERL10-sized workload: 10 actors (h = 72, L = 3, the bench's trained layers) x 13 conditions x 3 trials
of 80 s = 39 envs x 8001 steps per actor.  Every env flies the nominal build, and every arm has a zero output layer, so all
three hold trim and fly every step: the launch times compare the same number of executed steps (the actor still computes
every layer).  The incremental genomes take the attitude layer 0 with three zero input columns (last_u), the symmetric ones
its first two input columns (theta error, p) and the first output row.
The arms alternate, `rounds` times each, in one process; every launch is timed with CUDA events after a warm-up launch of
each, and each arm must reproduce its warm-up bits.  Prints one JSON object with the card, its power limit and its clocks.
usage: python scripts/time_eval_modes.py [rounds=3]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from serl_b200 import evaluation, rollout       # noqa: E402

rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
dev = torch.device('cuda:0')
H, L, POP, CONDS, TRIALS = 72, 3, 10, 13, 3


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm,clocks.mem'
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', '0'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def genomes(w, S, A):
    """[pop, P(7 -> 3)] -> [pop, P(S -> A)] with a zero output layer"""
    n = w.shape[0]
    w0 = w[:, :7 * H].reshape(n, H, 7)
    w0 = np.concatenate([w0, np.zeros((n, H, S - 7), np.float32)], axis=2) if S > 7 else w0[:, :, :S]
    mid = w[:, 7 * H:w.shape[1] - (3 * H + 3)]
    out = np.zeros((n, A * H + A), np.float32)
    return np.ascontiguousarray(np.concatenate([w0.reshape(n, -1), mid, out], axis=1))


def main():
    w = np.load(os.path.join(ROOT, 'tests', 'golden', 'actors.npz'))['serl10_pop_h72_tanh'][:POP]
    np.random.seed(7)
    refs = evaluation.eval_refs(TRIALS - 1) * CONDS
    sym_refs = evaluation.symmetric_refs(TRIALS - 1, 7) * CONDS
    n_envs = len(refs)
    arms = {}
    for name, (S, A, cond, rf) in {'attitude': (7, 3, 'nominal', refs), 'incremental': (10, 3, 'incremental', refs),
                                   'symmetric': (2, 1, 'PHlab_symmetric_nominal', sym_refs)}.items():
        shape = rollout.actor_shape(H, L, 'tanh', S, A)
        lv, st = evaluation._ref_arrays(rf)
        md = torch.full((n_envs,), evaluation.condition_env(cond, shape=shape).mode_code, dtype=torch.int32, device=dev)
        g = torch.as_tensor(genomes(w, S, A), device=dev)
        assert g.shape[1] == rollout.num_params(shape)
        arms[name] = (g, shape, torch.as_tensor(lv, device=dev), torch.as_tensor(st, device=dev), md, float(rf[0][0].smooth_width), S != 7 or A != 3)

    def run(a):
        g, shape, lv, st, md, sw, suite = arms[a]
        return rollout.population_rollout(g, shape, lv, st, md, horizon=8001, t_max=80.0, smooth_width=sw, fitness=False, track=True,
                                          cost=True, suite=suite)
    ref = {a: run(a) for a in arms}
    torch.cuda.synchronize()
    ms, same = {a: [] for a in arms}, True
    for _ in range(rounds):
        for a in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = run(a)
            e1.record()
            torch.cuda.synchronize()
            r.check()
            ms[a].append(e0.elapsed_time(e1))
            same = same and torch.equal(r.returns, ref[a].returns) and torch.equal(r.track, ref[a].track)
    out = {'card: name, power limit, sm clock, max sm clock, mem clock': card(), 'rounds': rounds, 'pop': POP, 'n_envs': n_envs,
           'horizon': 8001, 'hidden': H, 'bitwise_repeatable': bool(same)}
    for a in arms:
        steps = int(ref[a].steps.sum().item())
        med = float(np.median(ms[a]))
        out[a] = {'ms': [round(x, 2) for x in ms[a]], 'ms_median': round(med, 2), 'executed_env_steps': steps,
                  'ns_per_executed_step': round(med * 1e6 / steps, 4)}
    for a in ('incremental', 'symmetric'):
        out[a + '_over_attitude_ns_per_step'] = out[a]['ns_per_executed_step'] / out['attitude']['ns_per_executed_step']
    print(json.dumps(out))


if __name__ == '__main__':
    main()
