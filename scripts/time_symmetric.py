"""K1 flying symmetric control (SERL_ROLLOUT_SYMMETRIC: the elevator alone, obs = [e_theta, q]) against attitude control, on a
config-3-shaped population: pop 512 x 128 nominal envs x 2001 steps, h = 72.  The symmetric genomes take the hidden layers of
the bench's trained population, the first two input columns of its layer 0 (its theta error and p) and the first row of its
output layer, so the two arms share those weights.  Two workloads:
  trained    the populations as they are.  Their episodes end at different steps, and a warp runs until its last lane is
             done, so the time per executed step counts the idle lanes too.
  held_trim  the same genomes with a zero output layer: both arms command zero and every trajectory flies all 2001 steps,
             so the two launch times compare the same number of steps (the actor still computes every layer).
The arms alternate, `rounds` times each, in one process; every launch is timed with CUDA events after a warm-up launch of
both, and each arm must reproduce its warm-up bits.  Prints one JSON object with the card, its power limit and its clocks.
usage: python scripts/time_symmetric.py [rounds=3]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                    # noqa: E402  (the bench's trained population)
from serl_b200 import rollout, refsig           # noqa: E402

rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
dev = torch.device('cuda:0')


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm,clocks.mem'
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', '0'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def narrow(w, h):
    """[pop, P(7 -> 3)] -> [pop, P(2 -> 1)]: layer 0's first two input columns, the hidden layers, the output layer's first row"""
    n = w.shape[0]
    w0 = w[:, :7 * h].reshape(n, h, 7)[:, :, :2].reshape(n, -1)
    mid = w[:, 7 * h:w.shape[1] - (3 * h + 3)]
    wo = w[:, w.shape[1] - (3 * h + 3):w.shape[1] - (3 * h + 3) + h]
    bo = w[:, -3:-2]
    return np.ascontiguousarray(np.concatenate([w0, mid, wo, bo], axis=1))


def measure(h, pop, md):
    sym = narrow(pop, h)
    att_refs = [torch.as_tensor(x, device=dev) for x in refsig.make_ref_params(bench.N_ENVS)]
    sym_refs = [torch.as_tensor(x, device=dev) for x in refsig.make_ref_params(bench.N_ENVS, symmetric=True)]
    arms = {'attitude': (rollout.actor_shape(h, 3, 'tanh'), torch.from_numpy(pop).to(dev), att_refs),
            'symmetric': (rollout.actor_shape(h, 3, 'tanh', state_dim=2, action_dim=1), torch.from_numpy(sym).to(dev), sym_refs)}
    assert sym.shape[1] == rollout.num_params(arms['symmetric'][0])
    run = lambda arm: rollout.population_rollout(arms[arm][1], arms[arm][0], *arms[arm][2], md, horizon=bench.HORIZON)
    ref = {a: run(a) for a in arms}                            # warm-up, and the bits every timed launch reproduces
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
            same = same and torch.equal(r.returns, ref[a].returns) and torch.equal(r.steps, ref[a].steps)
    out = {'bitwise_repeatable': bool(same)}
    for a in arms:
        steps = int(ref[a].steps.sum().item())
        med = float(np.median(ms[a]))
        out[a] = {'ms': [round(x, 2) for x in ms[a]], 'ms_median': round(med, 2), 'executed_env_steps': steps,
                  'ns_per_executed_step': round(med * 1e6 / steps, 4)}
    out['symmetric_over_attitude_ns_per_step'] = out['symmetric']['ns_per_executed_step'] / out['attitude']['ns_per_executed_step']
    return out


def main():
    h = bench.HIDDEN
    pop = bench.population(bench.POP)
    trim = pop.copy()
    trim[:, -(3 * h + 3):] = 0.0                               # output layer Wo [3, h], bo [3]
    md = torch.full((bench.N_ENVS,), rollout.mode_code('nominal'), dtype=torch.int32, device=dev)
    out = {'card: name, power limit, sm clock, max sm clock, mem clock': card(), 'rounds': rounds, 'pop': bench.POP,
           'n_envs': bench.N_ENVS, 'horizon': bench.HORIZON, 'hidden': h}
    for name, w in (('trained', pop), ('held_trim', trim)):
        out[name] = measure(h, w, md)
        print(name, json.dumps(out[name]), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
