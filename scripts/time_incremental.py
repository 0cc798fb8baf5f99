"""K1 flying incremental control (SERL_ROLLOUT_INCREMENTAL: rate commands integrated into the deflection, a 10-entry
observation) against the absolute mode, on a config-3-shaped population: pop 512 x 128 nominal envs x 2001 steps, h = 72.
The incremental genomes are the bench's trained population with three zero input columns for last_u, so the two arms share
every other weight.  Two workloads:
  trained    the population as it is.  A rate command is not a deflection: the incremental arm's episodes end early, and a
             warp runs until its last lane is done, so its time per executed step counts the idle lanes too.
  held_trim  the same genomes with a zero output layer: both arms command zero and every trajectory flies all 2001 steps,
             so the two launch times compare the same work (the actor still computes every layer).
  h256_k1tc_held_trim  the same held trim for randomly initialised actors of h = 256, L = 3, which fly on K1-TC
             (serl_actor_tc_widths: [256] * 4).
The arms alternate, `rounds` times each, in one process; every launch is timed with CUDA events after a warm-up launch of
both, and each arm must reproduce its warm-up bits.  Prints one JSON object with the card, its power limit and its clocks.
usage: python scripts/time_incremental.py [rounds=3]"""
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                    # noqa: E402  (the bench's trained population)
from serl_b200 import rollout, refsig           # noqa: E402
from serl_b200.core import genetic_agent        # noqa: E402

rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 3
dev = torch.device('cuda:0')


def card():
    q = 'name,power.limit,clocks.sm,clocks.max.sm,clocks.mem'
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', '0'], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def widen(w, h):
    """[pop, P(7)] -> [pop, P(10)]: the first layer's rows [h, 7] get three zero columns (the last_u inputs)"""
    w0 = w[:, :7 * h].reshape(-1, h, 7)
    w0 = np.concatenate([w0, np.zeros((w.shape[0], h, 3), dtype=np.float32)], axis=2).reshape(w.shape[0], -1)
    return np.ascontiguousarray(np.concatenate([w0, w[:, 7 * h:]], axis=1))


def measure(h, pop, lv, st, md):
    arms = {'absolute': (rollout.actor_shape(h, 3, 'tanh'), torch.from_numpy(pop).to(dev)),
            'incremental': (rollout.actor_shape(h, 3, 'tanh', state_dim=10), torch.from_numpy(widen(pop, h)).to(dev))}
    run = lambda arm: rollout.population_rollout(arms[arm][1], arms[arm][0], lv, st, md, horizon=bench.HORIZON)
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
    out['incremental_over_absolute_ns_per_step'] = out['incremental']['ns_per_executed_step'] / out['absolute']['ns_per_executed_step']
    return out


def main():
    h = bench.HIDDEN
    pop = bench.population(bench.POP)
    trim = pop.copy()
    trim[:, -(3 * h + 3):] = 0.0                               # output layer Wo [3, h], bo [3]
    lv, st = (torch.as_tensor(x, device=dev) for x in refsig.make_ref_params(bench.N_ENVS))
    md = torch.full((bench.N_ENVS,), rollout.mode_code('nominal'), dtype=torch.int32, device=dev)
    out = {'card: name, power limit, sm clock, max sm clock, mem clock': card(), 'rounds': rounds, 'pop': bench.POP,
           'n_envs': bench.N_ENVS, 'horizon': bench.HORIZON, 'hidden': h}
    torch.manual_seed(7)
    ns = types.SimpleNamespace(hidden_size=256, num_layers=3, activation_actor='tanh', state_dim=7, action_dim=3)
    wide = torch.stack([genetic_agent.Actor(ns).flat().detach() for _ in range(bench.POP)]).numpy()
    wide[:, -(3 * 256 + 3):] = 0.0
    for name, hh, w in (('trained', h, pop), ('held_trim', h, trim), ('h256_k1tc_held_trim', 256, wide)):
        out[name] = measure(hh, w, lv, st, md)
        print(name, json.dumps(out[name]), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
