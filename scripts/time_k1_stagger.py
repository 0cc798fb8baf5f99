"""K1 with its two genome slots per CTA in lockstep against staggered by half a step (serl_rollout_desc.flags
SERL_ROLLOUT_STAGGER), on the bench's K1 workloads: BASELINE config 3 (pop 512 x 128 nominal envs), config 4 (the same
population on mixed fault / plant modes), config 2 (pop 50 x 64 envs), pop 64 x 128 envs and a random-init population.
The two schedules alternate, `rounds` times each, in one process; every launch is timed with CUDA events after a warm-up
launch of both, and returns and steps must be bitwise equal between the two.  Launches of one slot per CTA (config 2,
pop 64) run the same kernel either way: their two columns measure the run-to-run spread.  Prints one JSON object with the
card, its power limit and its clocks.
usage: python scripts/time_k1_stagger.py [rounds=3]"""
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                    # noqa: E402  (the bench's populations and mode mix)
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


def workloads():
    sh = rollout.actor_shape(bench.HIDDEN, 3, 'tanh')
    lv, st = (torch.as_tensor(x, device=dev) for x in refsig.make_ref_params(bench.N_ENVS))
    nominal = torch.full((bench.N_ENVS,), rollout.mode_code('nominal'), dtype=torch.int32, device=dev)
    mixed = torch.tensor([rollout.mode_code(m) for m in bench.mixed_modes(bench.N_ENVS)], dtype=torch.int32, device=dev)
    w = torch.from_numpy(bench.population(bench.POP)).to(dev)
    torch.manual_seed(7)
    a_ns = types.SimpleNamespace(hidden_size=bench.HIDDEN, num_layers=3, activation_actor='tanh', state_dim=7, action_dim=3)
    w0 = torch.stack([genetic_agent.Actor(a_ns).flat() for _ in range(bench.POP)]).to(dev)
    lv2, st2 = (torch.as_tensor(x, device=dev) for x in refsig.make_ref_params(64))
    return sh, {
        'config3_pop512_128envs': (w, lv, st, nominal, rollout.variant_sorted_order(nominal)),
        'config4_pop512_128envs_mixed': (w, lv, st, mixed, rollout.variant_sorted_order(mixed)),
        'config2_pop50_64envs': (torch.from_numpy(bench.population(50)).to(dev), lv2, st2, nominal[:64].contiguous(), None),
        'pop64_128envs': (w[:64].contiguous(), lv, st, nominal, None),
        'random_init_pop512_128envs': (w0, lv, st, nominal, None),
    }


def main():
    sh, wls = workloads()
    out = {'card: name, power limit, sm clock, max sm clock, mem clock': card(), 'rounds': rounds, 'horizon': bench.HORIZON}
    for name, (w, lv, st, md, order) in wls.items():
        run = lambda stagger: rollout.population_rollout(w, sh, lv, st, md, horizon=bench.HORIZON, env_order=order, stagger=stagger)
        ref = {m: run(m) for m in (False, True)}               # warm-up, and the results both schedules must reproduce
        torch.cuda.synchronize()
        same = torch.equal(ref[False].returns, ref[True].returns) and torch.equal(ref[False].steps, ref[True].steps)
        ms = {False: [], True: []}
        for _ in range(rounds):
            for m in (False, True):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                r = run(m)
                e1.record()
                torch.cuda.synchronize()
                r.check()
                ms[m].append(e0.elapsed_time(e1))
                same = same and torch.equal(r.returns, ref[m].returns) and torch.equal(r.steps, ref[m].steps)
        steps = int(ref[False].steps.sum().item())
        out[name] = {'executed_env_steps': steps, 'lockstep_ms': [round(x, 2) for x in ms[False]],
                     'stagger_ms': [round(x, 2) for x in ms[True]],
                     'lockstep_over_stagger_median': float(np.median(ms[False]) / np.median(ms[True])),
                     'lockstep_env_steps_per_sec_median': steps / (np.median(ms[False]) * 1e-3),
                     'bitwise_equal': bool(same)}
        print(name, json.dumps(out[name]), file=sys.stderr, flush=True)
    out['card after'] = card()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
