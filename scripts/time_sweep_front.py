"""Time the population rollouts of a Sweep, merged into one launch per launch group against one launch per run.

(a) A Sweep of S SERL10-shaped runs (pop 10, 3 envs, h = 72, fused_td3) for S = 1, 4, 8, 16: seconds per sweep generation
    (the first generation is a warm-up that also fills the replay past learn_start; the second is timed), and the
    population-rollout part of the heads on its own: every run's population drawn, launched and waited for (one merged
    launch per group here, one launch per run in a tree without launch_population_group), best and median of 5.
    Each S runs in a fresh process per tree, this tree and --parent alternated, so both arms see the same card state.
(b) The config-3-shaped population (pop 512 x 128 envs, h = 72, SERL10 genomes tiled with N(0, 1e-3) noise) on per-actor
    env blocks (512 x 128 distinct reference rows) against the shared 128 rows, alternated, best and median of 5 launches.
A synchronised host clock after warm-up.  Prints one JSON line with the card's name and power limit, read in the same call.

    python scripts/time_sweep_front.py [--parent DIR] [--sizes 1,4,8,16]

--parent: a built tree of the commit to compare against (its own serl_b200 package and libserl_b200.so).
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def launch_populations(sw):
    """draw and launch every run's population the way the tree's Sweep does (merged per group, or one launch per run)"""
    from serl_b200.core import agent as agent_mod
    from serl_b200 import sweep as sweep_mod
    keep = []
    if hasattr(agent_mod, 'launch_population_group'):
        fronts = []
        for r in sw.runs:
            with sweep_mod.rng_scope(r.rng):
                fronts.append(types.SimpleNamespace(pop_draws=r.agent._draw_population(), sm_limit=-3, pop=None))
        keys = [agent_mod.population_key(r.params, r.env) for r in sw.runs]
        for g in sweep_mod.launch_groups(keys):
            agent_mod.launch_population_group([(sw.runs[i].agent, fronts[i]) for i in g])
        keep = fronts
    else:
        for r in sw.runs:
            with sweep_mod.rng_scope(r.rng):
                keep.append(r.agent._launch_population(sm_limit=-3))
    return keep


def worker(S):
    import tempfile
    import torch
    from serl_b200.envs import config
    from serl_b200.sweep import Sweep
    with tempfile.TemporaryDirectory() as tmp:
        sw = Sweep([(serl10_params(7 + i, tmp), config.select_env('PHlab_attitude_nominal')) for i in range(S)])
        sw.train()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        stats = sw.train()
        torch.cuda.synchronize()
        gen = time.perf_counter() - t0
        assert all(s is not None for s in stats) and min(r.agent.rl_iteration for r in sw.runs) > 0
        launch_populations(sw)
        torch.cuda.synchronize()
        pops = []
        for _ in range(5):
            t0 = time.perf_counter()
            keep = launch_populations(sw)
            torch.cuda.synchronize()
            pops.append(time.perf_counter() - t0)
            del keep
    pops.sort()
    return {'s_per_generation': round(gen, 3), 'population_s_best': round(pops[0], 4), 'population_s_median': round(pops[2], 4)}


def config3():
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    from bench import population
    from oracle import refsig
    from serl_b200 import rollout
    dev = torch.device('cuda:0')
    pop, n_envs = 512, 128
    g = torch.as_tensor(population(pop), device=dev)
    sh = rollout.actor_shape(72)
    lv, st = refsig.make_ref_params(pop * n_envs)
    md = torch.full((pop, n_envs), rollout.mode_code('nominal'), dtype=torch.int32, device=dev)
    arms = {
        'shared': (torch.as_tensor(lv[:n_envs], device=dev), torch.as_tensor(st[:n_envs], device=dev), md[0].contiguous()),
        'per_actor': (torch.as_tensor(lv.reshape(pop, n_envs, 2, 6), device=dev), torch.as_tensor(st.reshape(pop, n_envs, 2, 6), device=dev), md),
    }
    res = {k: [] for k in arms}
    steps = {}
    for k, a in arms.items():
        rollout.population_rollout(g, sh, *a).check()
    for _ in range(5):
        for k, a in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = rollout.population_rollout(g, sh, *a)
            torch.cuda.synchronize()
            res[k].append(time.perf_counter() - t0)
            r.check()
            steps[k] = int(r.steps.sum())
    out = {}
    for k, v in res.items():
        v.sort()
        out[k] = {'s_best': round(v[0], 4), 's_median': round(v[2], 4), 'env_steps': steps[k]}
    out['ref_row_bytes'] = {'shared': n_envs * 2 * 2 * 6 * 8, 'per_actor': pop * n_envs * 2 * 2 * 6 * 8}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--parent', default=None, help='built tree of the commit to compare against')
    ap.add_argument('--sizes', default='1,4,8,16')
    ap.add_argument('--worker', type=int, default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker is not None:
        sys.path.insert(0, os.getcwd())
        print(json.dumps(worker(a.worker)))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('time_sweep_front.py measures on the GPU; no CUDA device found')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    trees = {'this': ROOT}
    if a.parent:
        trees['parent'] = os.path.abspath(a.parent)
    out = {'card': q, 'sweep': {}}
    for S in [int(s) for s in a.sizes.split(',') if s]:
        out['sweep'][S] = {}
        for name, tree in trees.items():
            r = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', str(S)], cwd=tree, capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit('worker S=%d (%s) failed:\n%s' % (S, name, r.stderr[-4000:]))
            out['sweep'][S][name] = json.loads(r.stdout.strip().splitlines()[-1])
            print('S = %d %s: %s' % (S, name, out['sweep'][S][name]), file=sys.stderr, flush=True)
    sys.path.insert(0, ROOT)
    out['config3_refs'] = config3()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
