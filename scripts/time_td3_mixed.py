"""Time K7's mixed-shape group launch (serl_td3_learn with learners of different shapes) and a mixed-shape sweep.

(a) Eight learners at batch 86, CAPS on, on a replay of 800,000 K1 flight rows, cluster size 8: the shapes (72, 3, tanh),
    (96, 3, relu), (32, 3, tanh) and (256, 3, tanh), two of each.  Three arms, alternated: ONE mixed launch, one uniform
    group launch per shape in sequence (the best one process could do before), and the per-shape group launches on a
    stream each.  Then each hidden class inside the mixed kernel against its own uniform group kernel: the class's
    learners take `steps` steps and the other class's learners one step (which forces td3_mixed_kernel), against the
    class's learners alone (td3_group_kernel of that class).
(b) SERL10-sized runs (pop 10 x 3 envs, fused_td3) of the same four shapes: seconds per generation of ONE mixed Sweep
    against one Sweep per shape run one after another, and the mixed Sweep's population phase (its deferred population
    launches, host clock around a device synchronise) with the per-group streams against all groups on one stream.  The
    first generation is a warm-up (it also fills the replay past learn_start).
CUDA events / a synchronised host clock after warm-up.  Prints one JSON line with the card's name and power limit.

    python scripts/time_td3_mixed.py [--steps 300] [--gens 2] [--no-sweep]
"""
import argparse
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
from serl_b200.td3_fused import FusedTD3  # noqa: E402
from time_td3 import fill_replay, learner_args, timed  # noqa: E402
from time_td3_group import serl10_params  # noqa: E402

SHAPES = [(72, 3, 'tanh'), (96, 3, 'relu'), (32, 3, 'tanh'), (256, 3, 'tanh')]


def learners(dev):
    """two learners of each shape, in shape order"""
    out = []
    for k, (h, L, act) in enumerate(s for s in SHAPES for _ in range(2)):
        a = learner_args(dev)
        a.hidden_size, a.num_layers, a.activation_actor, a.seed = h, L, act, 7 + k
        torch.manual_seed(7 + k)
        out.append(FusedTD3(a, cluster_size=8, seed=7 + k))
    return out


def time_k7(dev, mem, steps, warmup, reps):
    fs = learners(dev)
    by_shape = [fs[2 * i:2 * i + 2] for i in range(len(SHAPES))]
    narrow, wide = [f for f in fs if f.shape.hidden <= 128], [f for f in fs if f.shape.hidden > 128]
    streams = [torch.cuda.Stream(dev) for _ in SHAPES]

    def group(part, ns, mixed=True):
        td3_fused.train_group(part, [mem] * len(part), ns, [f.critic_steps + 1 for f in part], [False] * len(part),
                              mixed_shapes=mixed)

    def mixed(n):
        group(fs, [n] * len(fs))

    def sequential(n):
        for part in by_shape:
            group(part, [n] * len(part), mixed=False)

    def streamed(n):
        cur = torch.cuda.current_stream(dev)
        for s in streams:
            s.wait_stream(cur)
        for part, s in zip(by_shape, streams):
            with torch.cuda.stream(s):
                group(part, [n] * len(part), mixed=False)
        for s in streams:
            cur.wait_stream(s)

    def in_mixed(cls, other):
        return lambda n: group(cls + other, [n] * len(cls) + [1] * len(other))

    def uniform(cls):
        return lambda n: group(cls, [n] * len(cls))

    arms = {'mixed': mixed, 'sequential': sequential, 'streams': streamed,
            'narrow_in_mixed': in_mixed(narrow, wide), 'narrow_uniform': uniform(narrow),
            'wide_in_mixed': in_mixed(wide, narrow), 'wide_uniform': uniform(wide)}
    for fn in arms.values():
        fn(warmup)
    res = {k: [] for k in arms}
    for _ in range(reps):
        for name, fn in arms.items():
            res[name].append(round(timed(lambda: fn(steps)) / steps, 1))
    for f in fs:
        f.status.zero_()
        f.run(mem.data, len(mem), 5, f.critic_steps + 1, False).check()
    return {'us_per_step': res, 'best_us_per_step': {k: min(v) for k, v in res.items()},
            'learners': [[f.shape.hidden, f.shape.num_layers, f.args.activation_actor] for f in fs]}


def sweep_runs(tmp, shapes, seed0=7):
    from serl_b200.envs import config
    runs = []
    for k, (h, L, act) in enumerate(shapes):
        p = serl10_params(seed0 + k, tmp)
        p.hidden_size, p.num_layers, p.activation_actor = h, L, act
        runs.append((p, config.select_env('PHlab_attitude_nominal')))
    return runs


def generation(sw, pop_times=None):
    """one Sweep generation in seconds (synchronised host clock); with `pop_times`, the population phase is timed too"""
    if pop_times is not None:
        launch = type(sw)._launch_populations

        def timed_launch(fronts):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            launch(sw, fronts)
            torch.cuda.synchronize()
            pop_times.append(time.perf_counter() - t0)
        sw._launch_populations = timed_launch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    stats = sw.train()
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    sw.__dict__.pop('_launch_populations', None)
    assert all(s is not None for s in stats)
    return dt


def time_sweeps(gens):
    from serl_b200.sweep import Sweep
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        sw = Sweep(sweep_runs(tmp, SHAPES), mixed_shapes=True)
        generation(sw)                                          # warm-up, fills the replays
        dev = sw.runs[0].agent.device
        many = list(sw._streams)
        one = [torch.cuda.current_stream(dev)] * len(many)      # every launch group on the current stream
        per_gen, pop = {'streams': [], 'one_stream': []}, {'streams': [], 'one_stream': []}
        for _ in range(gens):
            for name, st in (('streams', many), ('one_stream', one)):
                sw._streams = st
                t = []
                per_gen[name].append(round(generation(sw, t), 3))
                pop[name].append(round(sum(t), 4))
        sw._streams = many
        out['mixed_sweep'] = {'s_per_generation': per_gen, 'population_phase_s': pop,
                              'rl_steps_per_run': [r.agent.rl_iteration for r in sw.runs]}
        del sw
        torch.cuda.empty_cache()
        alone = {}
        for k, shape in enumerate(SHAPES):
            s1 = Sweep(sweep_runs(tmp, [shape], seed0=7 + k))
            generation(s1)
            alone['%d,%d,%s' % shape] = [round(generation(s1), 3) for _ in range(gens)]
            del s1
            torch.cuda.empty_cache()
        out['one_sweep_per_shape'] = {'s_per_generation': alone,
                                      'sum_s': round(sum(min(v) for v in alone.values()), 3)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=300)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--gens', type=int, default=2, help='timed generations per sweep arm')
    ap.add_argument('--no-sweep', action='store_true')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_td3_mixed.py measures on the GPU; no CUDA device found')
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    mem = fill_replay(dev)
    out = {'card': q, 'replay_rows': len(mem), 'steps': a.steps, 'batch': 86, 'cluster_size': 8,
           'shapes': [list(s) for s in SHAPES], 'k7': time_k7(dev, mem, a.steps, a.warmup, a.reps)}
    del mem
    torch.cuda.empty_cache()
    if not a.no_sweep:
        out['sweep'] = time_sweeps(a.gens)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
