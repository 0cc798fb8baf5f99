"""Time checkpoint and resume (serl_b200/checkpoint.py) next to the generation they interrupt.

For each configuration: `--gens` generations of the run (the first fills the replay past learn_start; the last is timed as
the generation time), then a save (checkpoint size, and its time: the wait for the queued front, the device->host copies,
torch.save, fsync and rename), the uninterrupted run's next generation, then a fresh Agent / Sweep built from the same
Parameters, and load + its first train() (the same generation) timed together.  Configurations:
  serl10  pop 10 x 3 envs, h = 72, 800,000-row buffer, fused_td3;
  serl50  the same with pop 50;
  sweep8  a Sweep of 8 serl10 runs (seeds 7..14).
A synchronised host clock (save and load synchronise the device; train() ends in host reads of its results).  Prints one
JSON line with the card's name and power limit, read in the same call.

    python scripts/time_checkpoint.py [--configs serl10,serl50,sweep8] [--gens 2] [--dir DIR]
"""
import argparse
import json
import os
import random
import shutil
import subprocess
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from serl_b200.core import agent as agent_mod  # noqa: E402
from serl_b200.envs import config  # noqa: E402
from serl_b200.parameters import Parameters  # noqa: E402
from serl_b200.sweep import Sweep  # noqa: E402


def serl(pop, seed=7):
    p = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=seed, pop_size=pop, mut_type='normal', fused_td3=True))
    env = config.select_env('PHlab_attitude_nominal')
    p.action_dim, p.state_dim = env.action_space.shape[0], env.observation_space.shape[0]
    assert p.buffer_size == 800_000 and p.hidden_size == 72 and p.num_envs == 3
    return p, env


def build(p, env):
    env.seed(p.seed)
    torch.manual_seed(p.seed)
    np.random.seed(p.seed)
    random.seed(p.seed)
    return agent_mod.Agent(p, env)


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def size(path):
    if os.path.isdir(path):
        return sum(os.path.getsize(os.path.join(path, f)) for f in os.listdir(path))
    return os.path.getsize(path)


def time_agent(pop, gens, folder):
    a = build(*serl(pop))
    for _ in range(gens - 1):
        a.train()
    t_gen, _ = clock(a.train)
    path = os.path.join(folder, 'serl%d.pt' % pop)
    t_save, _ = clock(lambda: a.save_checkpoint(path))
    frames, steps = a.num_frames, a.rl_agent.critic_steps
    t_next, _ = clock(a.train)
    del a
    torch.cuda.empty_cache()
    b = agent_mod.Agent(*serl(pop))
    t_load, _ = clock(lambda: b.load_checkpoint(path))
    t_first, _ = clock(b.train)
    del b
    torch.cuda.empty_cache()
    return {'generation_s': t_gen, 'save_s': t_save, 'bytes': size(path), 'next_generation_s': t_next, 'load_s': t_load,
            'load_plus_first_train_s': t_load + t_first, 'num_frames': frames, 'k7_steps': steps}


def time_sweep(n_runs, gens, folder):
    runs = lambda: Sweep([serl(10, seed=7 + i) for i in range(n_runs)], mixed_shapes=True)
    s = runs()
    for _ in range(gens - 1):
        s.train()
    t_gen, _ = clock(s.train)
    path = os.path.join(folder, 'sweep%d' % n_runs)
    t_save, _ = clock(lambda: s.save_checkpoint(path))
    t_next, _ = clock(s.train)
    del s
    torch.cuda.empty_cache()
    s = runs()
    t_load, _ = clock(lambda: s.load_checkpoint(path))
    t_first, _ = clock(s.train)
    del s
    torch.cuda.empty_cache()
    return {'generation_s': t_gen, 'save_s': t_save, 'bytes': size(path), 'next_generation_s': t_next, 'load_s': t_load,
            'load_plus_first_train_s': t_load + t_first, 'runs': n_runs}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--configs', default='serl10,serl50,sweep8')
    ap.add_argument('--gens', type=int, default=2, help='generations before the save; the last is timed')
    ap.add_argument('--dir', default=None, help='where the checkpoints go (default: a temporary directory, removed after)')
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_checkpoint.py measures on the GPU; no CUDA device found')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    folder = a.dir or tempfile.mkdtemp(prefix='serl_ckpt_')
    work = tempfile.mkdtemp(prefix='serl_ckpt_cwd_')
    os.chdir(work)                                  # Parameters makes ./tmp/
    out = {'card': q, 'gens': a.gens}
    try:
        for c in a.configs.split(','):
            if c.startswith('sweep'):
                out[c] = time_sweep(int(c[5:]), a.gens, folder)
            else:
                out[c] = time_agent(int(c[4:]), a.gens, folder)
            print(c, json.dumps(out[c]), file=sys.stderr, flush=True)
    finally:
        if a.dir is None:
            shutil.rmtree(folder, ignore_errors=True)
        shutil.rmtree(work, ignore_errors=True)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
