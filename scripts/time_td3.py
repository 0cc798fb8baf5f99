"""Time the RL half's gradient steps: (a) today's torch loop (DeviceReplayMemory.sample + TD3.update_parameters, as
Agent.train_rl runs it), (b) K7 (the fused learner, csrc/td3.cu) per cluster size, (c) K7 over SERL10's per-generation step
count.  h = 72, L = 3, batch 86, CAPS on, a replay of 800,000 rows from K1 flights.  CUDA events after warm-up; (a) and (b)
alternate twice.  Prints one JSON line with the card's name and power limit.

    python scripts/time_td3.py [--steps 3000]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from serl_b200 import refsig, rollout  # noqa: E402
from serl_b200.core.replay_memory import DeviceReplayMemory  # noqa: E402
from serl_b200.core.td3 import TD3  # noqa: E402
from serl_b200.td3_fused import FusedTD3  # noqa: E402

SERL10_STEPS = 22_011          # frames stored in one SERL10 generation (pop 10 x 2001 + the exploration episode)


def learner_args(dev):
    return types.SimpleNamespace(device=dev, individual_bs=10_000, hidden_size=72, num_layers=3, activation_actor='tanh',
                                 state_dim=7, action_dim=3, lr=0.00018643512599969097, gamma=0.98, tau=0.005,
                                 noise_sd=0.2962183114680794, noise_clip=0.5, policy_update_freq=3, use_caps=True,
                                 batch_size=86, seed=7)


def fill_replay(dev, n=800_000, pop=400):
    """n replay rows from K1 flights of `pop` perturbed SERL10-like actors"""
    import bench
    mem = DeviceReplayMemory(n, dev, seed=7)
    w = torch.from_numpy(bench.population(pop)).to(dev)
    md = torch.zeros(1, dtype=torch.int32, device=dev)
    seed = 0
    while len(mem) < n:
        lv, st = refsig.make_ref_params(1, seed_base=7_000_000 + seed)
        r = rollout.population_rollout(w, rollout.actor_shape(72), torch.as_tensor(lv, device=dev), torch.as_tensor(st, device=dev), md,
                                       replay_env=0)
        sel = torch.arange(r.replay.shape[1], device=dev)[None, :] < r.steps[:, :1]
        mem.add_rows(r.replay[sel])
        seed += 1
    return mem


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3          # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=3000)
    ap.add_argument('--warmup', type=int, default=300)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_td3.py measures on the GPU; no CUDA device found')
    dev = torch.device('cuda:0')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    mem = fill_replay(dev)
    args = learner_args(dev)
    torch.manual_seed(7)
    ref = TD3(args)
    fused = FusedTD3(args)
    it = [0]

    def torch_loop(n):
        for _ in range(n):
            it[0] += 1
            ref.update_parameters(mem.sample(args.batch_size), it[0], False)

    def k7(n, cs):
        fused.run(mem.data, len(mem), n, fused.critic_steps + 1, False, cluster_size=cs)

    torch_loop(a.warmup)
    for cs in (1, 2, 4, 8):
        k7(a.warmup, cs)
    res = {'torch_us_per_step': [], 'k7_us_per_step': {cs: [] for cs in (1, 2, 4, 8)}}
    for _ in range(2):
        res['torch_us_per_step'].append(timed(lambda: torch_loop(a.steps)) / a.steps)
        for cs in (1, 2, 4, 8):
            res['k7_us_per_step'][cs].append(timed(lambda: k7(a.steps, cs)) / a.steps)
    best = min((1, 2, 4, 8), key=lambda cs: min(res['k7_us_per_step'][cs]))
    gen = {cs: timed(lambda: k7(SERL10_STEPS, cs)) / 1e3 for cs in sorted({best, 0})}
    fused.status.zero_()
    st = fused.run(mem.data, len(mem), 10, fused.critic_steps + 1, False)
    st.check()
    out = {'card': q, 'replay_rows': len(mem), 'steps': a.steps, 'batch': args.batch_size, 'hidden': 72, 'num_layers': 3,
           'a_torch_us_per_step': [round(x, 1) for x in res['torch_us_per_step']],
           'b_k7_us_per_step': {str(cs): [round(x, 2) for x in v] for cs, v in res['k7_us_per_step'].items()},
           'c_k7_serl10_generation_ms': {('default' if cs == 0 else str(cs)): round(v, 2) for cs, v in gen.items()},
           'c_steps': SERL10_STEPS}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
