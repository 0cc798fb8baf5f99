"""Time K7 (csrc/td3.cu) on actors wider than 128, where the actor's hidden blocks run as tiled phases, next to the torch
loop (DeviceReplayMemory.sample + TD3.update_parameters, as Agent.train_rl runs it) on the same shape.  Settings of
scripts/time_td3.py: batch 86, CAPS on, a replay of 800,000 rows from K1 flights, CUDA events after warm-up, the arms
alternated twice.  Arms: the torch loop at h = 256, L = 3; K7 at h = 256, L = 3 per cluster size; K7 at h = 320, L = 8;
K7 at h = 128, L = 3 (the untiled kernel) next to h = 129, L = 3 (the tiled one); one SERL10 generation (22,011 steps) at
h = 256.  Each arm's fp32 FLOP per step is counted from the shapes (a multiply-add is 2 FLOP; LayerNorm, activations and
Adam left out) and set against the fp32 peak of the SMs it runs on (CS SMs x 128 lanes x 2 FLOP x the SM clock read while
K7 runs).  Prints one JSON line with the card's name and power limit.

    python scripts/time_td3_wide.py [--steps 1000] [--torch-steps 200]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'scripts'))

from serl_b200.core.td3 import TD3  # noqa: E402
from serl_b200.td3_fused import FusedTD3  # noqa: E402
from time_td3 import SERL10_STEPS, fill_replay, learner_args, timed  # noqa: E402

CH, CI, SD, AD = 64, 10, 7, 3


def flop_per_step(h, L, B, caps=True, freq=3):
    """fp32 FLOP of one gradient step, averaged over critic-only and actor iterations"""
    actor = SD * h + L * h * h + h * AD                   # multiply-adds per row through the actor
    critic = CI * CH + CH * CH + CH                       # per row and head
    R = 2 * B if caps else B
    critic_step = B * actor + 2 * B * critic * 4          # target actor; target critic, critic forward, critic backward (x 2)
    actor_step = R * actor * 3 + B * critic * 2           # actor forward + backward (x 2); Q1 forward + input gradient
    return 2 * (critic_step + actor_step / freq)


def smi(query):
    return subprocess.run(['nvidia-smi', '--query-gpu=' + query, '--format=csv,noheader,nounits', '-i', '0'],
                          capture_output=True, text=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=1000)
    ap.add_argument('--torch-steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=100)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_td3_wide.py measures on the GPU; no CUDA device found')
    dev = torch.device('cuda:0')
    card = smi('name,power.limit')
    mem = fill_replay(dev)

    def learner(h, L, cls):
        args = learner_args(dev)
        args.hidden_size, args.num_layers = h, L
        torch.manual_seed(7)
        return args, cls(args)

    targs, ref = learner(256, 3, TD3)
    it = [0]

    def torch_loop(n):
        for _ in range(n):
            it[0] += 1
            ref.update_parameters(mem.sample(targs.batch_size), it[0], False)

    k7 = {(256, 3): learner(256, 3, FusedTD3)[1], (320, 8): learner(320, 8, FusedTD3)[1],
          (128, 3): learner(128, 3, FusedTD3)[1], (129, 3): learner(129, 3, FusedTD3)[1]}

    def run(key, n, cs):
        f = k7[key]
        return f.run(mem.data, len(mem), n, f.critic_steps + 1, False, cluster_size=cs)

    arms = [('k7_h256_L3_cs%d' % cs, (256, 3), cs) for cs in (1, 2, 4, 8)]
    arms += [('k7_h320_L8_cs8', (320, 8), 8), ('k7_h128_L3_cs8', (128, 3), 8), ('k7_h129_L3_cs8', (129, 3), 8)]
    torch_loop(a.warmup)
    for _, key, cs in arms:
        run(key, a.warmup, cs)
    res = {'torch_h256_L3': []}
    res.update({name: [] for name, _, _ in arms})
    for _ in range(2):
        res['torch_h256_L3'].append(timed(lambda: torch_loop(a.torch_steps)) / a.torch_steps)
        for name, key, cs in arms:
            res[name].append(timed(lambda: run(key, a.steps, cs)) / a.steps)
    # the SM clock while K7 runs (the launch returns at once; nvidia-smi reads the clock during the kernel)
    torch.cuda.synchronize()
    run((256, 3), 4 * a.steps, 8)
    clock_mhz = float(smi('clocks.sm'))
    torch.cuda.synchronize()
    gen_ms = timed(lambda: run((256, 3), SERL10_STEPS, 0)) / 1e3
    for f in k7.values():
        f.status.zero_()
        f.run(mem.data, len(mem), 10, f.critic_steps + 1, False).check()

    shapes = {'torch_h256_L3': (256, 3, None)}
    shapes.update({name: key + (cs,) for name, key, cs in arms})
    out = {'card': card, 'sm_clock_mhz_under_k7': clock_mhz, 'max_sm_clock_mhz': float(smi('clocks.max.sm')),
           'replay_rows': len(mem), 'batch': targs.batch_size, 'caps': True, 'k7_steps': a.steps, 'torch_steps': a.torch_steps,
           'us_per_step': {k: [round(x, 2) for x in v] for k, v in res.items()}, 'mflop_per_step': {}, 'gflop_per_s': {},
           'share_of_cs_sm_fp32_peak': {}}
    for name, (h, L, cs) in shapes.items():
        flop = flop_per_step(h, L, targs.batch_size)
        rate = flop / (min(res[name]) * 1e-6)
        out['mflop_per_step'][name] = round(flop / 1e6, 2)
        out['gflop_per_s'][name] = round(rate / 1e9, 1)
        if name.startswith('k7'):                           # against the CS SMs the cluster runs on
            out['share_of_cs_sm_fp32_peak'][name] = round(rate / (cs * 128 * 2 * clock_mhz * 1e6), 4)
    best = min(min(res['k7_h256_L3_cs%d' % cs]) for cs in (1, 2, 4, 8))
    out['torch_over_k7_h256'] = round(min(res['torch_h256_L3']) / best, 1)
    out['k7_h256_serl10_generation_ms'] = round(gen_ms, 1)
    out['serl10_steps'] = SERL10_STEPS
    print(json.dumps(out))


if __name__ == '__main__':
    main()
