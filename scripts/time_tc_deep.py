"""K1-TC on deep width lists: env-steps/s of [128]*4, [256]*4 (the reference's Actor at h = 128 / 256, num_layers = 3) and
[400, 300]; K1 against K1-TC on the same h = 128, L = 3 population (the tensor-core vs warp-GEMV crossover at the
reference's own architecture); the achieved TF32 rate of the tensor-core layers.  CUDA events after a warm-up launch.
Prints one JSON object, with the card and its power limit.
usage: python scripts/time_tc_deep.py [pop=256] [n_envs=128] [horizon=2001]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from serl_b200 import rollout, refsig          # noqa: E402
from oracle import actor as A                  # noqa: E402

pop = int(sys.argv[1]) if len(sys.argv) > 1 else 256
n_envs = int(sys.argv[2]) if len(sys.argv) > 2 else 128
horizon = int(sys.argv[3]) if len(sys.argv) > 3 else 2001
dev = torch.device('cuda:0')
TF32_PEAK = 494.7e12          # H100 SXM data sheet, dense TF32 tensor-core FLOP/s (989.4e12 is with sparsity)


def power_limit():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return 'unknown'


def genomes(widths, n, seed=7, out_gain=0.2):
    """random-init actors with output gain 0.2, tiled + N(0, 1e-3) noise (scripts/bench_config5.py): full-horizon episodes"""
    torch.manual_seed(seed)
    base = []
    for _ in range(min(n, 16)):
        m = A.WideActor(widths)
        with torch.no_grad():
            m.net[-2].weight.mul_(out_gain)
            m.net[-2].bias.mul_(out_gain)
        base.append(A.flatten(m))
    base = np.stack(base)
    rs = np.random.RandomState(seed)
    w = base[np.arange(n) % base.shape[0]] + rs.normal(0, 1e-3, size=(n, base.shape[1])).astype(np.float32)
    return torch.from_numpy(np.ascontiguousarray(w.astype(np.float32))).to(dev)


lv, st = refsig.make_ref_params(n_envs)
lv, st = torch.as_tensor(lv, device=dev), torch.as_tensor(st, device=dev)
md = torch.zeros(n_envs, dtype=torch.int32, device=dev)
props = torch.cuda.get_device_properties(dev)
out = {'device': props.name, 'sms': props.multi_processor_count, 'power_limit_W,max_sm_clock': power_limit(), 'pop': pop,
       'n_envs': n_envs, 'horizon': horizon, 'population': 'random-init actors, output gain 0.2, tiled + N(0,1e-3) noise'}


def timed(name, w, shape, widths):
    rollout.population_rollout(w, shape, lv, st, md, horizon=min(horizon, 50), widths=widths)        # warm-up (layout, scratch)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    res = rollout.population_rollout(w, shape, lv, st, md, horizon=horizon, widths=widths)
    e1.record()
    torch.cuda.synchronize()
    res.check()
    ms = e0.elapsed_time(e1)
    steps = int(res.steps.sum().item())
    rec = {'ms': round(ms, 2), 'executed_env_steps': steps, 'env_steps_per_sec': steps / (ms * 1e-3),
           'mean_episode_steps': steps / (pop * n_envs)}
    wl = widths or [shape.hidden] * (shape.num_layers + 1)
    if widths:
        # layers 1..n-1 on the tensor cores, three TF32 products per multiply-add (3xTF32); the padded work the kernel issues
        # (64-column accumulator blocks, K padded to 8) and the weight tiles it streams per step of 128 envs (both halves)
        macs = sum(a * b for a, b in zip(wl[:-1], wl[1:]))
        pad = lambda x, m: (x + m - 1) // m * m
        macs_pad = sum(pad(a, 8) * pad(b, 64) for a, b in zip(wl[:-1], wl[1:]))
        rate = 2 * 3 * macs * steps / (ms * 1e-3)
        rec.update({'tf32_flops_per_sec_algorithmic': rate, 'share_of_tf32_peak': rate / TF32_PEAK,
                    'weight_tile_bytes_per_group_step': 2 * 2 * 4 * macs_pad})
    out[name] = rec
    return res


w128 = genomes([128] * 4, pop)
sh128 = rollout.actor_shape(128, 3, 'tanh')
r_tc = timed('tc_128x4', w128, sh128, [128] * 4)
r_k1 = timed('k1_h128_l3', w128, sh128, None)
out['tc_vs_k1_h128_l3'] = {'speedup_tc_over_k1': out['k1_h128_l3']['ms'] / out['tc_128x4']['ms'],
                           'same_termination_steps': bool(torch.equal(r_tc.steps, r_k1.steps)),
                           'max_rel_return_diff': float(((r_tc.returns - r_k1.returns).abs() / r_k1.returns.abs()).max().item())}
del w128
timed('tc_256x4', genomes([256] * 4, pop), rollout.actor_shape(256, 3, 'tanh'), [256] * 4)
timed('tc_400_300', genomes([400, 300], pop), rollout.actor_shape(72), [400, 300])
print(json.dumps(out))
