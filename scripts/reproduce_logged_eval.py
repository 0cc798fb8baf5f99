"""Does SERL10's logged evaluation table reproduce?  CPU only: the reference-order actor (oracle/actor.py, torch fp32) on the
reference's plant binaries (oracle/phlab.py, backend 'auto'), the references of serl_b200.evaluation.eval_refs drawn after
np.random.seed(seed) as base/evaluate.py draws them, base/evaluate.py's error and u_lst bookkeeping, and nMAE / smoothness
per actor (mean over the num_trails + 1 trials), against tests/golden/eval_logged.npz.  One process per episode.

    python scripts/reproduce_logged_eval.py [--conditions nominal] [--num_trails 1,2,3] [--seed 7] [--actors 10]
Prints one JSON line per (condition, num_trails) with the largest relative differences in nMAE and smoothness.
"""
import argparse
import json
import os
import sys
from multiprocessing import Pool

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import actor as A, phlab  # noqa: E402
from serl_b200 import evaluation  # noqa: E402
from serl_b200.core.utils import calc_nMAE, calc_smoothness  # noqa: E402

T_MAX = 80


def episode(job):
    genome, mode, lv, st, smooth_w = job
    actor = A.unflatten(genome, hidden=72, num_layers=3, activation='tanh')
    env = phlab.CitationEnv(mode, 'auto', t_max=T_MAX)
    env.smooth_w = smooth_w
    obs = env.reset(lv, st)
    done, errs, us = False, [], []
    while not done:
        x_ctrl = env.x[[7, 6, 5]].copy()
        us.append(env.last_u.copy())
        ref = np.deg2rad(env.ref_deg())
        obs, _, done, _ = env.step(np.clip(actor.select_action(obs), -1, 1))
        errs.append(ref - x_ctrl)
    return calc_nMAE(np.asarray(errs)), calc_smoothness(np.asarray(us)), len(errs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--conditions', default='nominal')
    ap.add_argument('--num_trails', default='1,2,3')
    ap.add_argument('--seed', type=int, default=7)
    ap.add_argument('--actors', type=int, default=10)
    a = ap.parse_args()
    acts = np.load(os.path.join(ROOT, 'tests', 'golden', 'actors.npz'))['serl10_pop_h72_tanh'][:a.actors]
    logged = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_logged.npz'))
    modes = {'low-q': 'h10000-v90', 'high-q': 'h2000-v150'}
    with Pool() as pool:
        for c in a.conditions.split(','):
            for n in [int(x) for x in a.num_trails.split(',')]:
                np.random.seed(a.seed)
                refs = evaluation.eval_refs(n, T_MAX)
                lv, st = evaluation._ref_arrays(refs)
                jobs = [(g, modes.get(c, c), lv[i], st[i], float(refs[i][0].smooth_width)) for g in acts for i in range(len(refs))]
                res = np.array(pool.map(episode, jobs)).reshape(len(acts), len(refs), 3)
                nm, sm = res[..., 0].mean(axis=1), res[..., 1].mean(axis=1)
                want = logged['serl10_' + c][:len(acts)]
                print(json.dumps({'condition': c, 'num_trails': n, 'nmae': nm.tolist(), 'logged_nmae': want[:, 1].tolist(),
                                  'sm': sm.tolist(), 'logged_sm': want[:, 0].tolist(),
                                  'steps_min': int(res[..., 2].min()),
                                  'max_rel_nmae': float(np.max(np.abs(nm - want[:, 1]) / np.abs(want[:, 1]))),
                                  'max_rel_sm': float(np.max(np.abs(sm - want[:, 0]) / np.abs(want[:, 0])))}), flush=True)


if __name__ == '__main__':
    main()
