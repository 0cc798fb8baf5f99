"""The mutation-operator study of a trained run: the flags of the reference's base/evaluate_operators.py, without plots.

    python examples/evaluate_operators.py -agent_name <run dir> -env nominal -num_trails 3 -save_stats
    python examples/evaluate_operators.py -agent_name <run dir> -env all -mags 0.01,0.05,0.1,0.2

For every actor of the run's population: the parent flies num_trails + 1 evaluation episodes of 20 s and stores their
transitions, then one normal, one proximal and one safe child fly the same references; the relative change of each
child's return and safety cost against its parent is printed per operator (serl_b200.operators).  `-env` takes one
condition, a full env name, a comma list of one configuration, 'all' or 'PHlab_<configuration>_all'
(evaluation.env_conditions; 'PHlab_attitude_incremental' studies an incremental-control run, 'PHlab_symmetric_<mode>' a
symmetric one, except on 'gust' and 'test'); every condition runs the study on its own, seeded as a run of the reference script on
that condition alone.  `-mags m1,m2,...` repeats the study at several mutation magnitudes (default: the run's
mutation_mag).  -save_stats writes <run>/mutation_stats.toml (stats_cost, then stats_reward, the reference's layout; with
several conditions or magnitudes, the last ones run).
"""
import argparse
import os
import random
import sys
from pprint import pprint

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from serl_b200 import evaluation, operators            # noqa: E402
from serl_b200.parameters import Parameters           # noqa: E402

parser = argparse.ArgumentParser()
parser.add_argument('-env', type=str, default='nominal',
                    help="a condition, a full env name PHlab_<configuration>_<mode>, PHlab_<configuration>_all, a comma list, or 'all'")
parser.add_argument('-seed', type=int, default=7)
parser.add_argument('-agent_name', type=str, required=True, help='run directory (files/config.yaml, files/evo_nets.pkl)')
parser.add_argument('-save_stats', default=False, action='store_true')
parser.add_argument('-verbose', default=False, action='store_true')
parser.add_argument('-num_trails', default=0, type=int)
parser.add_argument('-mags', type=str, default=None, help='comma list of mutation magnitudes (default: the run\'s mutation_mag)')


def conditions(text):
    try:
        return evaluation.env_conditions(text)
    except ValueError as e:
        raise SystemExit(str(e))


def seed_all(seed):
    """base/evaluate_operators.py:76-79"""
    torch.manual_seed(seed)
    np.random.seed(seed)
    random.seed(seed)


def main(argv=None):
    cla = parser.parse_args(argv)
    mags = [float(m) for m in cla.mags.split(',')] if cla.mags else None
    params = evaluation.run_config(cla.agent_name, Parameters(cla))
    conds = conditions(cla.env)
    params.state_dim, params.action_dim = evaluation.env_dims(conds[0])       # from the env, as the reference sets them
    sym = evaluation.control_mode(params.state_dim, params.action_dim) == 'symmetric'
    pop = evaluation.load_pop(cla.agent_name, params)
    out = {}
    for c in conds:
        seed_all(cla.seed)
        refs = operators.study_refs(cla.num_trails, symmetric=sym, seed=cla.seed)
        runner = operators.OperatorRunner(params, c, num_trails=cla.num_trails)
        res = runner.test_mutation(pop, refs, mags)
        out[c] = res
        for mag, (sr, sc) in res.by_mag.items():
            print(f'{c}, mutation magnitude {mag}:')
            if cla.verbose:
                for i in range(len(pop)):
                    print(f'  Parent {i} {np.mean(res.parent_returns[i]):0.1f}, Cost: {np.mean(res.parent_costs[i]):0.1f}')
            pprint({'normal_r': np.mean(sr['Normal']), 'proximal_r': np.mean(sr['Proximal']), 'safe_r': np.mean(sr['Safe'])})
            pprint({'normal_c': np.mean(sc['Normal']), 'proximal_c': np.mean(sc['Proximal']), 'safe_c': np.mean(sc['Safe'])})
            pprint({'normal_nmae': np.mean(res.child_nmae['Normal'][res.mags.index(mag)]),
                    'proximal_nmae': np.mean(res.child_nmae['Proximal'][res.mags.index(mag)]),
                    'safe_nmae': np.mean(res.child_nmae['Safe'][res.mags.index(mag)])})
        if cla.save_stats:
            with open(os.path.join(cla.agent_name, 'mutation_stats.toml'), 'w', encoding='utf-8') as f:
                f.write(operators.mutation_stats_toml(res.stats_reward, res.stats_cost))
    return out


if __name__ == '__main__':
    main()
