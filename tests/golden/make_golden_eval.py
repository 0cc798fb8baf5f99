"""Generate tests/golden/eval_logged.npz from the reference tree's logged evaluation tables (runs only where /root/reference
exists; data only, no code of the reference).

  serl10_<condition>   [10, 2] (sm, nmae) per actor of SERL10's figures/<condition>/final_performance.csv (9 conditions)
  serl10_conditions    the 9 condition names
  serl10_champion      [9] champion_idx per condition of SERL10's stats.toml, same order
  td3_conditions       the conditions of TD3's stats.toml (the -eval_rl layout: one table per condition)
  td3_stats            [n, 4] (nmae, nmae_sd, sm, sm_sd) per condition, same order
"""
import glob
import os
import tomllib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference/logs/wandb'


def main():
    serl10 = glob.glob(REF + '/*_SERL10')[0]
    td3 = glob.glob(REF + '/*_TD3')[0]
    out = {}
    conds = sorted(os.listdir(os.path.join(serl10, 'figures')))
    with open(os.path.join(serl10, 'stats.toml'), 'rb') as f:
        st = tomllib.load(f)
    for c in conds:
        out['serl10_' + c] = np.loadtxt(os.path.join(serl10, 'figures', c, 'final_performance.csv'), delimiter=',')
    out['serl10_conditions'] = np.array(conds)
    out['serl10_champion'] = np.array([st[c]['champion_idx'] for c in conds])
    with open(os.path.join(td3, 'stats.toml'), 'rb') as f:
        t = tomllib.load(f)
    out['td3_conditions'] = np.array(list(t))
    out['td3_stats'] = np.array([[t[c][k] for k in ('nmae', 'nmae_sd', 'sm', 'sm_sd')] for c in t])
    np.savez(os.path.join(HERE, 'eval_logged.npz'), **out)


if __name__ == '__main__':
    main()
