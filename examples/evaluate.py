"""Evaluate a trained run on the evaluation references: the flags of the reference's base/evaluate.py, without plots.

    python examples/evaluate.py -agent_name <run dir> -env all -eval_pop -num_trails 2 -save_stats
    python examples/evaluate.py -agent_name <run dir> -env nominal -eval_actor -index 3
    python examples/evaluate.py -agent_name <run dir> -env be,jr -eval_rl

`-agent_name` is a run directory holding files/config.yaml and the checkpoints Agent.save_agent writes (files/evo_nets.pkl,
files/rl_net.pkl).  `-env` takes one condition ('nominal', 'be', ..., or a full env name 'PHlab_<configuration>_<mode>'), a
comma list of one configuration, 'all' (serl_b200.evaluation.CONDITIONS) or 'PHlab_<configuration>_all'.  The actor's
state_dim / action_dim come from the env, as in base/evaluate.py: 'PHlab_attitude_incremental' evaluates an incremental-control
run (10 -> 3), 'PHlab_symmetric_<mode>' a symmetric-control run (2 -> 1), whose references are evaluation.symmetric_refs
seeded from -seed.  Output folders are named after the mode token (figures/incremental/, figures/be/).  -eval_pop flies the whole population on every condition in one rollout launch per
sensor-noise group (evaluation.evaluate_population); -eval_actor and -eval_rl fly one actor per condition
(evaluation.validate_agent).  base/evaluate.py evaluates one condition per run and seeds every run alike, so every
condition here flies the same references and draws its sensor noise from the same generator state.  -save_stats writes
<run>/figures/<condition>/final_performance.csv and appends to <run>/stats.toml (-eval_pop), or appends the RL actor's
table per condition (-eval_rl); -save_trajectory writes the time traces of the champion (-eval_pop) or of the evaluated
actor on the last trial to <run>/figures/<condition>/nominal_trajectory.csv.
"""
import argparse
import os
import random
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from serl_b200 import evaluation, rollout              # noqa: E402
from serl_b200.parameters import Parameters           # noqa: E402

parser = argparse.ArgumentParser()
parser.add_argument('-env', type=str, default='nominal',
                    help="a condition, a full env name PHlab_<configuration>_<mode>, PHlab_<configuration>_all, a comma list, or 'all'")
parser.add_argument('-seed', type=int, default=7)
parser.add_argument('-agent_name', type=str, required=True, help='run directory (files/config.yaml, files/*.pkl)')
parser.add_argument('-eval_pop', default=False, action='store_true')
parser.add_argument('-eval_actor', default=False, action='store_true')
parser.add_argument('-index', type=int)
parser.add_argument('-eval_rl', default=False, action='store_true')
parser.add_argument('-save_stats', default=False, action='store_true')
parser.add_argument('-save_trajectory', default=False, action='store_true')
parser.add_argument('-verbose', default=False, action='store_true')
parser.add_argument('-num_trails', default=1, type=int)


def conditions(text):
    try:
        return evaluation.env_conditions(text)
    except ValueError as e:
        raise SystemExit(str(e))


folder, env_dims = evaluation.condition_folder, evaluation.env_dims


def seed_all(seed):
    """base/evaluate.py:156-159"""
    torch.manual_seed(seed)
    np.random.seed(seed)
    random.seed(seed)


def actor_shape(params):
    return rollout.actor_shape(params.hidden_size, params.num_layers, params.activation_actor, params.state_dim, params.action_dim)


def fly_one(genome, shape, cond, refs, cla, label, state):
    np.random.set_state(state)          # this condition's sensor noise, as a run of base/evaluate.py on it alone draws it
    data, stats = evaluation.validate_agent(genome, shape, evaluation.condition_env(cond, shape=shape), refs, cla.num_trails)
    print(f'{cond} {label}: nMAE: {stats.nmae:0.1f}% with STD: {stats.nmae_sd:0.1f}   Smoothness: {stats.sm:0.0f} with STD: {stats.sm_sd:0.1f}')
    if cla.save_trajectory:
        evaluation.write_trajectory(cla.agent_name, folder(cond), data)
    return stats


def main(argv=None):
    cla = parser.parse_args(argv)
    conds = conditions(cla.env)
    seed_all(cla.seed)
    params = evaluation.run_config(cla.agent_name, Parameters(cla))
    params.state_dim, params.action_dim = env_dims(conds[0])
    shape = actor_shape(params)
    refs = evaluation.eval_refs(cla.num_trails)
    if evaluation.control_mode(params.state_dim, params.action_dim) == 'symmetric':
        # the symmetric env draws its own theta reference per episode; eval_refs above still advances np.random as
        # base/evaluate.py's gen_refs calls do
        refs = evaluation.symmetric_refs(cla.num_trails, cla.seed)
    state = np.random.get_state()        # where each condition's sensor-noise draws start
    if cla.eval_actor or cla.eval_pop:
        pop = evaluation.load_pop(cla.agent_name, params)
    if cla.eval_actor:
        if cla.index is None:
            raise SystemExit('-eval_actor needs -index')
        for c in conds:
            fly_one(pop[cla.index], shape, c, refs, cla, f'actor {cla.index}', state)
    elif cla.eval_pop:
        res = evaluation.evaluate_population(pop, shape, conds, refs, cla.num_trails, noise_state=state)
        for c in conds:
            if cla.verbose:
                for i in range(len(pop)):
                    s = res.stats(i, c)
                    print(f'{c} actor {i}: nMAE: {s.nmae:0.1f}% with STD: {s.nmae_sd:0.1f}   Smoothness: {s.sm:0.0f} with STD: {s.sm_sd:0.1f}')
            idx, avg = res.champion(c), res.average(c)
            print(f'{c}: champion {idx}  nMAE {res.stats(idx, c).nmae:0.1f}%')
            print(f'{c}: average nMAE: {avg.nmae:0.1f} with SD: {avg.nmae_sd:0.1f}   average smoothness: {avg.sm:0.1f} with SD: {avg.sm_sd:0.1f}')
            if cla.save_trajectory:      # the champion's traces: one more (traced) launch
                np.random.set_state(state)
                env = evaluation.condition_env(c, shape=shape)
                if env.sensor_noise:     # skip the draws of the actors before the champion: the suite's trajectories again
                    evaluation.sensor_noise_draws(idx * (cla.num_trails + 1), int(round(env.t_max / env.dt)) + 1)
                data, _ = evaluation.validate_agent(pop[idx], shape, env, refs, cla.num_trails)
                evaluation.write_trajectory(cla.agent_name, folder(c), data)
            if cla.save_stats:
                ci = res.conditions.index(c)
                evaluation.write_final_performance(cla.agent_name, folder(c), res.sm[:, ci], res.nmae[:, ci])
                evaluation.append_stats_toml(cla.agent_name, folder(c), idx, res.stats(idx, c), avg)
        return res
    elif cla.eval_rl:
        rl = evaluation.load_rl_agent(cla.agent_name, params)
        out = {}
        for c in conds:
            out[c] = fly_one(rl[0], shape, c, refs, cla, 'RL actor', state)
            if cla.save_stats:
                evaluation.append_rl_stats_toml(cla.agent_name, folder(c), out[c])
        return out
    else:
        raise SystemExit('choose one of -eval_pop, -eval_actor, -eval_rl')


if __name__ == '__main__':
    main()
