"""Training driver with the call sequence of the reference's base/train.py:54-139 (parse -> Parameters -> select_env ->
seed -> Agent -> while frames: agent.train() -> save_agent), written against this repo's mirror modules.  A maintainer of
the reference keeps base/train.py unchanged and swaps the imported packages instead (INTEGRATION.md).

    python examples/train.py -frames 20000 -pop_size 10 -test_ea
    python examples/train.py -frames 800000 -fused_td3 -checkpoint_every 10          # ./tmp/checkpoint.pt every 10 generations
    python examples/train.py -frames 1600000 -fused_td3 -resume tmp/checkpoint.pt    # the same run, continued to 1.6M frames
"""
import argparse
import os
import random
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from serl_b200.core import agent as agent_mod          # noqa: E402
from serl_b200.parameters import Parameters             # noqa: E402
from serl_b200.envs import config as env_config         # noqa: E402

parser = argparse.ArgumentParser()
parser.add_argument('-env', type=str, default='PHlab_attitude_nominal')
parser.add_argument('-frames', type=int, required=True)
parser.add_argument('-pop_size', default=10, type=int)
parser.add_argument('-seed', type=int, default=7)
parser.add_argument('-mut_type', type=str, default='normal')
parser.add_argument('-test_ea', default=False, action='store_true')
parser.add_argument('-use_distil', default=False, action='store_true')
parser.add_argument('-distil_type', type=str, default='fitness')
parser.add_argument('-sync_period', type=int, default=1)
parser.add_argument('-num_envs', type=int, default=3)
parser.add_argument('-hidden_size', type=int, default=72)
parser.add_argument('-independent_refs', default=False, action='store_true',
                    help='every episode of every actor draws its own reference signals, as the reference does (default: the '
                         'actors of a generation share num_envs draws)')
parser.add_argument('-per', help='Use Prioritised Experience Replay', action='store_true')
parser.add_argument('-no_prefetch', dest='prefetch_generation', default=True, action='store_false',
                    help='strictly one generation per Agent.train() call (no rollouts of the next generation queued ahead)')
parser.add_argument('-fused_td3', default=False, action='store_true',
                    help="the RL half's gradient steps in one K7 launch per generation (serl_b200/td3_fused.py)")
parser.add_argument('-learn_start', type=int, default=None,
                    help='transitions in the shared buffer before the first gradient step (default: Parameters.learn_start)')
parser.add_argument('-checkpoint_every', type=int, default=0, metavar='N',
                    help='checkpoint every N generations (0: never): train.py writes <save_foldername>/checkpoint.pt, sweep.py '
                         'the folder <save_foldername>/checkpoint')
parser.add_argument('-resume', type=str, default=None, metavar='PATH',
                    help='continue the run (sweep.py: the sweep) saved at PATH, up to -frames; every other flag as when it started')

if __name__ == '__main__':
    cla = parser.parse_args()
    parameters = Parameters(cla)
    parameters.hidden_size = cla.hidden_size
    if cla.learn_start is not None:
        parameters.learn_start = cla.learn_start
    env = env_config.select_env(cla.env)
    parameters.action_dim = env.action_space.shape[0]
    parameters.state_dim = env.observation_space.shape[0]
    env.seed(parameters.seed)
    torch.manual_seed(parameters.seed)
    np.random.seed(parameters.seed)
    random.seed(parameters.seed)
    agent = agent_mod.Agent(parameters, env)
    stats = agent.load_checkpoint(cla.resume)['stats'] if cla.resume else None
    print('Running', parameters.env_name, ' State_dim:', parameters.state_dim, ' Action_dim:', parameters.action_dim)
    start_time = time.time()
    while agent.num_frames <= parameters.num_frames:
        stats = agent.train()
        if cla.checkpoint_every and agent.iterations % cla.checkpoint_every == 0:
            agent.save_checkpoint(os.path.join(parameters.save_foldername, 'checkpoint.pt'), extra={'stats': stats})
        print('Episodes:', agent.num_episodes, 'Frames:', agent.num_frames, ' Train Max: %.2f' % stats['best_train_fitness'],
              ' Test Max: %.2f' % stats['test_score'], ' Population Avg: %.2f' % stats['pop_avg'], ' Weakest: %.2f' % stats['pop_min'],
              ' Avg. ep. len: %.2fs' % stats['avg_ep_len'], ' RL Reward: %.2f' % stats['rl_reward'], ' time %.1fs' % (time.time() - start_time))
    agent.save_agent(parameters, stats['elite_index'])
