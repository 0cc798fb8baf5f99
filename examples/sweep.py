"""Train several SERL / TD3 runs in one process on one GPU: examples/train.py's flags, plus the seeds and a grid of
`Parameters` attributes whose Cartesian product makes the runs.  Every run's RL half shares one grouped K7 launch per
generation (serl_b200/sweep.py), and every run computes exactly what it computes when trained alone.  The runs may differ
in actor shape (hidden_size, num_layers, activation_actor): narrow and wide learners share the K7 launch, and each
shape's population flies in a launch of its own.  Runs with prioritized experience replay (-per, or per in the grid) share
the K7 launch with uniform ones, each sampling its own priority tree.

    python examples/sweep.py -frames 20000 -pop_size 10 -seeds 7 8 9 -grid lr=0.0002,0.0004 noise_sd=0.2,0.3
    python examples/sweep.py -frames 20000 -pop_size 10 -grid hidden_size=72,96 activation_actor=tanh,relu
    python examples/sweep.py -frames 20000 -pop_size 10 -seeds 7 8 9 -per                   # every run prioritized
    python examples/sweep.py -frames 20000 -pop_size 10 -seeds 7 8 9 -grid per=0,1          # PER against uniform replay
    python examples/sweep.py -frames 20000 -pop_size 10 -seeds 7 8 9 -checkpoint_every 5     # ./tmp/checkpoint/ every 5
    python examples/sweep.py -frames 40000 -pop_size 10 -seeds 7 8 9 -resume tmp/checkpoint    # continued to 40000 frames
"""
import itertools
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from train import parser                                 # noqa: E402  examples/train.py's flags
from serl_b200.envs import config as env_config         # noqa: E402
from serl_b200.parameters import Parameters             # noqa: E402
from serl_b200.sweep import Sweep                       # noqa: E402

parser.add_argument('-seeds', type=int, nargs='+', default=None, help='one run per seed (default: -seed)')
parser.add_argument('-grid', nargs='*', default=[], metavar='NAME=V1,V2',
                    help='Parameters attributes and their values, e.g. lr=0.0002,0.0004 batch_size=64,86')


def _value(template, text):
    """text parsed as the type of the attribute's default"""
    if isinstance(template, bool):
        return text.lower() in ('1', 'true', 'yes')
    if isinstance(template, int):
        return int(text)
    if isinstance(template, float):
        return float(text)
    return text


def make_runs(cla):
    axes = []
    for item in cla.grid:
        name, _, values = item.partition('=')
        if not values:
            raise SystemExit('-grid %s: expected NAME=V1,V2,...' % item)
        axes.append((name, values.split(',')))
    runs = []
    for seed in cla.seeds or [cla.seed]:
        for combo in itertools.product(*[v for _, v in axes]):
            cla.seed = seed
            p = Parameters(cla)
            p.hidden_size = cla.hidden_size
            p.fused_td3 = True
            if cla.learn_start is not None:
                p.learn_start = cla.learn_start
            label = ['seed=%d' % seed]
            for (name, _), text in zip(axes, combo):
                if not hasattr(p, name):
                    raise SystemExit('-grid: Parameters has no attribute %r' % name)
                setattr(p, name, _value(getattr(p, name), text))
                label.append('%s=%s' % (name, text))
            env = env_config.select_env(cla.env)
            p.action_dim = env.action_space.shape[0]
            p.state_dim = env.observation_space.shape[0]
            runs.append((' '.join(label), p, env))
    return runs


if __name__ == '__main__':
    cla = parser.parse_args()
    runs = make_runs(cla)
    sweep = Sweep([(p, env) for _, p, env in runs], mixed_shapes=True, per=True)
    if cla.resume:
        sweep.load_checkpoint(cla.resume)
    print('Sweep of %d runs on' % len(runs), runs[0][1].env_name)
    start_time = time.time()
    while not sweep.finished:
        for (label, _, _), r, stats in zip(runs, sweep.runs, sweep.train()):
            if stats is None:
                continue
            a = r.agent
            print('[%s]' % label, 'Episodes:', a.num_episodes, 'Frames:', a.num_frames, ' Train Max: %.2f' % stats['best_train_fitness'],
                  ' Test Max: %.2f' % stats['test_score'], ' Population Avg: %.2f' % stats['pop_avg'], ' Weakest: %.2f' % stats['pop_min'],
                  ' Avg. ep. len: %.2fs' % stats['avg_ep_len'], ' RL Reward: %.2f' % stats['rl_reward'], ' time %.1fs' % (time.time() - start_time))
        if cla.checkpoint_every and max(r.agent.iterations for r in sweep.runs) % cla.checkpoint_every == 0:
            sweep.save_checkpoint(os.path.join(runs[0][1].save_foldername, 'checkpoint'))
    sweep.save_agent()
