"""Hyper-parameter bag — mirror of base/parameters.py (same attribute names, same tuned constants :44-116), plus the
knobs of the B200 engine.  `Parameters(cla)` accepts the argparse namespace of base/train.py:16-51 unchanged.

Differences from the reference (documented in DESIGN.md):
  * distil_crossover defaults to False and mut_type 'proximal'/'safe' are rejected by SSNE: the engine implements the
    classic operators (crossover_inplace / mutate_inplace); distillation and Jacobian-scaled mutation need per-actor
    replay buffers + autograd and are listed as "next" (SURVEY.md 8(f) N3).
  * num_envs: environments per actor and generation flown by the rollout kernel (defaults to num_evals = 3).
  * independent_references: every population episode draws its own reference signals, as the reference does (default
    False: every actor of a generation flies the same num_envs draws).
"""
import os
from pprint import pprint

import torch


class Parameters:
    def __init__(self, cla, init=True):
        if not init:
            return
        g = lambda name, default: getattr(cla, name) if hasattr(cla, name) else default
        # the rollout / evolution engine always runs on CUDA; `device` is where the RL (TD3) half lives
        self.device = torch.device('cuda') if torch.cuda.is_available() else torch.device('cpu')
        self.env_name = g('env', 'PHlab_attitude_nominal')
        self.save_periodic = hasattr(cla, 'save_periodic')
        self.num_frames = g('frames', 800_000)
        self.rl_to_ea_synch_period = g('sync_period', 1)
        self.next_save = g('next_save', 1000)
        # RL (TD3) — parameters.py:37-73
        self.test_ea = g('test_ea', False)
        self.frac_frames_train = 0. if self.test_ea else 1.
        self.batch_size = 86
        self.buffer_size = 100_000
        self.lr = 0.0004335
        self.gamma = 0.98
        self.noise_sd = 0.2962183114680794
        self.use_done_mask = True
        self.use_ounoise = g('use_ounoise', False)
        self.tau = 0.005
        self.seed = g('seed', 7)
        self.num_layers = 3
        self.hidden_size = 72
        self.activation_actor = 'tanh'
        self.activation_critic = 'elu'
        self.learn_start = 10_000
        self.per = g('per', False)
        self.use_caps = g('use_caps', True)
        self.policy_update_freq = 3
        self.noise_clip = 0.5
        # the RL half's gradient steps in one K7 launch per generation (serl_b200/td3_fused.py) instead of the torch loop
        self.fused_td3 = bool(g('fused_td3', False))
        # neuro-evolution — parameters.py:76-116
        self.pop_size = g('pop_size', 10)
        self.use_champion_target = g('champion_target', False)
        self.individual_bs = 10_000
        if self.pop_size:
            self.smooth_fitness = g('smooth_fitness', False)
            self.buffer_size = 800_000
            self.lr = 0.00018643512599969097
            self.num_evals = 3
            self.elite_fraction = 0.2
            self.mutation_prob = 0.9
            self.mutation_mag = 0.0247682869654
            self.mutation_batch_size = self.batch_size
            self.mut_type = g('mut_type', 'normal')
            # 'proximal' (base/train.py's CLI default) and 'safe' are implemented batched on the device (serl_b200/evo_prox.py)
            self.distil_crossover = bool(g('use_distil', False))      # the reference hard-codes True (parameters.py:112)
            self.distil_type = g('distil_type', 'fitness')
            self.crossover_prob = 0.0
            self._verbose_mut = g('verbose_mut', False)
            self._verbose_crossover = g('verbose_crossover', False)
        # engine knobs
        self.num_envs = g('num_envs', getattr(self, 'num_evals', 3))
        # every episode of every actor draws its own reference signals, as base/core/agent.py:234-241 does (the default gives
        # all actors of a generation the same num_envs draws: fair ranking)
        self.independent_references = bool(g('independent_refs', False))
        # Agent.train() queues the next generation's rollouts before it waits for its own validation scores (core/agent.py)
        self.prefetch_generation = bool(g('prefetch_generation', True))
        self.state_dim = None
        self.action_dim = None
        self.save_foldername = './tmp/'
        self.should_log = g('should_log', False)
        if not os.path.exists(self.save_foldername):
            os.makedirs(self.save_foldername)

    def write_params(self, stdout=True):
        params = pprint(vars(self), indent=4)
        if stdout:
            print(params)

    def update_from_dict(self, new_config_dict: dict):
        self.__dict__.update(new_config_dict)
