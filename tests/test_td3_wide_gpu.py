"""K7 for actors wider than 128 (csrc/td3.cu, the WIDE instantiation: tiled phases for the actor's h x h blocks) against a
float64 reference, with the budget and harness of tests/test_td3_reference_gpu.py:

    ||K7 - f64|| <= C * ||torch32 - f64|| + FLOOR * scale      per tensor, all eight state blocks and the loss series,

K7's recorded draws replayed through the fp32 oracle (oracle/td3.py) and its float64 copy.  Tensors the float64 update
leaves bit-unchanged must stay bit-unchanged.  Cases: hidden 129, 160, 256, 320 x 1, 3, 8 layers x three activations;
batches 1, 86, 128; the CAPS variants; clipped critic and actor; warm Adam at iteration 1000 with a champion target; 300
steps on K1 flight rows.  Then the bits: cluster sizes 1, 2, 4, 8, a repeated launch and a 17 + 23 split give identical
state and losses, and an Agent with hidden 256 trains with fused_td3 end to end."""
import importlib.util
import os
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
_spec = importlib.util.spec_from_file_location('td3_reference_harness', os.path.join(HERE, 'test_td3_reference_gpu.py'))
R = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(R)

pytestmark = pytest.mark.gpu
DEV = R.DEV


def wide(hidden=256, num_layers=3, activation='tanh', **kw):
    f = R.fused(R.td3_args(hidden, num_layers, activation, **kw))
    return f, R.Reference(f)


# ---- shapes, batches, CAPS ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize('hidden', [129, 160, 256, 320])
@pytest.mark.parametrize('num_layers', [1, 3, 8])
@pytest.mark.parametrize('activation', ['tanh', 'elu', 'relu'])
def test_every_wide_shape_matches_float64(hidden, num_layers, activation):
    """iterations 1..3: two critic-only steps (the actor untouched) and one actor step"""
    f, ref = wide(hidden, num_layers, activation)
    rows = R.synthetic_rows(3000, seed=hidden + num_layers).to(DEV)
    R.run_and_check(f, ref, rows, 3, 1, 'h%d L%d %s' % (hidden, num_layers, activation))


@pytest.mark.parametrize('batch', [1, 86, 128])
def test_wide_batches_match_float64(batch):
    f, ref = wide(batch_size=batch)
    rows = R.synthetic_rows(3000, seed=batch).to(DEV)
    R.run_and_check(f, ref, rows, 3, 1, 'h256 B%d' % batch)


@pytest.mark.parametrize('lambda_t,lambda_s', [(0.1, 0.5), (0.0, 0.0), (0.1, 0.0)])
def test_wide_caps_terms_match_float64(lambda_t, lambda_s):
    """CAPS off (lambda_s = 0) halves the actor's rows: B instead of 2B"""
    f, ref = wide(320, 2, batch_size=128)
    f.caps_dict = {'lambda_t': lambda_t, 'lambda_s': lambda_s, 'eps_sd': 0.05}
    ref = R.Reference(f)
    rows = R.synthetic_rows(3000, seed=8).to(DEV)
    R.run_and_check(f, ref, rows, 3, 1, 'h320 CAPS lt %g ls %g' % (lambda_t, lambda_s))


# ---- clipping, warm Adam, long runs ---------------------------------------------------------------------------------------

def test_wide_clipped_critic_and_actor_match_float64():
    f, ref = wide()
    rows = R.synthetic_rows(3000, seed=5, reward_scale=30.0).to(DEV)
    _, norms = R.run_and_check(f, ref, rows, 3, 1, 'h256 critic clipped')
    assert all(n[0] > 10 for n in norms), norms
    f, _ = wide()
    with torch.no_grad():
        f.critic.q1[4].weight.mul_(300.0)
    ref = R.Reference(f)
    _, norms = R.run_and_check(f, ref, R.synthetic_rows(3000, seed=5).to(DEV), 3, 1, 'h256 both clipped')
    assert all(n[0] > 10 for n in norms) and norms[2][1] > 10, norms


@pytest.mark.parametrize('champion', [False, True])
def test_wide_warm_adam_at_iteration_1000_matches_float64(champion):
    f, ref = wide()
    R.warm_adam(f, ref, 999, 333)
    rows = R.synthetic_rows(3000, seed=3).to(DEV)
    R.run_and_check(f, ref, rows, 4, 1000, 'h256 warm Adam champion %d' % champion, champion=champion)
    assert (f.critic_steps, f.actor_steps) == (1003, 334)


def test_wide_300_steps_on_flight_rows_match_float64():
    f, ref = wide()
    R.run_and_check(f, ref, R.flight_rows(), 300, 1, 'h256 L3 300 steps, flight rows')


# ---- bits ----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('hidden,num_layers', [(256, 3), (320, 8)])
def test_wide_cluster_size_repeated_and_split_launches_are_bitwise_identical(hidden, num_layers):
    f, _ = wide(hidden, num_layers)
    rows = R.synthetic_rows(5000, seed=3).to(DEV)
    s0 = f.state.clone()

    def go(plan, cs):
        f.state.copy_(s0)
        f.critic_steps = f.actor_steps = 0
        first, losses = 1, []
        for n in plan:
            losses.append(f.run(rows, rows.shape[0], n, first, False, cluster_size=cs).losses)
            first += n
        torch.cuda.synchronize()
        return f.state.clone(), torch.cat(losses).nan_to_num(7.0)

    ref_state, ref_loss = go([40], 1)
    assert torch.isfinite(ref_loss).all() and not torch.equal(ref_state, s0)
    for plan, cs in (([40], 2), ([40], 4), ([40], 8), ([40], 8), ([17, 23], 4), ([17, 23], 8)):
        s, l = go(plan, cs)
        assert torch.equal(s, ref_state) and torch.equal(l, ref_loss), (plan, cs)


# ---- the Agent ---------------------------------------------------------------------------------------------------------

def test_agent_with_a_wide_fused_learner_trains(tmp_path, monkeypatch):
    from serl_b200 import rollout
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    from serl_b200.parameters import Parameters
    from serl_b200.td3_fused import FusedTD3
    routed = []
    tc_widths = rollout.tc_widths
    monkeypatch.setattr(rollout, 'tc_widths', lambda shape: routed.append(tc_widths(shape)) or routed[-1])
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        args = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=7, pop_size=4, mut_type='normal', test_ea=False,
                                                fused_td3=True))
    finally:
        os.chdir(cwd)
    args.save_foldername = str(tmp_path) + '/'
    args.state_dim, args.action_dim, args.hidden_size = 7, 3, 256
    args.learn_start, args.frac_frames_train = 300, 0.2
    torch.manual_seed(7)
    ag = agent_mod.Agent(args, config.select_env('PHlab_attitude_nominal'))
    assert isinstance(ag.rl_agent, FusedTD3) and ag.rl_agent.shape.hidden == 256
    before = torch.cat([p.detach().reshape(-1) for p in ag.rl_agent.actor.parameters()]).clone()
    for _ in range(2):
        stats = ag.train()
    assert np.isfinite(stats['TD_loss']) and np.isfinite(stats['PG_obj'])
    assert ag.rl_iteration > 0
    after = torch.cat([p.detach().reshape(-1) for p in ag.rl_agent.actor.parameters()])
    assert not torch.equal(before, after)
    # the population and the RL flights went through K1-TC
    assert routed and all(w == [256] * (args.num_layers + 1) for w in routed), routed
    # a critic weight edited through the evolver's module is what the next launch reads
    assert ag.evolver.critic is ag.rl_agent.critic
    rows = ag.replay_buffer.data[:len(ag.replay_buffer)]
    snap = ag.rl_agent.state.clone()
    steps = (ag.rl_agent.critic_steps, ag.rl_agent.actor_steps)
    l1 = ag.rl_agent.run(rows, rows.shape[0], 1, 1).losses.clone()
    ag.rl_agent.state.copy_(snap)
    ag.rl_agent.critic_steps, ag.rl_agent.actor_steps = steps
    with torch.no_grad():
        ag.evolver.critic.q1[4].bias.add_(1.0)
    l2 = ag.rl_agent.run(rows, rows.shape[0], 1, 1).losses
    assert l1[0, 0] != l2[0, 0]
