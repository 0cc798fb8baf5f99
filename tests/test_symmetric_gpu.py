"""Symmetric control on the H100: K1 (warp actor at h = 32/64/72/96/128, and the one-thread-per-env kernel) against the
symmetric oracle (tests/symmetric_oracle.py: the reference-order env on the C plant restatement + the kernel-order actor at
2 inputs and 1 output), K1-TC against the torch actor on the flown observations and against K1, the 2 -> 1 serl_actor_forward,
the time-split hand-over, per-actor env blocks, K6 on the padded deflection record, and Agent.train() on PHlab_symmetric_nominal
with the torch TD3, on K1 and on K1-TC."""
import os
import random
import types

import numpy as np
import pytest
import torch

from oracle import actor as A
from serl_b200 import refsig
from serl_b200.core.utils import calc_smoothness

from symmetric_oracle import KernelOrderActor, evaluate_population  # noqa: E402  (tests/ on sys.path)

pytestmark = pytest.mark.gpu
REL_TOL = 1e-4          # the bar of tests/test_parity_strict_gpu.py
DEV = torch.device('cuda:0')
MODES = ['nominal', 'be', 'se']


def genomes(n, hidden, activation, seed, scale=1.0):
    torch.manual_seed(seed)
    g = np.stack([A.flatten(A.Actor(state_dim=2, action_dim=1, hidden=hidden, num_layers=3, activation=activation)) for _ in range(n)])
    return (g * np.float32(scale)).astype(np.float32)


def fly(w, hidden, activation, lv, st, horizon, modes=None, num_layers=3, **kw):
    from serl_b200 import rollout
    sh = rollout.actor_shape(hidden, num_layers, activation, state_dim=2, action_dim=1)
    n_envs = lv.shape[-3]
    if modes is None:
        md = torch.full(lv.shape[:-2], rollout.mode_code('nominal'), dtype=torch.int32, device=DEV)
    else:
        md = torch.tensor([rollout.mode_code(m) for m in modes], dtype=torch.int32, device=DEV)
    r = rollout.population_rollout(torch.as_tensor(w, device=DEV), sh, torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV),
                                   md, horizon=horizon, **kw)
    torch.cuda.synchronize()
    r.check()
    assert n_envs == r.returns.shape[1]
    return r


def noise_draws(pop, n_envs, horizon, seed):
    rs = np.random.RandomState(seed)
    return np.clip(0.3 * rs.randn(pop, n_envs, horizon, 1), -0.5, 0.5).astype(np.float32)


# ---- strict parity against the symmetric oracle --------------------------------------------------------------------------
@pytest.mark.parametrize('hidden', [32, 64, 72, 96, 128, 50])          # 50: the one-thread-per-env kernel
@pytest.mark.parametrize('activation', ['tanh', 'elu', 'relu'])
@pytest.mark.parametrize('noisy', [False, True])
def test_k1_flies_symmetric_control_like_the_oracle(hidden, activation, noisy):
    horizon = 500
    w = genomes(2, hidden, activation, seed=hidden + 7, scale=2.0)
    w[1, -(hidden + 1):] *= np.float32(0.05)                # a gentle elevator: a long flight next to an early termination
    lv, st = refsig.make_ref_params(3, seed_base=hidden, symmetric=True)
    nz = noise_draws(2, 3, horizon, hidden) if noisy else None
    r = fly(w, hidden, activation, lv, st, horizon, modes=MODES, replay_env=1, actions=True, trace=True,
            action_noise=torch.as_tensor(nz, device=DEV) if noisy else None)
    oret, ostp, eps = evaluate_population(w, hidden, lv, st, MODES, activation=activation, horizon=horizon, noise=nz)
    ret, stp = r.returns.cpu().numpy(), r.steps.cpu().numpy()
    assert np.array_equal(stp, ostp), (stp, ostp)
    assert (np.abs(ret - oret) / np.abs(oret)).max() <= REL_TOL
    rp, acts, tr = r.replay.cpu().numpy(), r.actions.cpu().numpy(), r.trace.cpu().numpy()
    assert rp.shape == (2, horizon, 8)
    for a in range(2):
        for e in range(3):                                   # the padded deflection: [de, 0, 0]
            n = stp[a, e]
            assert not acts[a, e, :n, 1:].any() and not tr[a, e, :n, 13:15].any()
            assert np.abs(tr[a, e, :n, 12] - eps[a][e]['u']).max() <= 1e-12
        n = stp[a, 1]
        rows, orows = rp[a, :n], eps[a][1]['rows']
        assert np.abs(rows - orows).max() <= 1e-3 and np.array_equal(rows[:, 6:8], orows[:, 6:8])
        assert np.array_equal(rows[1:, 0:2], rows[:-1, 3:5]) and rows[0, 0] == 0.0


def test_actor_forward_two_to_one_is_bit_exact_with_the_kernel_order_oracle():
    from serl_b200 import rollout
    for hidden in (32, 64, 72, 96, 128, 50):
        for activation in ('tanh', 'elu', 'relu'):
            g = genomes(1, hidden, activation, seed=3, scale=3.0)[0]
            rs = np.random.RandomState(hidden)
            obs = np.concatenate([rs.randn(3000, 2) * 0.05, rs.randn(1000, 2), rs.randn(200, 2) * 30.0, np.zeros((1, 2))]).astype(np.float32)
            got = rollout.actor_forward(torch.as_tensor(g, device=DEV), rollout.actor_shape(hidden, 3, activation, state_dim=2, action_dim=1),
                                        torch.as_tensor(obs, device=DEV)).cpu().numpy()
            want = KernelOrderActor(g, hidden, 3, activation).forward(obs)
            assert got.shape == (obs.shape[0], 1)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (hidden, activation, np.abs(got - want).max())


# ---- K1-TC ---------------------------------------------------------------------------------------------------------------------
def genomes_wide(n, widths, activation, seed, scale=1.0):
    torch.manual_seed(seed)
    g = np.stack([A.flatten(A.WideActor(widths, state_dim=2, action_dim=1, activation=activation)) for _ in range(n)])
    return (g * np.float32(scale)).astype(np.float32)


def trace_observations(tr, n):
    """the observations the actor saw at steps 0..n-1 of one trajectory, rebuilt from its trace: reset()'s [0, q of the initial
    condition], then the theta error and q of the step before"""
    from oracle import plant as OP
    x_ic = np.asarray(OP.make_plant('h2000_v90', 'port').initial_state())
    first = np.asarray([[0.0, x_ic[1]]])
    rest = np.stack((tr[:n - 1, 19], tr[:n - 1, 1]), axis=1)
    return np.vstack((first, rest)).astype(np.float32)


@pytest.mark.parametrize('widths', [[400, 300], [256] * 4])
@pytest.mark.parametrize('activation', ['tanh', 'elu', 'relu'])
def test_k1_tc_actions_match_a_torch_actor_on_the_flown_observations(widths, activation):
    """K1-TC with a 2-input layer 0 and one action: every action of the trace (column 16; 17-18 stay 0) against the torch fp32
    actor (and float64) on the observations that step saw, at the K1-TC bars of tests/test_wide_actor_gpu.py"""
    g = genomes_wide(3, widths, activation, seed=len(widths) + widths[0])
    g[0, -(widths[-1] + 1):] *= np.float32(0.01)               # a long flight next to short ones
    lv, st = refsig.make_ref_params(2, seed_base=widths[0], symmetric=True)
    r = fly(g, widths[0], activation, lv, st, 400, trace=True, actions=True, widths=widths, replay_env=1)
    stp, tr, rp, acts = r.steps.cpu().numpy(), r.trace.cpu().numpy(), r.replay.cpu().numpy(), r.actions.cpu().numpy()
    assert rp.shape[2] == 8
    for a in range(3):
        net = A.WideActor(widths, state_dim=2, action_dim=1, activation=activation)
        torch.nn.utils.vector_to_parameters(torch.as_tensor(g[a]), net.parameters())
        for e in range(2):
            n = stp[a, e]
            assert not tr[a, e, :n, 17:19].any() and not acts[a, e, :n, 1:].any()
            obs = trace_observations(tr[a, e], n)
            got = tr[a, e, :n, 16:17].astype(np.float32)
            ref32 = net(torch.as_tensor(obs)).detach().numpy()
            ref64 = net.double()(torch.as_tensor(obs, dtype=torch.float64)).detach().numpy()
            net.float()
            base = np.abs(ref32 - ref64).max()
            assert np.abs(got - ref32).max() <= 2e-5, (a, e)
            assert np.abs(got - ref64).max() <= max(4 * base, 5e-6), (a, e)
        assert np.array_equal(rp[a, :stp[a, 1], 0:2], trace_observations(tr[a, 1], stp[a, 1]))


def test_k1_and_k1_tc_fly_zero_output_actors_to_the_same_bits():
    """h = 128, L = 3 fits K1; [128] * 4 on K1-TC flies the same genome.  With zero output weights both command tanh(bo): the
    steps, returns, traces and replay rows are bit-identical"""
    g = genomes(3, 128, 'tanh', seed=8)
    g[:, -(128 + 1):-1] = 0.0
    g[:, -1] = np.float32([0.0, 0.2, -0.4])
    lv, st = refsig.make_ref_params(3, seed_base=4, symmetric=True)
    k1 = fly(g, 128, 'tanh', lv, st, 2001, trace=True, actions=True, replay_env=2)
    tc = fly(g, 128, 'tanh', lv, st, 2001, trace=True, actions=True, replay_env=2, widths=[128] * 4)
    assert torch.equal(k1.steps, tc.steps) and torch.equal(k1.returns, tc.returns)
    assert (k1.steps.cpu().numpy() == 2001).any()
    stp = k1.steps.cpu().numpy()
    for a in range(3):
        for e in range(3):
            assert torch.equal(k1.trace[a, e, :stp[a, e]], tc.trace[a, e, :stp[a, e]]), (a, e)
        assert torch.equal(k1.replay[a, :stp[a, 2]], tc.replay[a, :stp[a, 2]]), a


def test_k1_tc_per_actor_env_blocks_equal_one_actor_per_launch():
    g = genomes_wide(3, [256] * 4, 'elu', seed=12, scale=0.5)
    lv, st = refsig.make_ref_params(3 * 4, seed_base=9, symmetric=True)
    lv, st = np.ascontiguousarray(lv.reshape(3, 4, 2, 6)), np.ascontiguousarray(st.reshape(3, 4, 2, 6))
    r = fly(g, 256, 'elu', lv, st, 300, widths=[256] * 4, replay_env=3)
    for a in range(3):
        s = fly(g[a:a + 1], 256, 'elu', np.ascontiguousarray(lv[a]), np.ascontiguousarray(st[a]), 300, widths=[256] * 4, replay_env=3)
        n = int(s.steps[0, 3])
        assert torch.equal(r.returns[a], s.returns[0]) and torch.equal(r.steps[a], s.steps[0]) and torch.equal(r.replay[a, :n], s.replay[0, :n])


# ---- scheduling is invisible ---------------------------------------------------------------------------------------------------
def test_time_split_launch_equals_an_unsplit_one():
    """sm_limit = 8 gives more tasks than CTA slots: slots hand trajectories over through HBM mid-episode, the 2-entry
    observation included.  Every result is the unsplit launch's, bit for bit."""
    g = genomes(40, 72, 'tanh', seed=4, scale=1.5)
    g[::2, -(72 + 1):] *= np.float32(0.05)
    lv, st = refsig.make_ref_params(13, seed_base=5, symmetric=True)
    one = fly(g, 72, 'tanh', lv, st, 400, actions=True, replay_env=12)
    split = fly(g, 72, 'tanh', lv, st, 400, actions=True, replay_env=12, sm_limit=8)
    steps = one.steps.cpu().numpy()
    assert (steps > 200).any()
    assert torch.equal(split.returns, one.returns) and torch.equal(split.steps, one.steps)
    for a in range(40):
        for e in range(13):
            assert torch.equal(split.actions[a, e, :steps[a, e]], one.actions[a, e, :steps[a, e]]), (a, e)
        assert torch.equal(split.replay[a, :steps[a, 12]], one.replay[a, :steps[a, 12]]), a


def test_per_actor_env_blocks_equal_one_actor_per_launch():
    g = genomes(4, 64, 'elu', seed=6, scale=1.5)
    lv, st = refsig.make_ref_params(4 * 5, seed_base=8, symmetric=True)
    lv, st = lv.reshape(4, 5, 2, 6), st.reshape(4, 5, 2, 6)
    r = fly(g, 64, 'elu', np.ascontiguousarray(lv), np.ascontiguousarray(st), 400, replay_env=4)
    for a in range(4):
        s = fly(g[a:a + 1], 64, 'elu', np.ascontiguousarray(lv[a]), np.ascontiguousarray(st[a]), 400, replay_env=4)
        n = int(s.steps[0, 4])
        assert torch.equal(r.returns[a], s.returns[0]) and torch.equal(r.steps[a], s.steps[0]) and torch.equal(r.replay[a, :n], s.replay[0, :n])


def test_k6_on_the_padded_deflections_equals_the_one_column_metric():
    from serl_b200 import rollout
    g = genomes(6, 72, 'tanh', seed=9, scale=2.0)
    g[::2, -(72 + 1):] *= np.float32(0.05)
    lv, st = refsig.make_ref_params(4, seed_base=11, symmetric=True)
    r = fly(g, 72, 'tanh', lv, st, 2001, actions=True)
    sm = rollout.smoothness(r.actions, r.steps).cpu().numpy()
    acts, steps = r.actions.cpu().numpy(), r.steps.cpu().numpy()
    for a in range(6):
        for e in range(4):
            n = steps[a, e]
            ref = calc_smoothness(acts[a, e, :n, :1].astype(np.float64), dt=0.01)
            if n // 2 - 1 <= 0:
                assert sm[a, e] == 0.0
                continue
            assert abs(sm[a, e] - ref) <= 2e-5 * abs(ref) + 1e-9, (a, e, n, sm[a, e], ref)


# ---- the training path ---------------------------------------------------------------------------------------------------
def _train_symmetric(hidden=32, num_layers=3, mut_type='proximal', generations=2):
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    from serl_b200.parameters import Parameters
    cla = types.SimpleNamespace(env='PHlab_symmetric_nominal', seed=7, pop_size=10, test_ea=False, mut_type=mut_type, use_distil=False,
                                smooth_fitness=True)
    os.makedirs('/tmp/serl_test_sym', exist_ok=True)
    cwd = os.getcwd(); os.chdir('/tmp/serl_test_sym')
    try:
        args = Parameters(cla)
    finally:
        os.chdir(cwd)
    args.save_foldername = '/tmp/serl_test_sym/'
    args.state_dim, args.action_dim, args.hidden_size, args.num_layers = 2, 1, hidden, num_layers
    args.smooth_fitness = True
    args.learn_start = 200
    args.frac_frames_train = 0.02
    env = config.select_env('PHlab_symmetric_nominal')
    torch.manual_seed(7); np.random.seed(7); random.seed(7)
    ag = agent_mod.Agent(args, env)
    ag.genomes_before = ag.pop.genomes.clone()
    stats = [ag.train() for _ in range(generations)]
    torch.cuda.synchronize()
    return ag, stats


def test_agent_trains_a_symmetric_population_with_proximal_mutation():
    ag, stats = _train_symmetric()
    for s in stats:
        for k in ('best_train_fitness', 'pop_avg', 'pop_min', 'test_score', 'rl_reward'):
            assert np.isfinite(s[k]), (k, s[k])
    assert any(np.isfinite(s['TD_loss']) for s in stats)
    assert ag.replay_buffer.data.shape[1] == 7 and len(ag.replay_buffer) > 0 and ag.pop.buffers.data.shape[2] == 7
    assert torch.isfinite(ag.replay_buffer._chronological_rows()).all()
    assert torch.isfinite(ag.pop.genomes).all() and not torch.equal(ag.genomes_before, ag.pop.genomes)


def test_agent_routes_a_deep_symmetric_actor_to_k1_tc():
    """hidden 128 at L = 4 does not fit K1: the Agent's population, exploration and validation flights go to K1-TC"""
    from serl_b200 import rollout
    ag, stats = _train_symmetric(hidden=128, num_layers=4, mut_type='normal')
    assert rollout.tc_widths(ag.shape) == [128] * 5
    assert all(np.isfinite(s['best_train_fitness']) and np.isfinite(s['test_score']) for s in stats)
    assert ag.replay_buffer.data.shape[1] == 7 and len(ag.replay_buffer) > 0
