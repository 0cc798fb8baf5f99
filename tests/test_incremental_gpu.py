"""Incremental control on the H100: K1 (warp actor at h = 32/64/72/96/128, and the one-thread-per-env kernel) against the
incremental oracle (tests/incremental_oracle.py: the reference-order env on the C plant restatement + the kernel-order actor at
10 inputs), the 10-input serl_actor_forward, the time-split hand-over of last_u, per-actor env blocks, and Agent.train() on
PHlab_attitude_incremental with the torch TD3."""
import os
import random
import types

import numpy as np
import pytest
import torch

from oracle import actor as A, refsig

from incremental_oracle import KernelOrderActor, evaluate_population  # noqa: E402  (tests/ on sys.path)

pytestmark = pytest.mark.gpu
REL_TOL = 1e-4          # the bar of tests/test_parity_strict_gpu.py
DEV = torch.device('cuda:0')


def genomes(n, hidden, activation, seed, scale=1.0):
    torch.manual_seed(seed)
    g = np.stack([A.flatten(A.Actor(state_dim=10, hidden=hidden, num_layers=3, activation=activation)) for _ in range(n)])
    return (g * np.float32(scale)).astype(np.float32)


def fly(w, hidden, activation, lv, st, horizon, num_layers=3, **kw):
    from serl_b200 import rollout
    sh = rollout.actor_shape(hidden, num_layers, activation, state_dim=10)
    n_envs = lv.shape[-3]
    md = torch.full(lv.shape[:-2], rollout.mode_code('nominal'), dtype=torch.int32, device=DEV)
    r = rollout.population_rollout(torch.as_tensor(w, device=DEV), sh, torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV),
                                   md, horizon=horizon, **kw)
    torch.cuda.synchronize()
    r.check()
    assert n_envs == r.returns.shape[1]
    return r


def noise_draws(pop, n_envs, horizon, seed):
    rs = np.random.RandomState(seed)
    return np.clip(0.3 * rs.randn(pop, n_envs, horizon, 3), -0.5, 0.5).astype(np.float32)


# ---- strict parity against the incremental oracle ------------------------------------------------------------------------
@pytest.mark.parametrize('hidden', [32, 64, 72, 96, 128, 50])          # 50: the one-thread-per-env kernel
@pytest.mark.parametrize('activation', ['tanh', 'elu', 'relu'])
@pytest.mark.parametrize('noisy', [False, True])
def test_k1_flies_incremental_control_like_the_oracle(hidden, activation, noisy):
    horizon = 500
    w = genomes(2, hidden, activation, seed=hidden + 7, scale=2.0)
    w[1, -(3 * hidden + 3):] *= np.float32(0.005)          # small rates: a long flight next to an early termination
    lv, st = refsig.make_ref_params(3, seed_base=hidden)
    nz = noise_draws(2, 3, horizon, hidden) if noisy else None
    r = fly(w, hidden, activation, lv, st, horizon, replay_env=1, actions=True, trace=True,
            action_noise=torch.as_tensor(nz, device=DEV) if noisy else None)
    oret, ostp, eps = evaluate_population(w, hidden, lv, st, activation=activation, horizon=horizon, noise=nz)
    ret, stp = r.returns.cpu().numpy(), r.steps.cpu().numpy()
    assert np.array_equal(stp, ostp), (stp, ostp)
    assert (np.abs(ret - oret) / np.abs(oret)).max() <= REL_TOL
    rp, acts, tr = r.replay.cpu().numpy(), r.actions.cpu().numpy(), r.trace.cpu().numpy()
    assert rp.shape == (2, horizon, 26)
    for a in range(2):
        n = stp[a, 1]
        rows, orows = rp[a, :n], eps[a][1]['rows']
        # the stored transitions are the oracle's (to the device plant's last bits), done and cost flags exactly
        assert np.abs(rows - orows).max() <= 1e-3 and np.array_equal(rows[:, 24:26], orows[:, 24:26])
        # and hang together: next_obs is the next obs; obs[7:10] is the integrated deflection, which actions / trace record
        assert np.array_equal(rows[1:, 0:10], rows[:-1, 13:23]) and not rows[0, 7:10].any()
        assert np.array_equal(rows[:, 20:23], acts[a, 1, :n]) and np.array_equal(rows[:, 20:23], tr[a, 1, :n, 12:15].astype(np.float32))
        assert np.abs(tr[a, 1, :n, 12:15] - eps[a][1]['u']).max() <= 1e-6


def test_full_episodes_and_early_terminations_at_h72():
    """output layers scaled by 0, 0.01, 0.05, 0.2: from the trim held for the whole 20 s to an early termination"""
    w = genomes(4, 72, 'tanh', seed=1)
    for i, s in enumerate([0.0, 0.01, 0.05, 0.2]):
        w[i, -(3 * 72 + 3):] *= np.float32(s)
    lv, st = refsig.make_ref_params(2, seed_base=9)
    r = fly(w, 72, 'tanh', lv, st, 2001)
    oret, ostp, _ = evaluate_population(w, 72, lv, st, horizon=2001)
    assert (ostp == 2001).any() and (ostp < 1200).any()
    assert np.array_equal(r.steps.cpu().numpy(), ostp)
    assert (np.abs(r.returns.cpu().numpy() - oret) / np.abs(oret)).max() <= REL_TOL
    print('incremental h72 steps', ostp.tolist())


def test_integrator_is_bit_exact_on_constant_commands():
    """Zero output weights and output biases b: the actor commands tanh(b) whatever it observes, so the deflection the trace
    records (columns 12-14) depends on the integrator alone and must be the oracle's u bit for bit, on K1, the simple kernel
    and K1-TC (two widths and deep)."""
    bo = np.float32([0.3, -0.2, 0.05])
    lv, st = refsig.make_ref_params(2, seed_base=12)
    for hidden, widths in ((72, None), (50, None), (128, [128, 128]), (128, [128] * 4)):
        L = 1 if widths == [128, 128] else 3
        w = genomes(1, hidden, 'tanh', seed=2) if L == 3 else genomes_wide(1, widths, 'tanh', seed=2)
        w[0, -(3 * hidden + 3):] = 0.0
        w[0, -3:] = bo
        r = fly(w, hidden, 'tanh', lv, st, 600, trace=True, widths=widths, num_layers=L)
        _, ostp, eps = evaluate_population(w, hidden, lv, st, num_layers=L, horizon=600)
        stp, tr = r.steps.cpu().numpy(), r.trace.cpu().numpy()
        assert np.array_equal(stp, ostp), (hidden, widths)
        for e in range(2):
            assert np.array_equal(tr[0, e, :stp[0, e], 12:15], eps[0][e]['u']), (hidden, widths, e)


# ---- K1-TC ---------------------------------------------------------------------------------------------------------------------
def genomes_wide(n, widths, activation, seed, scale=1.0):
    torch.manual_seed(seed)
    g = np.stack([A.flatten(A.WideActor(widths, state_dim=10, activation=activation)) for _ in range(n)])
    return (g * np.float32(scale)).astype(np.float32)


def trace_observations(tr, n):
    """the observations the actor saw at steps 0..n-1 of one trajectory, rebuilt from its trace: reset()'s [0, 0, 0, p q r alpha
    of the initial condition, 0, 0, 0], then the tracking error, p q r alpha and last_u of the step before"""
    from oracle import plant as OP
    x_ic = np.asarray(OP.make_plant('h2000_v90', 'port').initial_state())
    first = np.hstack((np.zeros(3), x_ic[[0, 1, 2, 4]], np.zeros(3)))[None]
    rest = np.hstack((tr[:n - 1, 19:22], tr[:n - 1, [0, 1, 2, 4]], tr[:n - 1, 12:15]))
    return np.vstack((first, rest)).astype(np.float32)


@pytest.mark.parametrize('widths', [[400, 300], [256] * 4, [128] * 4])
@pytest.mark.parametrize('activation', ['tanh', 'elu', 'relu'])
def test_k1_tc_actions_match_a_torch_actor_on_the_flown_observations(widths, activation):
    """K1-TC with a 10-input layer 0: every action of the trace (columns 16-18) against the torch fp32 actor (and float64) on
    the observations that step saw, at the K1-TC bars of tests/test_wide_actor_gpu.py"""
    g = genomes_wide(3, widths, activation, seed=len(widths) + widths[0])
    g[0, -(3 * widths[-1] + 3):] *= np.float32(0.01)           # a long flight next to short ones
    lv, st = refsig.make_ref_params(2, seed_base=widths[0])
    r = fly(g, widths[0], activation, lv, st, 400, trace=True, widths=widths, replay_env=1)
    stp, tr, rp = r.steps.cpu().numpy(), r.trace.cpu().numpy(), r.replay.cpu().numpy()
    assert rp.shape[2] == 26
    for a in range(3):
        net = A.WideActor(widths, state_dim=10, activation=activation)
        torch.nn.utils.vector_to_parameters(torch.as_tensor(g[a]), net.parameters())
        for e in range(2):
            n = stp[a, e]
            obs = trace_observations(tr[a, e], n)
            got = tr[a, e, :n, 16:19].astype(np.float32)
            ref32 = net(torch.as_tensor(obs)).detach().numpy()
            ref64 = net.double()(torch.as_tensor(obs, dtype=torch.float64)).detach().numpy()
            net.float()
            base = np.abs(ref32 - ref64).max()
            assert np.abs(got - ref32).max() <= 2e-5, (a, e)
            assert np.abs(got - ref64).max() <= max(4 * base, 5e-6), (a, e)
        assert np.array_equal(rp[a, :stp[a, 1], 0:10], trace_observations(tr[a, 1], stp[a, 1]))


def test_k1_and_k1_tc_fly_zero_output_actors_to_the_same_bits():
    """h = 128, L = 3 fits K1; [128] * 4 on K1-TC flies the same genome.  With zero output weights both command tanh(bo): the
    steps, returns and traces are bit-identical"""
    g = genomes(3, 128, 'tanh', seed=8)
    g[:, -(3 * 128 + 3):-3] = 0.0
    g[:, -3:] = np.float32([[0.0, 0.0, 0.0], [0.2, -0.1, 0.05], [-0.4, 0.3, -0.2]])
    lv, st = refsig.make_ref_params(3, seed_base=4)
    k1 = fly(g, 128, 'tanh', lv, st, 2001, trace=True, actions=True)
    tc = fly(g, 128, 'tanh', lv, st, 2001, trace=True, actions=True, widths=[128] * 4)
    assert torch.equal(k1.steps, tc.steps) and torch.equal(k1.returns, tc.returns)
    assert (k1.steps.cpu().numpy() == 2001).any()
    stp = k1.steps.cpu().numpy()
    for a in range(3):
        for e in range(3):
            assert torch.equal(k1.trace[a, e, :stp[a, e]], tc.trace[a, e, :stp[a, e]]), (a, e)


def test_agent_routes_a_wide_incremental_actor_to_k1_tc():
    """hidden 128 at L = 4 does not fit K1: the Agent's population, exploration and validation flights go to K1-TC"""
    from serl_b200 import rollout
    stats, ag = _train(hidden=128, num_layers=4, generations=2)
    assert rollout.tc_widths(ag.shape) == [128] * 5
    assert all(np.isfinite(s['best_train_fitness']) and np.isfinite(s['test_score']) for s in stats)
    assert ag.replay_buffer.data.shape[1] == 25 and len(ag.replay_buffer) > 0


# ---- the actor alone ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('hidden', [32, 64, 72, 96, 128, 50])
@pytest.mark.parametrize('activation', ['tanh', 'elu', 'relu'])
def test_actor_forward_at_ten_inputs_is_bit_exact_with_the_kernel_order_oracle(hidden, activation):
    from serl_b200 import rollout
    g = genomes(1, hidden, activation, seed=3, scale=3.0)[0]
    rs = np.random.RandomState(hidden)
    obs = np.concatenate([rs.randn(3000, 10) * 0.05, rs.randn(1000, 10), rs.randn(200, 10) * 30.0, np.zeros((1, 10))]).astype(np.float32)
    got = rollout.actor_forward(torch.as_tensor(g, device=DEV), rollout.actor_shape(hidden, 3, activation, state_dim=10),
                                torch.as_tensor(obs, device=DEV)).cpu().numpy()
    want = KernelOrderActor(g, hidden, 3, activation).forward(obs)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.abs(got - want).max()


# ---- scheduling is invisible ---------------------------------------------------------------------------------------------------
def test_time_split_hand_over_carries_last_u():
    """300 actors x 13 envs is more tasks than CTA slots: slots hand trajectories over through HBM mid-episode, last_u and the
    10-entry observation included.  Every actor gets the bits of the 10-actor launch."""
    g = genomes(10, 72, 'tanh', seed=4, scale=1.5)
    g[::2, -(3 * 72 + 3):] *= np.float32(0.01)                   # half of them fly the whole 400 steps
    lv, st = refsig.make_ref_params(13, seed_base=5)
    one = fly(g, 72, 'tanh', lv, st, 400, actions=True, replay_env=12)
    many = fly(np.tile(g, (30, 1)), 72, 'tanh', lv, st, 400, actions=True, replay_env=12)
    steps = one.steps.cpu().numpy()
    assert (steps > 200).any()                                   # trajectories that are handed over mid-flight
    for a in range(300):
        b = a % 10
        assert torch.equal(many.returns[a], one.returns[b]) and torch.equal(many.steps[a], one.steps[b]), a
        for e in range(13):                                      # rows past an episode's end are not written
            assert torch.equal(many.actions[a, e, :steps[b, e]], one.actions[b, e, :steps[b, e]]), (a, e)
        assert torch.equal(many.replay[a, :steps[b, 12]], one.replay[b, :steps[b, 12]]), a


def test_per_actor_env_blocks_equal_one_block_per_launch():
    g = genomes(4, 64, 'elu', seed=6, scale=1.5)
    lv, st = refsig.make_ref_params(4 * 5, seed_base=8)
    lv, st = lv.reshape(4, 5, 2, 6), st.reshape(4, 5, 2, 6)
    r = fly(g, 64, 'elu', np.ascontiguousarray(lv), np.ascontiguousarray(st), 400, replay_env=4)
    for a in range(4):
        s = fly(g[a:a + 1], 64, 'elu', np.ascontiguousarray(lv[a]), np.ascontiguousarray(st[a]), 400, replay_env=4)
        n = int(s.steps[0, 4])
        assert torch.equal(r.returns[a], s.returns[0]) and torch.equal(r.steps[a], s.steps[0]) and torch.equal(r.replay[a, :n], s.replay[0, :n])


# ---- the training path ---------------------------------------------------------------------------------------------------
def make_args(pop=10, hidden=32, **kw):
    from serl_b200.parameters import Parameters
    cla = types.SimpleNamespace(env='PHlab_attitude_incremental', seed=7, pop_size=pop, test_ea=False, **kw)
    os.makedirs('/tmp/serl_test_inc', exist_ok=True)
    cwd = os.getcwd(); os.chdir('/tmp/serl_test_inc')
    try:
        args = Parameters(cla)
    finally:
        os.chdir(cwd)
    args.save_foldername = '/tmp/serl_test_inc/'
    args.state_dim, args.action_dim, args.hidden_size = 10, 3, hidden
    args.learn_start = 200               # the torch TD3 takes gradient steps within the three generations ...
    args.frac_frames_train = 0.02        # ... a few hundred per generation
    return args


def _train(prefetch=True, independent=False, mut_type='normal', distil=False, hidden=32, num_layers=3, generations=3):
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    args = make_args(hidden=hidden, mut_type=mut_type, use_distil=distil)
    args.num_layers = num_layers
    args.prefetch_generation = prefetch
    args.independent_references = independent
    env = config.select_env('PHlab_attitude_incremental')
    torch.manual_seed(7); np.random.seed(7); random.seed(7)
    ag = agent_mod.Agent(args, env)
    stats = [ag.train() for _ in range(generations)]
    torch.cuda.synchronize()
    return stats, ag


@pytest.mark.parametrize('independent', [False, True])
def test_agent_trains_an_incremental_population(independent):
    stats, ag = _train(independent=independent)
    for s in stats:
        for k in ('best_train_fitness', 'pop_avg', 'pop_min', 'test_score', 'rl_reward'):
            assert np.isfinite(s[k]), (k, s[k])
    assert any(np.isfinite(s['TD_loss']) for s in stats)                    # the torch TD3 trained
    assert ag.replay_buffer.data.shape[1] == 25 and len(ag.replay_buffer) > 0
    assert ag.pop.buffers.data.shape[2] == 25
    rows = ag.replay_buffer._chronological_rows()
    assert torch.isfinite(rows).all()


def test_prefetched_generation_changes_no_incremental_result():
    a, aga = _train(prefetch=True)
    b, agb = _train(prefetch=False)
    for x, y in zip(a, b):
        for k in x:
            assert (x[k] == y[k]) or (np.isnan(x[k]) and np.isnan(y[k])), k
    assert torch.equal(aga.pop.genomes, agb.pop.genomes)
    assert torch.equal(aga.replay_buffer._chronological_rows(), agb.replay_buffer._chronological_rows())


@pytest.mark.parametrize('mut_type,distil', [('proximal', False), ('safe', False), ('normal', True)])
def test_mutation_operators_and_distillation_on_ten_input_actors(mut_type, distil):
    stats, ag = _train(mut_type=mut_type, distil=distil)
    assert all(np.isfinite(s['best_train_fitness']) for s in stats)
    assert torch.isfinite(ag.pop.genomes).all()
