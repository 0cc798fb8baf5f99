"""The reference's Actor beyond hidden 128: width lists of any depth [w0, w1, ..., w_{n-1}] on the tensor-core rollout kernel
(csrc/rollout_tc.cu tc_actor_forward_deep), and uniform actors K1 cannot hold routed to it by population_rollout.

Bars as in test_wide_actor_gpu.py: forward |action - torch fp32| <= 2e-5 and not worse than 4x the float32 forward pass's own
distance from float64; closed loop identical termination steps and returns within 1e-4 relative on gentle policies."""
import os
import random
import types

import numpy as np
import pytest
import torch

from oracle import actor as A, fast, refsig

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def wide_genomes(n, widths, activation, seed, out_gain=1.0):
    torch.manual_seed(seed)
    gs = []
    for _ in range(n):
        m = A.WideActor(widths, activation=activation)
        with torch.no_grad():
            m.net[-2].weight.mul_(out_gain)
            m.net[-2].bias.mul_(out_gain)
        gs.append(A.flatten(m))
    return np.stack(gs)


def refs(n, seed, **kw):
    lv, st = refsig.make_ref_params(n, seed_base=seed, **kw)
    return lv, st, torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV)


def modes_tensor(modes):
    from serl_b200 import rollout
    return torch.as_tensor(np.array([rollout.mode_code(m) for m in modes], dtype=np.int32), device=DEV)


@pytest.mark.parametrize('widths,activation', [([128] * 4, 'tanh'), ([256] * 4, 'elu'), ([108] * 4, 'tanh'),
                                               ([96, 200, 64, 320], 'relu'), ([64] * 9, 'tanh')])
def test_deep_forward_matches_torch_fp32(widths, activation):
    from serl_b200 import rollout
    g = wide_genomes(1, widths, activation, 3)[0]
    assert g.size == rollout.num_params_wide(widths)
    rs = np.random.RandomState(5)
    obs = np.concatenate([rs.randn(700, 7) * [0.05, 0.05, 0.01, 0.02, 0.02, 0.02, 0.05], rs.randn(300, 7), np.zeros((1, 7))]).astype(np.float32)
    got = rollout.actor_forward_wide(torch.as_tensor(g, device=DEV), widths, activation, torch.as_tensor(obs, device=DEV)).cpu().numpy()
    net = A.unflatten_wide(g, widths, activation)
    ref32 = net(torch.as_tensor(obs)).detach().numpy()
    ref64 = net.double()(torch.as_tensor(obs, dtype=torch.float64)).detach().numpy()
    err = np.abs(got - ref64).max()
    base = np.abs(ref32 - ref64).max()
    print('widths', widths, activation, 'max |tc - f64| %.2e   max |torch f32 - f64| %.2e' % (err, base))
    assert np.abs(got - ref32).max() <= 2e-5
    assert err <= max(4 * base, 5e-6)


@pytest.mark.parametrize('widths,activation', [([128] * 4, 'tanh'), ([108] * 4, 'elu'), ([256] * 4, 'tanh')])
def test_deep_closed_loop_against_the_c_episode_port(widths, activation):
    from serl_b200 import rollout
    w = wide_genomes(3, widths, activation, 11, out_gain=0.2)
    modes = ['nominal', 'ice', 'be', 'cg', 'sa', 'jr']
    lv, st, dlv, dst = refs(len(modes), 505)
    r = rollout.population_rollout(torch.as_tensor(w, device=DEV), rollout.actor_shape(72, 3, activation), dlv, dst, modes_tensor(modes),
                                   horizon=600, widths=widths)
    torch.cuda.synchronize()
    r.check()
    oret, ostp = fast.evaluate_population_wide(w, widths, lv, st, modes, activation=activation, horizon=600)
    ret, stp = r.returns.cpu().numpy(), r.steps.cpu().numpy()
    assert np.array_equal(stp, ostp), (stp, ostp)
    rel = np.abs(ret - oret) / np.abs(oret)
    print(widths, 'max rel return diff %.2e' % rel.max())
    assert rel.max() <= 1e-4, rel.max()
    assert np.allclose(r.fitness.cpu().numpy(), oret.mean(1), rtol=1e-4)


def test_k1_and_k1_tc_fly_the_same_h128_l3_genomes():
    """The reference Actor at h = 128, L = 3 through K1 (shape) and through K1-TC ([128] * 4): the same episodes"""
    from serl_b200 import rollout
    sh = rollout.actor_shape(128, 3, 'tanh')
    assert rollout.tc_widths(sh) is None                     # K1 flies it by default
    w = torch.as_tensor(wide_genomes(4, [128] * 4, 'tanh', 17, out_gain=0.2), device=DEV)
    modes = ['nominal', 'ice', 'be', 'cg', 'h2000-v150', 'se']
    _, _, dlv, dst = refs(len(modes), 71)
    md = modes_tensor(modes)
    k1 = rollout.population_rollout(w, sh, dlv, dst, md, horizon=800)
    tc = rollout.population_rollout(w, sh, dlv, dst, md, horizon=800, widths=[128] * 4)
    torch.cuda.synchronize()
    k1.check()
    tc.check()
    assert torch.equal(tc.steps, k1.steps)
    rel = ((tc.returns - k1.returns).abs() / k1.returns.abs()).max().item()
    assert rel <= 1e-4, rel


def test_constant_action_gives_bit_identical_steps_returns_and_traces_on_both_kernels():
    """Zero output weights: both kernels emit am_tanh1(bo), so the env / plant code they share must give the same bits, traces
    included, through the gust pulse of the `gust` and `test` builds"""
    from serl_b200 import rollout
    g = wide_genomes(1, [128] * 4, 'tanh', 3)[0]
    g[-3 - 3 * 128:-3] = 0.0
    g[-3:] = [0.02, -0.01, 0.01]
    w = torch.as_tensor(g[None], device=DEV)
    modes = ['gust', 'test', 'nominal', 'cg-timed', 'be', 'ice']
    _, _, dlv, dst = refs(len(modes), 77, t_max=25)
    md = modes_tensor(modes)
    sh = rollout.actor_shape(128, 3, 'tanh')
    run = lambda widths: rollout.population_rollout(w, sh, dlv, dst, md, horizon=2501, t_max=25.0, widths=widths, gust=True, trace=True,
                                                    actions=True)
    k1, tc = run(None), run([128] * 4)
    torch.cuda.synchronize()
    k1.check()
    tc.check()
    assert torch.equal(tc.steps, k1.steps) and torch.equal(tc.returns, k1.returns)
    assert torch.equal(tc.actions, k1.actions)
    steps = tc.steps.cpu().numpy()[0]
    assert (steps[:2] > 2301).all(), steps                  # the gust envs flew the whole pulse
    for e, k in enumerate(steps):
        assert torch.equal(tc.trace[0, e, :k], k1.trace[0, e, :k]), e
        assert torch.isfinite(tc.trace[0, e, :k]).all()


def test_more_tasks_than_slots_tiled_genomes_and_repeated_launches_are_deterministic():
    from serl_b200 import rollout
    widths = [160] * 4
    g = wide_genomes(3, widths, 'tanh', 21, out_gain=0.3)
    w = torch.as_tensor(np.tile(g, (120, 1)), device=DEV)
    _, _, dlv, dst = refs(256, 9)
    md = torch.zeros(256, dtype=torch.int32, device=DEV)
    sh = rollout.actor_shape(160, 3, 'tanh')
    assert rollout.tc_widths(sh) == widths
    runs = [rollout.population_rollout(w, sh, dlv, dst, md, horizon=40) for _ in range(2)]
    torch.cuda.synchronize()
    for r in runs:
        r.check()
    ret = runs[0].returns.cpu().numpy()
    assert np.isfinite(ret).all() and (runs[0].steps.cpu().numpy() == 40).all()
    for a in range(3, 360):
        assert np.array_equal(ret[a], ret[a % 3]), a
    assert torch.equal(runs[0].returns, runs[1].returns) and torch.equal(runs[0].steps, runs[1].steps)
    explicit = rollout.population_rollout(w, rollout.actor_shape(72), dlv, dst, md, horizon=40, widths=widths)
    torch.cuda.synchronize()
    assert torch.equal(explicit.returns, runs[0].returns)


def _agent(tmp_path, seed, test_ea):
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    from serl_b200.parameters import Parameters
    tmp_path.mkdir(exist_ok=True)
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        args = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=seed, pop_size=4, mut_type='normal', test_ea=test_ea))
    finally:
        os.chdir(cwd)
    args.save_foldername = str(tmp_path) + '/'
    args.state_dim, args.action_dim, args.hidden_size, args.num_layers = 7, 3, 256, 3
    args.learn_start, args.frac_frames_train = 300, 0. if test_ea else 0.2
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    return agent_mod.Agent(args, config.select_env('PHlab_attitude_nominal'))


EA_STATS = ('best_train_fitness', 'test_score', 'pop_avg', 'pop_min', 'avg_ep_len')      # smoothness: NaN unless requested


def _finite(stats):
    assert np.isfinite([float(stats[k]) for k in EA_STATS]).all(), stats


def _same(a, b):
    return a.keys() == b.keys() and all(np.array_equal(np.asarray(a[k], dtype=object if a[k] is None else float),
                                                       np.asarray(b[k], dtype=object if b[k] is None else float),
                                                       equal_nan=a[k] is not None) for k in a)


def test_agent_trains_an_h256_l3_actor(tmp_path):
    """Agent with hidden_size = 256, num_layers = 3: K1 cannot hold the genome, so every flight goes to K1-TC"""
    from serl_b200 import rollout
    runs = []
    for rep in range(2):
        ag = _agent(tmp_path / ('ea%d' % rep), 7, True)
        assert rollout.tc_widths(ag.shape) == [256] * 4
        before = ag.pop.genomes.clone()
        stats = [ag.train() for _ in range(2)]
        for s in stats:
            _finite(s)
        assert not torch.equal(before, ag.pop.genomes)
        runs.append(stats)
    assert all(_same(a, b) for a, b in zip(*runs)), runs
    ag = _agent(tmp_path / 'rl', 7, False)
    stats = ag.train()
    _finite(stats)
    assert len(ag.replay_buffer) > 0


def test_validate_agent_flies_an_h256_actor_over_80_s():
    from serl_b200 import evaluation, rollout, signals
    from serl_b200.envs import config
    w = wide_genomes(1, [256] * 4, 'tanh', 5, out_gain=0.2)
    t_max = 80
    times = np.linspace(0., t_max, 6)
    user = [(signals.SmoothedStepSequence(times, [0, 12, 3, -4, -8, 2], smooth_width=t_max // 10),
             signals.SmoothedStepSequence(times, [2, -2, 2, 10, 2, -6], smooth_width=t_max // 10))] * 2
    env = config.select_env('PHlab_attitude_nominal')
    env.set_eval_mode(t_max)
    sh = rollout.actor_shape(256, 3, 'tanh')
    data, stats = evaluation.validate_agent(w[0], sh, env, user, num_trails=1)
    assert np.isfinite(data).all() and np.isfinite([stats.nmae, stats.sm]).all()
    th, ph = user[0]
    lv, st = np.stack([th.levels, ph.levels])[None], np.stack([th.starts, ph.starts])[None]
    oret, ostp = fast.evaluate_population_wide(w, [256] * 4, lv, st, ['nominal'], t_max=float(t_max), smooth_w=float(th.smooth_width),
                                               horizon=int(round(t_max / 0.01)) + 1)
    assert data.shape[0] == ostp[0, 0]
    ret = data[:, -1].sum()
    assert abs(ret - oret[0, 0]) <= 1e-4 * abs(oret[0, 0]), (ret, oret)
