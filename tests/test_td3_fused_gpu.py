"""K7, the fused TD3 learner (csrc/td3.cu, serl_b200/td3_fused.py), on the GPU.  Every launch records its random draws
(batch rows, clipped target-policy noise, CAPS uniforms) and the fp32 oracle (oracle/td3.py: TD3.update_parameters with
the draws given, on the CPU) replays them.  The kernel's summation order is not torch's, so the comparison is a tolerance:
  * one step: losses to 1e-5 relative; Adam first moments per tensor to 1e-4 x that tensor's max |m|; parameters and targets
    to 1e-3 lr on >= 99.9 % of the elements and 2 lr everywhere (Adam's first step is sign-like where a gradient is within
    rounding of zero);
  * 300 steps on replay rows of a real K1 flight: the td / pg series to 1e-5 relative over the first 50 steps, 1e-4 over all
    (measured on an H100: at most 7e-7 over all 300);
and bitwise: cluster sizes 1, 2, 4, 8, repeated launches and split launches give identical bits."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import td3 as O

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def td3_args(hidden=72, num_layers=3, activation='tanh', use_caps=True, device='cuda', lr=0.00018643512599969097):
    return types.SimpleNamespace(device=torch.device(device), individual_bs=100, hidden_size=hidden, num_layers=num_layers,
                                 activation_actor=activation, state_dim=7, action_dim=3, lr=lr, gamma=0.98, tau=0.005,
                                 noise_sd=0.2962183114680794, noise_clip=0.5, policy_update_freq=3, use_caps=use_caps,
                                 batch_size=86, seed=7)


def synthetic_rows(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn((n, 19), generator=g) * 0.3
    rows[:, 7:10] = torch.rand((n, 3), generator=g) * 2 - 1
    rows[:, 17] = -torch.rand(n, generator=g)
    rows[:, 18] = (torch.rand(n, generator=g) < 0.05).float()
    return rows


def flight_rows():
    """replay rows (the stored transitions) of one K1 flight of the ten golden SERL10 actors"""
    from oracle import refsig
    from serl_b200 import rollout
    acts = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'actors.npz'))
    g = torch.as_tensor(acts['serl10_pop_h72_tanh'], device=DEV)
    lv, st = refsig.make_ref_params(1)
    md = torch.tensor([rollout.mode_code('nominal')], dtype=torch.int32, device=DEV)
    r = rollout.population_rollout(g, rollout.actor_shape(72), torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV), md,
                                   replay_env=0)
    steps = r.steps[:, 0].cpu()
    rows = torch.cat([r.replay[i, :int(steps[i]), :19] for i in range(g.shape[0])]).contiguous()
    assert rows.shape[0] > 2000 and torch.isfinite(rows).all()
    return rows


def fused_and_oracle(args):
    """a FusedTD3 and a CPU TD3 holding the same weights (fresh Adam state in both)"""
    from serl_b200.core.td3 import TD3
    from serl_b200.td3_fused import FusedTD3
    torch.manual_seed(11)
    f = FusedTD3(args)
    ora = TD3(types.SimpleNamespace(**dict(vars(args), device=torch.device('cpu'))))
    for mf, mo in ((f.actor, ora.actor), (f.actor_target, ora.actor_target), (f.critic, ora.critic), (f.critic_target, ora.critic_target)):
        for pf, po in zip(mf.parameters(), mo.parameters()):
            po.data.copy_(pf.data.cpu())
    return f, ora


def replay_oracle(ora, rows_cpu, launch, first_iteration, champion, use_caps):
    idx, noise, caps = launch.indices.cpu().long(), launch.noise.cpu(), launch.caps.cpu()
    out = []
    for k in range(idx.shape[0]):
        pg, td = O.update_parameters(ora, rows_cpu[idx[k]], first_iteration + k, noise[k], caps[k] if use_caps else None, champion)
        out.append((float(td), float('nan') if pg is None else float(pg)))
    return np.array(out)


def moments(opt, params):
    return [opt.state[p]['exp_avg'] if p in opt.state else torch.zeros_like(p) for p in params]


def views(flat, params):
    out, off = [], 0
    for p in params:
        out.append(flat[off:off + p.numel()].view(p.shape).cpu())
        off += p.numel()
    return out


@pytest.mark.parametrize('hidden,num_layers', [(32, 1), (72, 3), (128, 1), (128, 3), (32, 3), (72, 1)])
@pytest.mark.parametrize('activation', ['tanh', 'elu', 'relu'])
@pytest.mark.parametrize('iteration', [1, 3])
@pytest.mark.parametrize('use_caps,champion', [(True, False), (False, True), (True, True), (False, False)])
def test_one_step_matches_the_oracle(hidden, num_layers, activation, iteration, use_caps, champion):
    args = td3_args(hidden, num_layers, activation, use_caps)
    f, ora = fused_and_oracle(args)
    rows = synthetic_rows(3000, seed=hidden + num_layers)
    r = f.run(rows.to(DEV), rows.shape[0], 1, iteration, champion, record=True)
    r.check()
    got = r.losses.cpu().numpy()
    want = replay_oracle(ora, rows, r, iteration, champion, use_caps)
    assert np.isnan(got[0, 1]) == (iteration % 3 != 0)
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-7)
    lr = args.lr
    pa = sum(p.numel() for p in ora.actor.parameters())
    pc = sum(p.numel() for p in ora.critic.parameters())
    st = f.state
    ma, mc = st[2 * pa:3 * pa], st[4 * pa + 2 * pc:4 * pa + 3 * pc]
    for flat, opt, mod in ((mc, ora.critic_optim, ora.critic), (ma, ora.actor_optim, ora.actor)):
        for k, (mk, mo) in enumerate(zip(views(flat, list(mod.parameters())), moments(opt, list(mod.parameters())))):
            assert (mk - mo).abs().max() <= 1e-4 * mo.abs().max() + 1e-30, (k, (mk - mo).abs().max(), mo.abs().max())
    for mf, mo in ((f.actor, ora.actor), (f.actor_target, ora.actor_target), (f.critic, ora.critic), (f.critic_target, ora.critic_target)):
        d = torch.cat([(pf.detach().cpu() - po.detach()).reshape(-1).abs() for pf, po in zip(mf.parameters(), mo.parameters())])
        assert d.max() <= 2 * lr and (d <= 1e-3 * lr).float().mean() >= 0.999, (d.max(), (d > 1e-3 * lr).sum())


def test_300_steps_on_flight_rows_track_the_oracle():
    args = td3_args()
    f, ora = fused_and_oracle(args)
    rows = flight_rows()
    r = f.run(rows, rows.shape[0], 300, 1, False, record=True)
    r.check()
    got = r.losses.cpu().numpy()
    want = replay_oracle(ora, rows.cpu(), r, 1, False, True)
    rel = np.abs(got - want) / np.maximum(np.abs(want), 1e-6)
    td_rel, pg_rel = rel[:, 0], rel[2::3, 1]          # actor steps: iterations 3, 6, ...
    print('td rel max first 50 %.2e all %.2e; pg rel max first 50 %.2e all %.2e'
          % (td_rel[:50].max(), td_rel.max(), pg_rel[:17].max(), pg_rel.max()))
    assert np.isnan(got[:, 1]).sum() == 200
    assert td_rel[:50].max() <= 1e-5 and pg_rel[:17].max() <= 1e-5
    assert td_rel.max() <= 1e-4 and pg_rel.max() <= 1e-4


def test_cluster_size_repeated_and_split_launches_are_bitwise_identical():
    args = td3_args()
    from serl_b200.td3_fused import FusedTD3
    torch.manual_seed(5)
    f = FusedTD3(args)
    rows = synthetic_rows(5000, seed=3).to(DEV)
    s0 = f.state.clone()

    def go(plan, cs):
        f.state.copy_(s0)
        f.critic_steps = f.actor_steps = 0
        first, losses = 1, []
        for n in plan:
            losses.append(f.run(rows, rows.shape[0], n, first, False, cluster_size=cs).losses)
            first += n
        torch.cuda.synchronize()
        return f.state.clone(), torch.cat(losses)

    ref_state, ref_loss = go([40], 1)
    assert torch.isfinite(ref_loss[:, 0]).all()
    for cs in (2, 4, 8):
        s, l = go([40], cs)
        assert torch.equal(s, ref_state) and torch.equal(l.nan_to_num(7.0), ref_loss.nan_to_num(7.0)), cs
    s, l = go([40], 8)
    assert torch.equal(s, ref_state)                                    # two identical launches
    s, l = go([17, 23], 4)                                              # n = n1 + n2 in two launches
    assert torch.equal(s, ref_state) and torch.equal(l.nan_to_num(7.0), ref_loss.nan_to_num(7.0))


def test_sampler_draws_distinct_uniform_rows_and_honours_given_indices():
    from scipy import stats
    args = td3_args(hidden=32, num_layers=1, use_caps=False)
    from serl_b200.td3_fused import FusedTD3
    f = FusedTD3(args)
    n = 1000
    rows = synthetic_rows(n, seed=9).to(DEV)
    r = f.run(rows, n, 2000, 1, False, record=True)
    idx = r.indices.cpu().numpy()
    assert idx.min() >= 0 and idx.max() < n
    assert all(len(np.unique(b)) == b.size for b in idx)
    counts = np.bincount(idx.reshape(-1), minlength=n)
    p = stats.chisquare(counts).pvalue
    assert p > 1e-4, p
    # the rows a given index array names are the rows the step uses
    given = torch.as_tensor(np.stack([np.random.RandomState(k).permutation(n)[:86] for k in range(3)]), dtype=torch.int32, device=DEV)
    r2 = f.run(rows, n, 3, 1, False, indices=given, record=True)
    assert torch.equal(r2.indices, given)


def test_agent_with_fused_td3_trains_through_live_views(tmp_path):
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    from serl_b200.parameters import Parameters
    from serl_b200.td3_fused import FusedTD3
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        args = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=7, pop_size=4, mut_type='normal', test_ea=False,
                                                fused_td3=True))
    finally:
        os.chdir(cwd)
    args.save_foldername = str(tmp_path) + '/'
    args.state_dim, args.action_dim, args.hidden_size = 7, 3, 32
    args.learn_start, args.frac_frames_train = 300, 0.2
    torch.manual_seed(7)
    ag = agent_mod.Agent(args, config.select_env('PHlab_attitude_nominal'))
    assert isinstance(ag.rl_agent, FusedTD3)
    assert ag.evolver.critic is ag.rl_agent.critic
    before = torch.cat([p.detach().reshape(-1) for p in ag.rl_agent.actor.parameters()]).clone()
    for _ in range(2):
        stats = ag.train()
    assert np.isfinite(stats['TD_loss']) and np.isfinite(stats['PG_obj'])
    assert ag.rl_iteration > 0
    after = torch.cat([p.detach().reshape(-1) for p in ag.rl_agent.actor.parameters()])
    assert not torch.equal(before, after)
    # a critic weight edited through the module is what the next launch reads
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
    # the checkpoint keys are the torch learner's
    ag.save_agent(args, elite_index=0)
    sd = torch.load(os.path.join(args.save_foldername, 'rl_net.pkl'))
    from serl_b200.core.genetic_agent import Actor
    assert list(sd) == list(Actor(args).state_dict())
