"""K7's group launch (serl_td3_learn, td3_fused.train_group) and the sweep driver (serl_b200/sweep.py) on the GPU.
Every comparison is bitwise against the same learners trained alone (FusedTD3.run, Agent.train) from copies of the same
initial state: the learner state, the losses, the recorded draws (batch rows, target noise, CAPS uniforms), the status
word and the Adam step counts."""
import os
import random
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def synthetic_rows(n, seed, cols=19):
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn((n, cols), generator=g) * 0.3
    rows[:, 7:10] = torch.rand((n, 3), generator=g) * 2 - 1
    rows[:, 17] = -torch.rand(n, generator=g)
    rows[:, 18] = (torch.rand(n, generator=g) < 0.05).float()
    return rows.to(DEV)


# learners that differ in everything a group lets differ: seed, lr, gamma, tau, noise, policy_update_freq, CAPS, champion
# target, batch, n_steps, replay rows / n_valid / row stride, first iteration and Adam step counts
SPECS = [
    dict(seed=7, lr=0.00018643512599969097, gamma=0.98, tau=0.005, noise_sd=0.2962, freq=3, caps=True, champ=False, batch=86,
         n=300, n_valid=3000, cols=19, first=1),
    dict(seed=8, lr=4e-4, gamma=0.99, tau=0.01, noise_sd=0.2, freq=2, caps=False, champ=True, batch=32, n=517, n_valid=1500,
         cols=20, first=11),
    dict(seed=9, lr=1e-3, gamma=0.95, tau=0.02, noise_sd=0.1, freq=3, caps=True, champ=True, batch=128, n=1, n_valid=128,
         cols=19, first=3),
    dict(seed=10, lr=3e-4, gamma=0.9, tau=0.005, noise_sd=0.3, freq=2, caps=False, champ=False, batch=86, n=0, n_valid=500,
         cols=19, first=1),
    dict(seed=11, lr=2e-4, gamma=0.97, tau=0.003, noise_sd=0.25, freq=3, caps=True, champ=False, batch=128, n=300, n_valid=2500,
         cols=20, first=40),
    dict(seed=12, lr=6e-4, gamma=0.98, tau=0.008, noise_sd=0.15, freq=2, caps=False, champ=True, batch=32, n=129, n_valid=700,
         cols=19, first=7),
]


def learner(spec, hidden=72, num_layers=3, cluster_size=0):
    """a FusedTD3 of `spec`, its weights drawn from torch's CPU generator seeded with spec['seed'] (the same every call)"""
    from serl_b200.td3_fused import FusedTD3
    args = types.SimpleNamespace(device=DEV, individual_bs=100, hidden_size=hidden, num_layers=num_layers, activation_actor='tanh',
                                 state_dim=7, action_dim=3, lr=spec['lr'], gamma=spec['gamma'], tau=spec['tau'],
                                 noise_sd=spec['noise_sd'], noise_clip=0.5, policy_update_freq=spec['freq'], use_caps=spec['caps'],
                                 batch_size=spec['batch'], seed=spec['seed'])
    torch.manual_seed(spec['seed'])
    f = FusedTD3(args, cluster_size=cluster_size)
    f.critic_steps = spec['first'] - 1
    f.actor_steps = (spec['first'] - 1) // spec['freq']
    return f


def replay(spec):
    return synthetic_rows(3000, spec['seed'], spec['cols'])[:spec['n_valid']]


def solo(specs, **kw):
    out = []
    for s in specs:
        f = learner(s, **kw)
        r = f.run(replay(s), s['n_valid'], s['n'], s['first'], s['champ'], record=True)
        out.append((f, r))
    torch.cuda.synchronize()
    return out


def group(specs, record=True, **kw):
    from serl_b200 import td3_fused
    fs = [learner(s, **kw) for s in specs]
    rs = td3_fused.train_group(fs, [replay(s) for s in specs], [s['n'] for s in specs], [s['first'] for s in specs],
                               [s['champ'] for s in specs], record=record)
    torch.cuda.synchronize()
    return list(zip(fs, rs))


def assert_same(a, b, record=True):
    (fa, ra), (fb, rb) = a, b
    assert torch.equal(fa.state, fb.state)
    assert torch.equal(ra.losses.nan_to_num(7.0), rb.losses.nan_to_num(7.0))
    if record:
        assert torch.equal(ra.indices, rb.indices) and torch.equal(ra.noise, rb.noise) and torch.equal(ra.caps, rb.caps)
    assert int(ra.status.item()) == int(rb.status.item()) == 0
    assert (fa.critic_steps, fa.actor_steps) == (fb.critic_steps, fb.actor_steps)


def test_group_equals_solo_runs_bit_for_bit():
    ref = solo(SPECS)
    assert all(torch.isfinite(r.losses[:, 0]).all() for _, r in ref)
    got = group(SPECS)
    for a, b in zip(ref, got):
        assert_same(a, b)
    # the learner with no steps is untouched
    assert torch.equal(got[3][0].state, learner(SPECS[3]).state)
    # group losses come back in one copy, equal to each learner's own
    from serl_b200 import td3_fused
    for h, (_, r) in zip(td3_fused.group_losses([r for _, r in got]), got):
        assert np.array_equal(np.nan_to_num(h, nan=7.0), r.losses.nan_to_num(7.0).cpu().numpy())


def test_group_order_and_cluster_size_do_not_change_the_bits():
    ref = solo(SPECS)
    perm = [4, 0, 5, 2, 3, 1]
    got = group([SPECS[i] for i in perm])
    for j, i in enumerate(perm):
        assert_same(ref[i], got[j])
    for cs in (1, 2, 4, 8):
        got = group(SPECS[:3] + SPECS[4:], cluster_size=cs)
        for a, b in zip(ref[:3] + ref[4:], got):
            assert_same(a, b)


def test_wide_group_equals_solo_runs():
    specs = [dict(SPECS[0], n=40), dict(SPECS[1], n=25), dict(SPECS[2], n=0), dict(SPECS[4], n=33)]
    ref = solo(specs, hidden=256, num_layers=3)
    got = group(specs, hidden=256, num_layers=3)
    for a, b in zip(ref, got):
        assert_same(a, b)


def test_full_group_runs_in_waves_and_matches():
    """SERL_TD3_MAX_GROUP learners of 8 CTAs: more clusters than the GPU holds at once"""
    from serl_b200 import _native
    G = _native.TD3_MAX_GROUP
    specs = [dict(SPECS[k % len(SPECS)], seed=100 + k, n=1 + k % 4) for k in range(G)]
    got = group(specs, record=False, cluster_size=8)
    sample = [0, 5, 17, 40, G - 1]
    ref = solo([specs[k] for k in sample], cluster_size=8)
    for k, a in zip(sample, ref):
        assert_same(a, got[k], record=False)


def test_group_split_into_chunks_and_launches_equals_one_launch(monkeypatch):
    from serl_b200 import _native, td3_fused
    one = group(SPECS)
    before = _native.lib().serl_launch_count()
    monkeypatch.setattr(td3_fused, 'LAUNCH_STEPS', 100)
    monkeypatch.setattr(_native, 'TD3_MAX_GROUP', 2)
    split = group(SPECS)
    # ceil(517 / 100) = 6 chunks; learners with steps left per chunk: 5, 4, 3, 1, 1, 1 -> 3 + 2 + 2 + 1 + 1 + 1 launches
    assert _native.lib().serl_launch_count() - before == 10
    for a, b in zip(one, split):
        assert_same(a, b)


def test_bad_index_in_one_learn_call_sets_only_its_learners_status():
    from serl_b200 import _native
    specs = [dict(s, n=5) for s in SPECS[:3]]
    fs = [learner(s) for s in specs]
    rs, descs = [], (_native.TD3Desc * 3)()
    rows = [replay(s) for s in specs]
    bad = torch.zeros((5, specs[1]['batch']), dtype=torch.int32, device=DEV)
    bad[2, 7] = specs[1]['n_valid']                       # one past the valid rows
    for j, (f, s) in enumerate(zip(fs, specs)):
        r = f._launch(5, False)
        rs.append(r)
        descs[j] = f._desc(rows[j], s['n_valid'], 5, s['first'], s['champ'], bad if j == 1 else None, r, 0)
    _native.call('serl_td3_learn', descs, None, 3, device=DEV)
    torch.cuda.synchronize()
    assert [int(r.status.item()) for r in rs] == [0, _native.TD3_STATUS_INDEX, 0]
    with pytest.raises(_native.NativeError):
        rs[1].check()


# ---------------------------------------------------------------------------------------------------------------- Sweep
def _run_params(tmp_path, seed, **kw):
    from serl_b200.parameters import Parameters
    cwd = os.getcwd()
    os.chdir(tmp_path)
    try:
        p = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=seed, pop_size=kw.pop('pop_size', 4),
                                             mut_type='normal', test_ea=False, fused_td3=True))
    finally:
        os.chdir(cwd)
    p.save_foldername = str(tmp_path) + '/'
    p.state_dim, p.action_dim, p.hidden_size = 7, 3, 32
    p.num_envs = p.num_evals = 2                # num_evals: Parameters sets it only with a population
    p.learn_start, p.frac_frames_train = 300, 0.2
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _snapshot(ag, stats):
    return dict(stats=stats, num_frames=ag.num_frames, rl_iteration=ag.rl_iteration, state=ag.rl_agent.state.clone(),
                genomes=ag.pop.genomes.clone() if len(ag.pop) else None,
                replay=ag.replay_buffer.data[:len(ag.replay_buffer)].clone())


def _same_stats(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        x, y = np.asarray(a[k], dtype=np.float64), np.asarray(b[k], dtype=np.float64)
        assert np.array_equal(x, y, equal_nan=True), (k, a[k], b[k])


def test_sweep_runs_equal_the_same_runs_trained_alone(tmp_path):
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    from serl_b200.sweep import Sweep
    kws = [dict(), dict(lr=4e-4, use_caps=False), dict(pop_size=0, smooth_fitness=False)]
    seeds = [7, 8, 9]
    gens = 3
    random.seed(123); np.random.seed(123); torch.manual_seed(123)
    outer = (random.getstate(), np.random.get_state()[1].copy(), torch.get_rng_state())
    cuda_rng = torch.cuda.get_rng_state()
    sw = Sweep([(_run_params(tmp_path, s, **dict(kw)), config.select_env('PHlab_attitude_nominal')) for s, kw in zip(seeds, kws)])
    swept = [[] for _ in seeds]
    for _ in range(gens):
        for i, st in enumerate(sw.train()):
            swept[i].append(_snapshot(sw.runs[i].agent, st))
    # the caller's generators are untouched, and nothing drew from torch's default CUDA generator
    assert random.getstate() == outer[0] and np.array_equal(np.random.get_state()[1], outer[1])
    assert torch.equal(torch.get_rng_state(), outer[2])
    assert torch.equal(torch.cuda.get_rng_state(), cuda_rng)
    for seed, r in zip(seeds, sw.runs):
        torch.cuda.manual_seed(seed)
        assert torch.equal(r.rng.cuda, torch.cuda.get_rng_state())   # seeded like base/train.py, then never drawn from
    assert all(s[-1]['rl_iteration'] > 0 for s in swept)           # K7 stepped in every run
    for i, (seed, kw) in enumerate(zip(seeds, kws)):
        p = _run_params(tmp_path, seed, **dict(kw))
        env = config.select_env('PHlab_attitude_nominal')
        env.seed(p.seed)
        torch.manual_seed(p.seed)
        np.random.seed(p.seed)
        random.seed(p.seed)
        ag = agent_mod.Agent(p, env)
        for g in range(gens):
            a, b = swept[i][g], _snapshot(ag, ag.train())
            _same_stats(a['stats'], b['stats'])
            assert a['num_frames'] == b['num_frames'] and a['rl_iteration'] == b['rl_iteration'], (i, g)
            assert torch.equal(a['state'], b['state']), (i, g)
            assert torch.equal(a['replay'], b['replay']), (i, g)
            assert (a['genomes'] is None) == (b['genomes'] is None)
            if a['genomes'] is not None:
                assert torch.equal(a['genomes'], b['genomes']), (i, g)
    sw.save_agent(str(tmp_path / 'sweep'))
    for i in range(len(seeds)):
        assert os.path.exists(os.path.join(str(tmp_path), 'sweep', 'run%d' % i, 'rl_net.pkl'))
