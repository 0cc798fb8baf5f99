"""Edge cases of the C-ABI on the GPU: degenerate sizes, multi-chunk env grids, argument errors, determinism."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import actor as A, phlab, refsig

pytestmark = pytest.mark.gpu
ACT = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'actors.npz'))


def run(w, hidden, lv, st, modes, horizon=2001, act='tanh'):
    from serl_b200 import rollout
    dev = torch.device('cuda:0')
    sh = rollout.actor_shape(hidden, 3, act)
    md = torch.tensor([rollout.mode_code(m) for m in modes], dtype=torch.int32, device=dev)
    r = rollout.population_rollout(torch.as_tensor(np.ascontiguousarray(w, dtype=np.float32), device=dev), sh,
                                   torch.as_tensor(lv, device=dev), torch.as_tensor(st, device=dev), md, horizon=horizon)
    torch.cuda.synchronize()
    return r


def test_single_actor_single_env_single_step():
    w = ACT['serl10_elite_h72_tanh'][None]
    lv, st = refsig.make_ref_params(1)
    r = run(w, 72, lv, st, ['nominal'], horizon=1)
    assert int(r.steps[0, 0]) == 1
    env = phlab.CitationEnv('nominal', 'auto')
    obs = env.reset(lv[0], st[0])
    _, rew, _, _ = env.step(A.unflatten(w[0], hidden=72).select_action(obs))
    assert abs(float(r.returns[0, 0]) - rew) < 1e-9


def test_env_grid_with_several_chunks_and_odd_population():
    """n_envs = 200 -> two env chunks per actor (second one ragged); pop = 5 -> last CTA holds one actor."""
    w = ACT['serl50_pop8_h32_tanh'][:5]
    lv, st = refsig.make_ref_params(200, seed_base=4242)
    r = run(w, 32, lv, st, ['nominal'] * 200, horizon=50)
    assert (r.steps.cpu().numpy() == 50).all()
    ret = r.returns.cpu().numpy()
    # env e of this launch == env 0 of a launch that only has env e
    for e in (0, 127, 128, 199):
        r1 = run(w, 32, lv[e:e + 1], st[e:e + 1], ['nominal'], horizon=50)
        assert np.array_equal(r1.returns.cpu().numpy()[:, 0], ret[:, e])       # bitwise: no cross-talk between lanes
    assert np.allclose(r.fitness.cpu().numpy(), ret.mean(1), rtol=1e-12)


def test_hidden_64_goes_through_the_warp_kernel():
    torch.manual_seed(3)
    w = np.stack([A.flatten(A.Actor(hidden=64)) for _ in range(2)])
    lv, st = refsig.make_ref_params(2, seed_base=9)
    r = run(w, 64, lv, st, ['nominal', 'ice'])
    env = {m: phlab.CitationEnv(m, 'auto') for m in ('nominal', 'ice')}
    for a in range(2):
        for e, m in enumerate(('nominal', 'ice')):
            o = phlab.run_episode(env[m], A.unflatten(w[a], hidden=64), lv[e], st[e])
            assert int(r.steps[a, e]) == o['steps']
            assert abs(float(r.returns[a, e]) - o['fitness']) <= 1e-4 * abs(o['fitness'])


def test_hidden_128_runs_with_tables_in_global_memory():
    """h = 128: the 207 KB genome fills shared memory, plant tables are read through L1 (kernel variant TABS=false)."""
    torch.manual_seed(11)
    w = np.stack([A.flatten(A.Actor(hidden=128)) for _ in range(2)])
    lv, st = refsig.make_ref_params(2, seed_base=19)
    r = run(w, 128, lv, st, ['nominal', 'cg'])
    env = {m: phlab.CitationEnv(m, 'auto') for m in ('nominal', 'cg')}
    for a in range(2):
        for e, m in enumerate(('nominal', 'cg')):
            o = phlab.run_episode(env[m], A.unflatten(w[a], hidden=128), lv[e], st[e])
            assert int(r.steps[a, e]) == o['steps']
            assert abs(float(r.returns[a, e]) - o['fitness']) <= 1e-4 * abs(o['fitness'])


def test_repeat_launches_are_bitwise_deterministic():
    w = ACT['serl10_pop_h72_tanh'][:3]
    lv, st = refsig.make_ref_params(5, seed_base=77)
    modes = ['nominal', 'be', 'ice', 'sa', 'cg']
    a = run(w, 72, lv, st, modes, horizon=300).returns.cpu().numpy()
    b = run(w, 72, lv, st, modes, horizon=300).returns.cpu().numpy()
    assert np.array_equal(a, b)


def test_rollout_run_argument_errors_are_reported():
    from serl_b200 import _native, rollout
    L = _native.lib()
    sh = rollout.actor_shape(72)
    dev = torch.device('cuda:0')
    w = torch.zeros((1, rollout.num_params(sh)), device=dev)
    lv = torch.zeros((1, 2, 6), dtype=torch.float64, device=dev)
    md = torch.zeros(1, dtype=torch.int32, device=dev)
    ret = torch.zeros((1, 1), dtype=torch.float64, device=dev)
    stp = torch.zeros((1, 1), dtype=torch.int32, device=dev)

    def run(weights, pop, shape):
        d = _native.RolloutDesc()
        d.d_weights, d.pop, d.shape = weights, pop, shape
        d.d_ref_levels, d.d_ref_starts, d.d_env_mode, d.n_envs, d.horizon = lv.data_ptr(), lv.data_ptr(), md.data_ptr(), 1, 10
        d.d_returns, d.d_steps = ret.data_ptr(), stp.data_ptr()
        return L.serl_rollout_run(ctypes.byref(d), None)
    rc = run(None, 1, sh)
    assert rc == -1 and b'null pointer' in L.serl_last_error()
    rc = run(w.data_ptr(), 0, sh)
    assert rc == -1
    bad = rollout.actor_shape(72); bad.state_dim = 9
    rc = run(w.data_ptr(), 1, bad)
    assert rc == -1 and b'state_dim' in L.serl_last_error()
    big = rollout.actor_shape(160)
    wb = torch.zeros((1, rollout.num_params(big)), device=dev)
    rc = run(wb.data_ptr(), 1, big)
    assert rc == -3          # SERL_ERR_UNSUPPORTED: a h=160 genome (324 KB) does not fit in shared memory
    with pytest.raises(_native.NativeError):
        _native.check(rc, 'serl_rollout_run')
    assert L.serl_ssne_select(None, 4, None, 0, None, None, None) == -1


@pytest.mark.parametrize('pop,n_envs,hidden,key', [(50, 64, 32, 'serl50_pop8_h32_tanh'), (512, 128, 72, 'serl10_pop_h72_tanh')])
def test_baseline_config_sizes_through_size_independent_properties(pop, n_envs, hidden, key):
    """BASELINE configs 2 and 3 at full size (too big for the oracle): determinism, duplicate genomes -> duplicate rows,
    env-permutation equivariance (returns columns permute exactly), fitness = row mean, step bounds."""
    base = ACT[key]
    w = base[np.arange(pop) % base.shape[0]].copy()
    lv, st = refsig.make_ref_params(n_envs, seed_base=31337)
    modes = ['nominal'] * n_envs
    r1 = run(w, hidden, lv, st, modes)
    ret, stp = r1.returns.cpu().numpy(), r1.steps.cpu().numpy()
    assert np.isfinite(ret).all() and (stp >= 1).all() and (stp <= 2001).all()
    nb = base.shape[0]
    assert np.array_equal(ret[:nb], ret[nb:2 * nb]) and np.array_equal(stp[:nb], stp[nb:2 * nb])      # duplicated genomes
    assert np.allclose(r1.fitness.cpu().numpy(), ret.mean(1), rtol=1e-12, atol=0)
    perm = np.random.RandomState(0).permutation(n_envs)
    r2 = run(w, hidden, lv[perm], st[perm], modes)
    assert np.array_equal(r2.returns.cpu().numpy(), ret[:, perm])                                    # equivariance + determinism
    assert np.array_equal(r2.steps.cpu().numpy(), stp[:, perm])
