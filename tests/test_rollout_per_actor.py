"""Per-actor env blocks without a GPU: the C-ABI refuses the combinations the kernels do not take before any CUDA call, the
Agent's reference draws follow the reference's evaluation loop, and the Sweep's launch-group rule."""
import ctypes
import os
import re
import types

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_constant_matches_the_binding():
    from serl_b200 import _native
    text = open(os.path.join(ROOT, 'include', 'serl_b200.h')).read()
    bits = {k: int(v) for k, v in re.findall(r'#define (SERL_ROLLOUT_[A-Z_]+) (\d+)', text)}
    assert bits['SERL_ROLLOUT_PER_ACTOR_REFS'] == _native.ROLLOUT_PER_ACTOR_REFS
    assert len(set(bits.values())) == len(bits) and all(v & (v - 1) == 0 for v in bits.values())      # distinct single bits


@pytest.mark.parametrize('widths', [None, [128, 128]])
@pytest.mark.parametrize('field', ['d_env_order', 'd_track'])
def test_per_actor_refs_refuse_env_order_and_track_before_any_cuda_call(widths, field):
    """K1 and K1-TC: SERL_ERR_ARG, no kernel launched, and the device pointers (fake, non-null) are never read"""
    from serl_b200 import build, _native, rollout
    build.build()
    L = _native.lib()
    warr = (ctypes.c_int32 * 2)(*(widths or [0, 0]))
    d = _native.RolloutDesc()
    fake = iter(range(0x10000, 0x100000, 0x1000))
    for f in ('d_weights', 'd_ref_levels', 'd_ref_starts', 'd_env_mode', 'd_returns', 'd_steps', 'd_replay', 'd_status'):
        setattr(d, f, next(fake))
    d.pop, d.shape, d.n_envs, d.horizon, d.replay_env = 4, rollout.actor_shape(72), 8, 100, 0
    if widths:
        d.widths, d.n_widths = ctypes.cast(warr, ctypes.c_void_p), 2
    d.flags = _native.ROLLOUT_PER_ACTOR_REFS | _native.ROLLOUT_GUST
    setattr(d, field, next(fake))
    launches = L.serl_launch_count()
    rc = L.serl_rollout_run(ctypes.byref(d), None)
    assert rc == -1, (rc, L.serl_last_error())
    assert 'PER_ACTOR_REFS' in L.serl_last_error().decode()
    assert L.serl_launch_count() == launches


def _env(name='PHlab_attitude_nominal'):
    from serl_b200.envs import config
    return config.select_env(name)


def _agent_draws(args, env, pop):
    """Agent._draw_population on a stand-in Agent (the real one needs a device)"""
    from serl_b200.core import agent as agent_mod
    me = types.SimpleNamespace(args=args, env=env, pop=[None] * pop)
    me._n_envs = lambda: int(args.num_envs)
    return agent_mod.Agent._draw_population(me)


def test_independent_draws_follow_the_reference_evaluation_loop():
    """pop 4 x 3 envs: the draw_reference() sequence of `for net in pop: for i in range(num_evals): reset()`
    (base/core/agent.py:234-241; every reset() draws through init_ref), laid out [actor, env]; off: today's n_envs draws"""
    pop, n_envs = 4, 3
    env = _env()
    np.random.seed(11)
    want = []
    for _net in range(pop):
        for _i in range(n_envs):
            want.append(env.draw_reference())
    after = np.random.get_state()[1].copy(), np.random.get_state()[2]
    args = types.SimpleNamespace(num_envs=n_envs, independent_references=True)
    np.random.seed(11)
    d = _agent_draws(args, env, pop)
    assert np.array_equal(np.random.get_state()[1], after[0]) and np.random.get_state()[2] == after[1]
    assert d.levels.shape == d.starts.shape == (pop, n_envs, 2, 6)
    for a in range(pop):
        for e in range(n_envs):
            assert np.array_equal(d.levels[a, e], want[a * n_envs + e][0]) and np.array_equal(d.starts[a, e], want[a * n_envs + e][1])
    # off: the n_envs draws every actor shares, exactly the first n_envs of the same stream
    args.independent_references = False
    np.random.seed(11)
    d = _agent_draws(args, env, pop)
    assert d.levels.shape == (n_envs, 2, 6)
    for e in range(n_envs):
        assert np.array_equal(d.levels[e], want[e][0]) and np.array_equal(d.starts[e], want[e][1])
    np.random.seed(11)
    _agent_draws(args, env, pop)
    state_agent = np.random.get_state()[1].copy()
    np.random.seed(11)
    for _ in range(n_envs):
        env.draw_reference()
    assert np.array_equal(state_agent, np.random.get_state()[1])


def test_parameters_and_cli_carry_the_option(tmp_path, monkeypatch):
    from serl_b200.parameters import Parameters
    monkeypatch.chdir(tmp_path)
    assert Parameters(types.SimpleNamespace()).independent_references is False
    assert Parameters(types.SimpleNamespace(independent_refs=True)).independent_references is True
    import sys
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    try:
        from train import parser
    finally:
        sys.path.pop(0)
    assert parser.parse_args(['-frames', '1', '-independent_refs']).independent_refs is True
    assert parser.parse_args(['-frames', '1']).independent_refs is False


def _params(tmp_path, monkeypatch, **kw):
    from serl_b200.parameters import Parameters
    monkeypatch.chdir(tmp_path)
    p = Parameters(types.SimpleNamespace(env='PHlab_attitude_nominal', seed=7, pop_size=kw.pop('pop_size', 4), mut_type='normal',
                                         test_ea=False, fused_td3=True))
    p.state_dim, p.action_dim, p.hidden_size = 7, 3, 32
    p.num_envs = p.num_evals = 2
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def test_sweep_launch_groups(tmp_path, monkeypatch):
    """runs share a population launch when shape, num_envs, horizon / t_max, gust, the smoothness actions and the stored
    transitions agree; seeds, learning rates, CAPS, fault modes and independent draws do not split a group; pop_size = 0
    joins none"""
    from serl_b200.core.agent import population_key
    from serl_b200.sweep import launch_groups
    long_env = _env()
    long_env.t_max = 40
    runs = [
        (_params(tmp_path, monkeypatch), _env()),                                          # 0
        (_params(tmp_path, monkeypatch, lr=4e-4, use_caps=False), _env('PHlab_attitude_be')),   # 1: same group as 0
        (_params(tmp_path, monkeypatch, num_envs=3), _env()),                              # 2
        (_params(tmp_path, monkeypatch), long_env),                                        # 3: t_max 40 -> horizon 4001
        (_params(tmp_path, monkeypatch), _env('PHlab_attitude_gust')),                     # 4
        (_params(tmp_path, monkeypatch, smooth_fitness=True), _env()),                     # 5
        (_params(tmp_path, monkeypatch, pop_size=0, smooth_fitness=False), _env()),         # 6: no population
        (_params(tmp_path, monkeypatch, independent_references=True), _env('PHlab_attitude_ice')),  # 7: same group as 0
        (_params(tmp_path, monkeypatch, frac_frames_train=0.0), _env()),                   # 8: stores no transitions
        (_params(tmp_path, monkeypatch, num_envs=3), _env('PHlab_attitude_jr')),           # 9: with 2
    ]
    keys = [population_key(p, e) for p, e in runs]
    assert keys[6] is None
    assert launch_groups(keys) == [[0, 1, 7], [2, 9], [3], [4], [5], [8]]
    assert launch_groups([None, None]) == []
