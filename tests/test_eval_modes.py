"""The evaluation suite and the operator study for incremental and symmetric control, without a GPU: the symmetric nMAE
rule, which conditions an actor of each control mode may fly, the SERL_ROLLOUT_SUITE descriptor rules, the CLIs' -env
grammar, and base/evaluate.py's loop on the oracle envs against the errors the suite rebuilds from a trace."""
import ctypes
import os
import sys
import types

import numpy as np
import pytest
import torch

from serl_b200 import evaluation, rollout
from serl_b200.core.utils import calc_nMAE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ATT = rollout.actor_shape(72, 3, 'tanh')
INC = rollout.actor_shape(72, 3, 'tanh', state_dim=10)
SYM = rollout.actor_shape(72, 3, 'tanh', state_dim=2, action_dim=1)


@pytest.mark.parametrize('mean_deg', [0.3, -0.7, 2.5, -6.0])
def test_symmetric_nmae_from_track_is_calc_nmae_of_the_one_column_errors(mean_deg):
    rng = np.random.default_rng(int(abs(mean_deg) * 10))
    for n in (1, 7, 8001):
        e = np.deg2rad(mean_deg) + np.deg2rad(0.5) * rng.standard_normal((n, 1))
        track = np.array([np.abs(e[:, 0]).sum(), 0.0, 0.0, e[:, 0].sum()])
        got = evaluation.nmae_from_track(track, n, symmetric=True)
        want = calc_nMAE(e)
        assert abs(got - want) <= 1e-12 * abs(want), (n, got, want)
    # batched: [..., 4] sums with [...] steps
    tracks = np.stack([track, track * 2])
    assert np.allclose(evaluation.nmae_from_track(tracks, np.array([n, 2 * n]), symmetric=True), want, rtol=1e-12)


def test_conditions_must_match_the_actors_control_mode():
    # bare names are attitude control with absolute commands
    for c in ('nominal', 'be', 'gust', 'PHlab_attitude_cg-shift'):
        assert not evaluation.condition_env(c).incremental
        for sh, mode in ((INC, 'incremental control'), (SYM, 'symmetric control')):
            with pytest.raises(ValueError, match=mode):
                evaluation.condition_env(c, shape=sh)
    # incremental: any mode containing 'incremental', nominal build
    for c in ('incremental', 'PHlab_attitude_incremental', 'gust-incremental'):
        env = evaluation.condition_env(c, shape=INC)
        assert env.incremental and not env.sensor_noise and env.mode == 'nominal' and env.t_max == 80
        for sh, mode in ((None, 'incremental control'), (ATT, 'incremental control'), (SYM, 'symmetric control')):
            with pytest.raises(ValueError, match=mode):
                evaluation.condition_env(c, shape=sh)
    # symmetric: every condition of the attitude list under the symmetric configuration
    for c in evaluation.CONDITIONS:
        env = evaluation.condition_env('PHlab_symmetric_' + c, shape=SYM)
        assert env.symmetric and env.t_max == 80
        for sh in (None, ATT, INC):
            with pytest.raises(ValueError, match='symmetric control'):
                evaluation.condition_env('PHlab_symmetric_' + c, shape=sh)
    # the suite's refusals of mismatched pairs come before any device work
    with pytest.raises(ValueError, match='incremental control'):
        evaluation.evaluate_population(np.zeros((1, 1)), INC, ['nominal'], [])
    with pytest.raises(ValueError, match='symmetric control'):
        evaluation.evaluate_population(np.zeros((1, 1)), SYM, ['nominal'], [])
    with pytest.raises(ValueError, match='symmetric control'):
        evaluation.evaluate_population(np.zeros((1, 1)), ATT, ['PHlab_symmetric_nominal'], [])
    with pytest.raises(ValueError, match='incremental control'):
        evaluation.evaluate_population(np.zeros((1, 1)), ATT, ['nominal', 'incremental'], [])


def test_operator_runner_takes_the_conditions_of_the_actors_mode():
    from serl_b200 import operators
    base = dict(hidden_size=72, num_layers=3, activation_actor='tanh')
    cpu = torch.device('cpu')
    inc = types.SimpleNamespace(state_dim=10, action_dim=3, **base)
    sym = types.SimpleNamespace(state_dim=2, action_dim=1, **base)
    r = operators.OperatorRunner(inc, 'incremental', device=cpu)
    assert r.shape_tuple == (10, 3, 72, 3) and r.horizon == 2001
    r = operators.OperatorRunner(sym, 'PHlab_symmetric_noise', device=cpu)
    assert r.shape_tuple == (2, 1, 72, 3) and r.env.sensor_noise
    for c in ('gust', 'test'):       # per-actor replay launches: no gust instantiation for symmetric parents
        with pytest.raises(ValueError, match='gust'):
            operators.OperatorRunner(sym, 'PHlab_symmetric_' + c, device=cpu)
    with pytest.raises(ValueError, match='incremental control'):
        operators.OperatorRunner(inc, device=cpu)
    with pytest.raises(ValueError, match='symmetric control'):
        operators.OperatorRunner(sym, 'nominal', device=cpu)
    with pytest.raises(ValueError, match='incremental control'):
        operators.OperatorRunner(types.SimpleNamespace(state_dim=7, **base), 'incremental', device=cpu)
    refs = operators.study_refs(2, symmetric=True, seed=3)
    assert len(refs) == 3 and all(th.smooth_width == 20 // 6.7 for th, _ in refs)


def test_symmetric_references_are_seeded_draws_of_the_symmetric_grammar():
    a, b = evaluation.symmetric_refs(3, seed=11), evaluation.symmetric_refs(3, seed=11)
    assert len(a) == 4
    for (th, ph), (th2, _) in zip(a, b):
        assert np.array_equal(th.levels, th2.levels) and np.array_equal(th.starts, th2.starts)
        assert th.smooth_width == 11.0 and th.levels[0] == 0.0 and not ph.levels.any()
        assert np.array_equal(th.starts, 16.0 * np.arange(6))         # block width t_max // 5, no timing jitter
    assert not np.array_equal(evaluation.symmetric_refs(3, seed=12)[0][0].levels, a[0][0].levels) or \
        not np.array_equal(evaluation.symmetric_refs(3, seed=12)[1][0].levels, a[1][0].levels)


def _lib():
    from serl_b200 import _native, build
    build.build()
    return _native, _native.lib()


def test_suite_flag_rules_are_checked_before_any_cuda_call():
    _native, L = _lib()
    I, S, U, G, P = (_native.ROLLOUT_INCREMENTAL, _native.ROLLOUT_SYMMETRIC, _native.ROLLOUT_SUITE, _native.ROLLOUT_GUST,
                     _native.ROLLOUT_PER_ACTOR_REFS)
    bad_widths = (ctypes.c_int32 * 2)(4, 128)          # refused by K1-TC's own checks, before any CUDA call

    def run(dims, flags, pop=4, tc=False, **kw):
        d = _native.RolloutDesc()
        fake = iter(range(0x10000, 0x100000, 0x1000))      # non-null, never read
        for f in ('d_weights', 'd_ref_levels', 'd_ref_starts', 'd_env_mode', 'd_returns', 'd_steps', 'd_status'):
            setattr(d, f, next(fake))
        d.pop, d.shape, d.n_envs, d.horizon, d.flags = pop, _native.ActorShape(dims[0], dims[1], 72, 3, 0), 8, 100, flags
        d.t_max, d.smooth_width = 80.0, 11.0
        if tc:
            d.widths, d.n_widths = ctypes.cast(bad_widths, ctypes.c_void_p), 2
        for k, v in kw.items():
            setattr(d, k, v)
        return L.serl_rollout_run(ctypes.byref(d), None), L.serl_last_error().decode()

    trk, cost, noise = dict(d_track=0x9000), dict(d_track=0x9000, d_cost=0xa000), dict(d_sensor_noise=0xb000)
    refused = [((7, 3), U, {}), ((10, 3), U, {}), ((2, 1), U | I | S, {}), ((10, 3), U | I | S, {}),
               ((10, 3), I | U | G, trk), ((10, 3), I | U, noise), ((10, 3), I | U, dict(noise, **trk)),
               ((2, 1), S | U | G, {}), ((2, 1), S | U | G, noise),
               ((10, 3), I | U | P, trk), ((2, 1), S | U | P, trk), ((7, 3), P, trk)]
    for tc in (False, True):
        for dims, flags, kw in refused:
            rc, msg = run(dims, flags, tc=tc, **kw)
            assert rc == -1 and 'serl_rollout' in msg and 'pop must be' not in msg, (dims, flags, kw, msg)
    # without the suite flag every refusal of both modes holds, with its message
    for dims, flags, want in [((10, 3), I, 'incremental control (SERL_ROLLOUT_INCREMENTAL) does not take d_track / d_cost'),
                              ((2, 1), S, 'symmetric control (SERL_ROLLOUT_SYMMETRIC) does not take d_track / d_cost')]:
        rc, msg = run(dims, flags, **trk)
        assert rc == -1 and msg.endswith(want), msg
    # the allowed combinations pass the shared checks and fail only in the kernel's own (pop > 65535 on K1, w0 < 8 on K1-TC)
    allowed = [((10, 3), I | U, {}), ((10, 3), I | U, trk), ((10, 3), I | U, cost),
               ((2, 1), S | U, {}), ((2, 1), S | U, trk), ((2, 1), S | U, cost), ((2, 1), S | U | G, trk),
               ((2, 1), S | U | G, dict(noise, **cost)), ((2, 1), S | U, noise), ((2, 1), S | U | P, noise)]
    for dims, flags, kw in allowed:
        rc, msg = run(dims, flags, pop=70000, **kw)
        assert rc == -1 and 'pop must be <= 65535' in msg, (dims, flags, kw, msg)
        rc, msg = run(dims, flags, tc=True, **kw)
        assert rc == -3 and 'w0' in msg, (dims, flags, kw, msg)


def test_cli_takes_full_names_of_every_configuration():
    sys.path.insert(0, os.path.join(ROOT, 'examples'))
    try:
        import evaluate as cli
        import evaluate_operators as ops_cli
    finally:
        sys.path.pop(0)
    for c in (cli, ops_cli):
        assert c.conditions('PHlab_symmetric_all') == ['PHlab_symmetric_' + m for m in evaluation.CONDITIONS]
        assert c.conditions('PHlab_attitude_all') == list(evaluation.CONDITIONS) == c.conditions('all')
        assert c.conditions('PHlab_attitude_incremental') == ['incremental']
        assert c.conditions('PHlab_attitude_be') == ['be']
        assert c.conditions('PHlab_symmetric_be,PHlab_symmetric_gust') == ['PHlab_symmetric_be', 'PHlab_symmetric_gust']
        for mixed in ('PHlab_symmetric_be,nominal', 'all,PHlab_symmetric_nominal', 'PHlab_attitude_be,PHlab_symmetric_be'):
            with pytest.raises(SystemExit):
                c.conditions(mixed)
    assert evaluation.env_dims('PHlab_symmetric_be') == (2, 1)
    assert evaluation.env_dims('PHlab_attitude_incremental') == (10, 3)
    assert evaluation.env_dims('be') == (7, 3)
    assert [evaluation.condition_folder(c) for c in ('be', 'incremental', 'PHlab_symmetric_cg-shift')] == ['be', 'incremental', 'cg-shift']


# ---- base/evaluate.py's loop (evaluate(), :62-113) on the oracle envs, against the suite's rebuild from a trace ----------
def _evaluate_loop(env, actor, levels, starts, ref_fn, symmetric):
    """base/evaluate.py's evaluate() on an oracle env, and the trace rows the rollout kernels write for the same episode"""
    obs = env.reset(levels, starts)
    x0 = np.array(env.x[:12], dtype=np.float64)
    done, x_lst, u_lst, errors, ref_lst, rewards, rows = False, [], [], [], [], [], []
    ctrl = [7] if symmetric else [7, 6, 5]
    while not done:
        x_lst.append(np.array(env.x[:12]))
        u_lst.append(np.atleast_1d(env.last_u).copy())
        x_ctrl = np.asarray(env.x)[ctrl]
        action = np.clip(actor.select_action(obs), -1, 1)
        ref_value = np.deg2rad(ref_fn(env))
        obs, reward, done, _ = env.step(action.flatten())
        errors.append(ref_value - x_ctrl)
        ref_lst.append(ref_value)
        rewards.append(reward)
        row = np.full(rollout.TRACE_COLS, np.nan)
        row[rollout.TRACE_X] = np.asarray(env.x)[:12]
        row[rollout.TRACE_U] = np.pad(np.atleast_1d(env.last_u), (0, 3 - len(ctrl)))
        row[rollout.TRACE_R] = reward
        row[rollout.TRACE_ERR] = np.pad(np.atleast_1d(env.error)[:len(ctrl)], (0, 3 - len(ctrl)))
        rows.append(row)
    data = np.concatenate((np.array(ref_lst), np.asarray(u_lst), np.asarray(x_lst), np.asarray(rewards).reshape(-1, 1)), axis=1)
    return np.asarray(errors), np.asarray(u_lst), data, np.asarray(rows), x0


@pytest.mark.parametrize('mode', ['incremental', 'symmetric'])
def test_the_reference_loop_gives_the_errors_the_suite_rebuilds_from_a_trace(mode):
    from oracle import refsig as orefsig
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    try:
        if mode == 'incremental':
            import incremental_oracle as O
            env = O.IncrementalCitationEnv(t_max=80)
            refs = evaluation.eval_refs(1)[-1]
            env.smooth_w = float(refs[0].smooth_width)          # the user references' smooth width, t_max // 10
            levels, starts = np.stack([refs[0].levels, refs[1].levels]), np.stack([refs[0].starts, refs[1].starts])
            S, A = 10, 3
            ref_fn = lambda e: e.ref_deg()
        else:
            import symmetric_oracle as O
            env = O.SymmetricCitationEnv('nominal', t_max=80)
            th, ph = evaluation.symmetric_refs(0, seed=5)[0]
            levels, starts = np.stack([th.levels, ph.levels]), np.stack([th.starts, ph.starts])
            S, A = 2, 1
            ref_fn = lambda e: np.array([orefsig.ref_value_deg(e.levels[0], e.starts[0], e.t, O.THETA_TRIM, e.smooth_w, e.t_max)])
    finally:
        sys.path.pop(0)
    sh = rollout.actor_shape(32, 1, 'tanh', state_dim=S, action_dim=A)
    P = S * 32 + 32 + (32 * 32 + 3 * 32) + 32 * A + A
    genome = (np.random.default_rng(3).standard_normal(P) * 0.2).astype(np.float32)
    actor = O.KernelOrderActor(genome, 32, 1, 'tanh')
    errors, u_lst, data, rows, x0 = _evaluate_loop(env, actor, levels, starts, ref_fn, mode == 'symmetric')
    assert len(errors) > 100
    e2, u2, d2 = evaluation.rebuild_trial(rows, x0, mode == 'symmetric')
    assert d2.shape[1] == (15 if mode == 'symmetric' else 19) == data.shape[1]
    assert np.abs(e2 - errors).max() <= 1e-12
    assert np.array_equal(u2, u_lst) and np.abs(d2 - data).max() <= 1e-12
    assert abs(calc_nMAE(e2) - calc_nMAE(errors)) <= 1e-9 * calc_nMAE(errors)
    # the kernels' sums of the same errors give the same nMAE
    c = errors[:, 0]
    track = np.array([np.abs(c).sum(), 0, 0, c.sum()]) if mode == 'symmetric' else \
        np.array([np.abs(errors[:, 0]).sum(), np.abs(errors[:, 1]).sum(), np.abs(errors[:, 2]).sum(), errors[:, 2].sum()])
    assert abs(evaluation.nmae_from_track(track, len(errors), symmetric=mode == 'symmetric') - calc_nMAE(errors)) <= 1e-12 * calc_nMAE(errors)
    assert sh.state_dim == S
