"""The mutation-operator study without a GPU: the C-ABI's cost-tally field and its refusal, the statistics of
OperatorRunner.test_mutation, the study's references and the mutation_stats.toml layout."""
import ctypes
import os
import random
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_names_the_cost_tally_last_and_the_binding_mirrors_it():
    from serl_b200 import _native
    text = open(os.path.join(ROOT, 'include', 'serl_b200.h')).read()
    body = re.search(r'typedef struct \{(.*?)\} serl_rollout_desc;', text, re.S).group(1)
    assert re.search(r'double\* d_track;\s*int32_t\* d_cost;\s*$', body.strip() + '\n', re.M)      # appended: no field moved
    assert _native.RolloutDesc._fields_[-1] == ('d_cost', ctypes.c_void_p)
    assert [f for f, _ in _native.RolloutDesc._fields_][-2] == 'd_track'


@pytest.mark.parametrize('widths', [None, [128, 128]])
def test_cost_without_track_is_refused_before_any_cuda_call(widths):
    """K1 and K1-TC: SERL_ERR_ARG, no kernel launched, the (fake, non-null) device pointers never read"""
    from serl_b200 import build, _native, rollout
    build.build()
    L = _native.lib()
    warr = (ctypes.c_int32 * 2)(*(widths or [0, 0]))
    d = _native.RolloutDesc()
    fake = iter(range(0x10000, 0x100000, 0x1000))
    for f in ('d_weights', 'd_ref_levels', 'd_ref_starts', 'd_env_mode', 'd_returns', 'd_steps', 'd_status', 'd_cost'):
        setattr(d, f, next(fake))
    d.pop, d.shape, d.n_envs, d.horizon = 4, rollout.actor_shape(72), 8, 100
    if widths:
        d.widths, d.n_widths = ctypes.cast(warr, ctypes.c_void_p), 2
    launches = L.serl_launch_count()
    rc = L.serl_rollout_run(ctypes.byref(d), None)
    assert rc == -1, (rc, L.serl_last_error())
    assert 'd_cost' in L.serl_last_error().decode()
    assert L.serl_launch_count() == launches


def _test_mutation_restated(pr_t, pc_t, child_r, child_c):
    """operator_runner.py:127-206 line by line on per-trial scores / costs (validate_agent's averages broadcast)"""
    N, T = pr_t.shape
    pr, pc = np.zeros((N, T)), np.zeros((N, T))
    out_r = {k: np.zeros((N, T)) for k in ('Normal', 'Proximal', 'Safe')}
    out_c = {k: np.zeros((N, T)) for k in out_r}
    with np.errstate(divide='ignore', invalid='ignore'):
        for i in range(N):
            pr[i, :] = np.average(pr_t[i])
            pc[i, :] = np.average(pc_t[i])
            for k in out_r:
                r = np.zeros(T); c = np.zeros(T)
                r[:] = np.average(child_r[k][i]); c[:] = np.average(child_c[k][i])
                out_r[k][i, :] = 1 - r / pr[i, :]
                out_c[k][i, :] = c / pc[i, :] - 1
    return {k: v.flatten() for k, v in out_r.items()}, {k: v.flatten() for k, v in out_c.items()}


def test_statistics_match_the_reference_arithmetic_including_a_zero_cost_parent():
    from serl_b200 import operators
    rng = np.random.default_rng(3)
    N, T = 5, 4
    pr = -rng.uniform(100, 2000, (N, T))
    pc = rng.integers(0, 50, (N, T)).astype(np.int64)
    pc[1] = 0                                                  # zero-cost parent: x / 0 -> inf, 0 / 0 -> nan
    child_r = {k: -rng.uniform(100, 2000, (N, T)) for k in operators.OPERATORS}
    child_c = {k: rng.integers(0, 50, (N, T)) for k in operators.OPERATORS}
    child_c['Safe'][1] = 0
    want_r, want_c = _test_mutation_restated(pr, pc, child_r, child_c)
    got_r, got_c = operators.mutation_stats(pr, pc, child_r, child_c)
    assert list(got_r) == list(got_c) == ['Normal', 'Proximal', 'Safe']
    for k in operators.OPERATORS:
        assert got_r[k].shape == (N * T,)
        np.testing.assert_array_equal(got_r[k], want_r[k])
        np.testing.assert_array_equal(got_c[k], want_c[k])
        assert np.all(got_r[k].reshape(N, T) == got_r[k].reshape(N, T)[:, :1])      # broadcast over the trial columns
    assert np.isnan(got_c['Safe'].reshape(N, T)[1]).all()
    assert np.isinf(got_c['Normal'].reshape(N, T)[1]).all() or np.isnan(got_c['Normal'].reshape(N, T)[1]).all()


def test_study_wraps_magnitudes_and_unpacks_like_the_reference():
    from serl_b200 import operators
    rng = np.random.default_rng(4)
    N, T, M = 3, 2, 2
    parent = operators.ParentFlight(-rng.uniform(1, 9, (N, T)), rng.integers(1, 9, (N, T)), None, None, None)
    cr = {k: -rng.uniform(1, 9, (M, N, T)) for k in operators.OPERATORS}
    cc = {k: rng.integers(0, 9, (M, N, T)) for k in operators.OPERATORS}
    study = operators.MutationStudy([0.1, 0.2], parent, cr, cc, cr, None)
    sr, sc = study
    for m, mag in enumerate([0.1, 0.2]):
        r1, c1 = operators.mutation_stats(parent.returns, parent.costs, {k: v[m] for k, v in cr.items()}, {k: v[m] for k, v in cc.items()})
        for k in operators.OPERATORS:
            np.testing.assert_array_equal(study.by_mag[mag][0][k], r1[k])
            np.testing.assert_array_equal(sr[k][m * N * T:(m + 1) * N * T], r1[k])
            np.testing.assert_array_equal(sc[k][m * N * T:(m + 1) * N * T], c1[k])


@pytest.mark.parametrize('num_trails', [0, 3])
def test_study_references_are_the_reference_scripts(num_trails):
    """base/evaluate_operators.py:85-104 at t_max = 20, restated on the same seeded stream"""
    from serl_b200 import operators, signals
    t_max = 20
    np.random.seed(7)
    time_array = np.linspace(0., t_max, 6)
    base_theta = signals.SmoothedStepSequence(time_array, [0, 12, 3, -4, -8, 2], smooth_width=t_max // 10)
    base_phi = signals.SmoothedStepSequence(time_array, [2, -2, 2, 10, 2, -6], smooth_width=t_max // 10)

    def gen_refs(ampl_max):
        # base/evaluation_utils.py gen_refs
        grid = np.linspace(-ampl_max, ampl_max, 6)
        times = list(time_array)
        out = []
        for _ in range(num_trails):
            levels = np.random.choice(grid, size=6, replace=True)
            levels[0] = 0.0
            times = times[:1] + [t + np.random.uniform(-0.05, 0.05) for t in times[1:]]
            out.append(signals.SmoothedStepSequence(times, levels, smooth_width=t_max // 10))
        return out
    theta, phi = gen_refs(12.0), gen_refs(10.0)
    want = list(zip(theta + [base_theta], phi + [base_phi]))
    np.random.seed(7)
    got = operators.study_refs(num_trails)
    assert len(got) == num_trails + 1
    for (gt, gp), (wt, wp) in zip(got, want):
        for g, w in ((gt, wt), (gp, wp)):
            np.testing.assert_array_equal(g.levels, w.levels)
            np.testing.assert_array_equal(g.starts, w.starts)
            assert g.smooth_width == w.smooth_width == 2


def test_toml_layout_is_the_reference_scripts():
    """stats_cost first, a blank line, then stats_reward; keys Normal, Proximal, Safe; arrays as toml.TomlNumpyEncoder
    writes them"""
    from serl_b200 import operators
    sr = {'Normal': np.array([0.5, -0.25]), 'Proximal': np.array([1e-7, 2.0]), 'Safe': np.array([0.0, 3.0])}
    sc = {'Normal': np.array([np.inf, np.nan]), 'Proximal': np.array([-1.0, 0.125]), 'Safe': np.array([1e20, -0.5])}
    text = operators.mutation_stats_toml(sr, sc)
    assert text == ('[stats_cost]\n'
                    'Normal = [ inf, nan,]\n'
                    'Proximal = [ -1.0, 0.125,]\n'
                    'Safe = [ 1e+20, -0.5,]\n'
                    '\n'
                    '[stats_reward]\n'
                    'Normal = [ 0.5, -0.25,]\n'
                    'Proximal = [ 1e-7, 2.0,]\n'
                    'Safe = [ 0.0, 3.0,]\n')


def test_normal_mutation_planner_consumes_the_streams_like_plan_epoch():
    """evo.plan_mutate_inplace is plan_epoch's mutation body: fed the same ssne_probabilities it makes the same ops and
    leaves the stdlib stream where oracle.ssne's mutate_inplace leaves it"""
    from serl_b200 import evo
    from oracle import ssne
    table, P = evo.param_table(7, 3, 16, 2)
    random.seed(5); np.random.seed(5)
    lists = ([], [], [], [])
    for i in range(3):
        evo.plan_mutate_inplace(table, i, np.random.uniform(0, 1, len(table)) * 2, *lists)
    after = random.getstate(), np.random.get_state()[2]
    random.seed(5); np.random.seed(5)
    o = ssne.SSNE(3, (7, 3, 16, 2))
    W = np.random.RandomState(0).randn(3, P).astype(np.float32)
    random.seed(5); np.random.seed(5)
    for i in range(3):
        o.mutate_inplace(W, i, 0.1)
    assert random.getstate() == after[0] and np.random.get_state()[2] == after[1]
    seg, off, kind, z = evo.mutation_arrays(*lists)
    assert seg.shape[1] == 3 and off.shape == kind.shape == z.shape and z.dtype == np.float32
