"""The evaluation suite and the operator study of incremental and symmetric control on the device: the tracking launches'
sums against the errors validate_agent rebuilds from its trace, the tracking instantiations' dynamics against the training
ones, validate_agent against base/evaluate.py's loop on the oracle envs, evaluate_population against validate_agent, and the
mutation-operator study of both modes."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from serl_b200 import evaluation, operators, rollout
from serl_b200.core.genetic_agent import Actor
from serl_b200.core.utils import calc_nMAE, calc_smoothness

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
DEV = torch.device('cuda:0')
SYM_CONDS = ['PHlab_symmetric_' + c for c in evaluation.CONDITIONS]
DIMS = {'incremental': (10, 3), 'symmetric': (2, 1)}


class Args:
    def __init__(self, S, A, hidden, layers, act):
        self.state_dim, self.action_dim = S, A
        self.hidden_size, self.num_layers, self.activation_actor = hidden, layers, act


def genomes(mode, n, hidden, layers, act='tanh', seed=0):
    S, A = DIMS[mode]
    torch.manual_seed(seed)
    g = np.stack([Actor(Args(S, A, hidden, layers, act)).flat().detach().numpy() for _ in range(n)]).astype(np.float32)
    if mode == 'incremental':         # small rates: the integrated deflections stay flyable for much of the 80 s
        g[:, -(A * hidden + A):] *= 0.02
    return g


def wide_genomes(mode, widths, n, seed=1):
    S, A = DIMS[mode]
    P = rollout.num_params_wide(widths, S, A)
    return (np.random.default_rng(seed).standard_normal((n, P)) * 0.05).astype(np.float32)


# K1 warp (h = 72), the one-thread-per-env kernel (h = 48), K1-TC ([256] * 4 routed from the uniform actor, and [400, 300])
CASES = {
    'k1_h72': lambda m: (genomes(m, 2, 72, 3), rollout.actor_shape(72, 3, 'tanh', *DIMS[m]), None),
    'simple_h48': lambda m: (genomes(m, 2, 48, 1, 'elu'), rollout.actor_shape(48, 1, 'elu', *DIMS[m]), None),
    'tc_256x4': lambda m: (genomes(m, 2, 256, 3, 'relu'), rollout.actor_shape(256, 3, 'relu', *DIMS[m]), None),
    'tc_400_300': lambda m: (wide_genomes(m, [400, 300], 2), rollout.actor_shape(8, 1, 'tanh', *DIMS[m]), [400, 300]),
}


def refs_for(mode, num_trails, t_max=evaluation.T_MAX):
    np.random.seed(7)
    refs = evaluation.eval_refs(num_trails, t_max)
    return evaluation.symmetric_refs(num_trails, 7, t_max) if mode == 'symmetric' else refs


def host_sums(errors, symmetric):
    e = np.asarray(errors)
    if symmetric:
        return np.array([np.abs(e[:, 0]).sum(), 0.0, 0.0, e[:, 0].sum()])
    return np.array([np.abs(e[:, 0]).sum(), np.abs(e[:, 1]).sum(), np.abs(e[:, 2]).sum(), e[:, 2].sum()])


@pytest.mark.parametrize('case', list(CASES))
@pytest.mark.parametrize('mode', ['incremental', 'symmetric'])
def test_track_sums_equal_host_sums_of_validate_agents_errors(mode, case):
    g, shape, widths = CASES[case](mode)
    sym = mode == 'symmetric'
    conds = ['incremental'] if not sym else SYM_CONDS if case == 'k1_h72' else \
        ['PHlab_symmetric_' + c for c in ('nominal', 'gust', 'test', 'noise', 'cg-shift', 'be')]
    refs = refs_for(mode, 1)
    for c in conds:
        env = evaluation.condition_env(c, shape=shape)
        np.random.seed(3)
        f = evaluation.fly_traced(g[1], shape, env, refs, 1, widths=widths)
        assert f.track.shape == (2, 4) and f.data.shape[1] == (15 if sym else 19)
        for i, e in enumerate(f.errors):
            assert len(e) == f.steps[i] and e.shape[1] == (1 if sym else 3)
            want = host_sums(e, sym)
            got = f.track[i]
            assert np.all(np.abs(got - want) <= 1e-12 * np.abs(want) + 1e-300), (c, i, got, want)
            if sym:
                assert got[1] == 0.0 and got[2] == 0.0
            assert evaluation.nmae_from_track(got, f.steps[i], symmetric=sym) == pytest.approx(calc_nMAE(e), rel=1e-12)


@pytest.mark.parametrize('mode', ['incremental', 'symmetric'])
def test_time_split_hand_over_carries_the_tracking_sums(mode):
    """K1's time-split schedule (more tasks than slots, sm_limit) hands every trajectory's sums, observation and (incremental
    control) last_u to the next slot: the tiled launch equals the small one bit for bit"""
    g, shape, _ = CASES['k1_h72'](mode)
    sym = mode == 'symmetric'
    conds = ['incremental'] * 2 if not sym else ['PHlab_symmetric_' + c for c in ('nominal', 'gust', 'noise', 'be')]
    codes = np.array([evaluation.condition_env(c, shape=shape).mode_code for c in conds], dtype=np.int32)
    lv, st = evaluation._ref_arrays(refs_for(mode, 0, 20) * len(conds))
    sw = 20 // 6.7 if sym else 2.0
    gust = any(rollout.mode_gust(int(c)) for c in codes)
    z = np.random.default_rng(5).standard_normal((1, len(conds), 2002, 7)).astype(np.float32) if sym else None

    def launch(w, **kw):
        zz = None if z is None else torch.as_tensor(np.ascontiguousarray(np.repeat(z, w.shape[0], 0)), device=DEV)
        r = rollout.population_rollout(torch.as_tensor(w, device=DEV), shape, torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV),
                                       torch.as_tensor(codes, device=DEV), horizon=2001, t_max=20.0, smooth_width=sw, fitness=False,
                                       track=True, cost=True, suite=True, gust=gust, sensor_noise=zz, **kw)
        r.check()
        return r
    small = launch(g)
    big = launch(np.tile(g, (30, 1)), sm_limit=2)
    assert torch.equal(big.track, small.track.repeat(30, 1, 1)) and torch.equal(big.cost, small.cost.repeat(30, 1))
    assert torch.equal(big.steps, small.steps.repeat(30, 1)) and torch.equal(big.returns, small.returns.repeat(30, 1))


@pytest.mark.parametrize('case', ['k1_h72', 'simple_h48', 'tc_256x4'])
@pytest.mark.parametrize('mode', ['incremental', 'symmetric'])
def test_tracking_instantiations_fly_the_training_dynamics(mode, case):
    g, shape, widths = CASES[case](mode)
    cond = 'incremental' if mode == 'incremental' else 'PHlab_symmetric_nominal'
    refs = refs_for(mode, 2)
    lv, st = evaluation._ref_arrays(refs)
    md = torch.full((len(refs),), evaluation.condition_env(cond, shape=shape).mode_code, dtype=torch.int32, device=DEV)
    kw = dict(horizon=8001, t_max=80.0, smooth_width=float(refs[0][0].smooth_width), widths=widths, actions=True)
    args = (torch.as_tensor(g, device=DEV), shape, torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV), md)
    train = rollout.population_rollout(*args, **kw)
    track = rollout.population_rollout(*args, track=True, cost=True, suite=True, **kw)
    train.check(); track.check()
    assert torch.equal(train.returns, track.returns) and torch.equal(train.steps, track.steps)
    live = torch.arange(8001, device=DEV)[None, None, :] < train.steps[..., None]      # the record of executed steps
    assert torch.equal(train.actions[live], track.actions[live])


def _oracle(mode):
    sys.path.insert(0, HERE)
    try:
        import test_eval_modes as T
        if mode == 'incremental':
            import incremental_oracle as O
        else:
            import symmetric_oracle as O
    finally:
        sys.path.pop(0)
    return T, O


@pytest.mark.parametrize('cond', ['incremental', 'PHlab_symmetric_nominal', 'PHlab_symmetric_be', 'PHlab_symmetric_noise'])
def test_validate_agent_matches_the_reference_loop_on_the_oracle_env(cond):
    mode = 'incremental' if cond == 'incremental' else 'symmetric'
    sym = mode == 'symmetric'
    T, O = _oracle(mode)
    from oracle import refsig as orefsig
    g, shape, _ = CASES['k1_h72'](mode)
    refs = refs_for(mode, 1)
    env = evaluation.condition_env(cond, shape=shape)
    horizon = 8001
    np.random.seed(11)
    state = np.random.get_state()
    _, stats = evaluation.validate_agent(g[0], shape, env, refs, 1)
    np.random.set_state(state)
    z = evaluation.sensor_noise_draws(len(refs), horizon) if env.sensor_noise else None
    mode_name = cond.split('_')[-1]
    oenv = O.IncrementalCitationEnv(t_max=80) if not sym else O.SymmetricCitationEnv(mode_name if mode_name != 'noise' else 'nominal', t_max=80)
    actor = O.KernelOrderActor(g[0], 72, 3, 'tanh')
    nm, sm = [], []
    for i, (th, ph) in enumerate(refs):
        if z is not None:
            oenv.noise_z = z[i]
        if sym:
            ref_fn = lambda e: np.array([orefsig.ref_value_deg(e.levels[0], e.starts[0], e.t, O.THETA_TRIM, e.smooth_w, e.t_max)])
        else:
            oenv.smooth_w = float(th.smooth_width)
            ref_fn = lambda e: e.ref_deg()
        errors, u_lst, _, _, _ = T._evaluate_loop(oenv, actor, np.stack([th.levels, ph.levels]), np.stack([th.starts, ph.starts]), ref_fn, sym)
        nm.append(calc_nMAE(errors))
        sm.append(calc_smoothness(u_lst))
    assert stats.nmae == pytest.approx(np.average(nm), rel=1e-5) and stats.sm == pytest.approx(np.average(sm), rel=1e-5)


@pytest.mark.parametrize('mode', ['incremental', 'symmetric'])
def test_evaluate_population_equals_validate_agent(mode):
    g, shape, widths = CASES['k1_h72'](mode)
    conds = ['incremental'] if mode == 'incremental' else \
        ['PHlab_symmetric_' + c for c in ('nominal', 'noise', 'gust', 'be', 'cg-shift')]
    refs = refs_for(mode, 1)
    np.random.seed(4)
    state = np.random.get_state()
    want = {}
    for c in conds:
        env = evaluation.condition_env(c, shape=shape)
        for a in range(len(g)):
            want[a, c] = evaluation.validate_agent(g[a], shape, env, refs, 1)[1]
    np.random.set_state(state)
    res = evaluation.evaluate_population(g, shape, conds, refs, 1)
    for (a, c), s in want.items():
        got = res.stats(a, c)
        assert got.nmae == pytest.approx(s.nmae, rel=1e-12) and got.nmae_sd == pytest.approx(s.nmae_sd, rel=1e-9, abs=1e-12), (a, c)
        assert abs(got.sm - s.sm) <= 2e-5 * abs(s.sm) + 1e-9, (a, c, got.sm, s.sm)


@pytest.mark.parametrize('cond', ['incremental', 'PHlab_symmetric_nominal', 'PHlab_symmetric_noise'])
def test_operator_study_runs_for_both_modes(cond):
    mode = 'incremental' if cond == 'incremental' else 'symmetric'
    S, A = DIMS[mode]
    g = genomes(mode, 3, 32, 1, seed=2)
    args = types.SimpleNamespace(state_dim=S, action_dim=A, hidden_size=32, num_layers=1, activation_actor='tanh', individual_bs=4000,
                                 mutation_batch_size=64, mutation_mag=0.05, seed=7)
    np.random.seed(7)
    refs = operators.study_refs(1, symmetric=mode == 'symmetric', seed=7)
    runner = operators.OperatorRunner(args, cond, num_trails=1, device=DEV)
    study = runner.test_mutation(g, refs)
    stats_reward, stats_cost = study
    for op in operators.OPERATORS:
        assert stats_reward[op].shape == (3 * 2,) and np.isfinite(study.child_nmae[op]).all()
    # the parents' per-actor replay launch against a tracking launch of the same genomes, references and draws
    z = None
    if runner.env.sensor_noise:
        np.random.seed(9)
        z = np.stack([evaluation.sensor_noise_draws(2, runner.horizon) for _ in range(3)])
    parent = runner.validate_parents(torch.as_tensor(g, device=DEV), refs, z)
    ret, cost, _ = runner.fly_children(torch.as_tensor(g, device=DEV), refs, z)
    assert np.array_equal(parent.returns, ret) and np.array_equal(parent.costs, cost)
    assert parent.buffers.data.shape[-1] == rollout.transition_cols(S, A)
    # the children's nMAE against each child flown alone by validate_agent (noiseless conditions: the same references)
    if not runner.env.sensor_noise:
        shape = rollout.actor_shape(32, 1, 'tanh', S, A)
        env = evaluation.condition_env(cond, operators.T_MAX, shape=shape)
        for o, op in enumerate(operators.OPERATORS):
            for i in range(3):
                s = evaluation.validate_agent(study.child_genomes[o, 0, i], shape, env, refs, 1)[1]
                assert np.average(study.child_nmae[op][0, i]) == pytest.approx(s.nmae, rel=1e-12), (op, i)
    if mode == 'symmetric':
        with pytest.raises(ValueError, match='gust'):
            operators.OperatorRunner(args, 'PHlab_symmetric_gust', device=DEV)
