"""K6 (csrc/smoothness.cu) against calc_smoothness (base/core/utils.py:82-120) in float64 on the exact float32 input the
kernel reads, across every horizon it accepts: the Bluestein FFT path (horizon <= 2048) and the direct DFT (2049 ..
10240), lengths with no bin, one bin and many, the precomputed full-length chirp and the per-trajectory one, three dt,
DC-dominated and near-Nyquist signals, and real K1 / K1-TC action histories.  Then the bits of a trajectory in any batch
and on any stream, and the two consumers that turn K6 into a fitness and an evaluation statistic."""
import os
import random

import numpy as np
import pytest
import torch

from oracle import actor as OA, refsig
from serl_b200 import evaluation, rollout
from serl_b200.core.utils import calc_smoothness
from test_k6_domain import DIRECT_MAX_HORIZON, FFT_MAX_HORIZON

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ACT = np.load(os.path.join(HERE, 'golden', 'actors.npz'))
DEV = torch.device('cuda:0')
REL, ABS = 2e-5, 1e-9                    # |K6 - ref| <= REL |ref| + ABS
DTS = [0.01, 0.02, 0.005]
FFT_HORIZONS = [5, 64, 1000, 2001, 2047, FFT_MAX_HORIZON]
DIRECT_HORIZONS = [FFT_MAX_HORIZON + 1, 8001, DIRECT_MAX_HORIZON]
# signals whose metric is 0 up to the float64 reference's rounding: the absolute term of the bar must hold alone
ZERO_KINDS = ('constant', 'saturated', 'zeros')
KINDS = ('mix', 'trim_ripple_1e-3', 'trim_ripple_1e-4', 'alternating', 'impulse', 'scales') + ZERO_KINDS
WORST = {'fft': {'rel': 0.0, 'abs_at_zero': 0.0}, 'direct': {'rel': 0.0, 'abs_at_zero': 0.0}}


@pytest.fixture(scope='module', autouse=True)
def report_margins():
    yield
    for path, w in WORST.items():
        print('\nK6 %-6s path: worst relative error %.3e (bar %.0e), worst |error| on zero-metric signals %.3e (bar %.0e)'
              % (path, w['rel'], REL, w['abs_at_zero'], ABS))


def signal(kind, n, rng):
    """[n, 3] float64 action history of `kind` (seeded by rng)"""
    k = np.arange(n)[:, None]
    slow = lambda amp: amp * np.sin(2 * np.pi * rng.uniform(0.05, 0.5, 3) * 0.01 * k + rng.uniform(0, 2 * np.pi, 3))
    if kind == 'mix':
        return 0.05 + slow(0.1) + 0.01 * rng.randn(n, 3)
    if kind == 'constant':
        return np.broadcast_to([-0.12, 0.03, 0.01], (n, 3))
    if kind == 'saturated':
        return np.broadcast_to([1.0, -1.0, 1.0], (n, 3))
    if kind.startswith('trim_ripple_'):       # a trimmed elevator under a small ripple: what a smooth actor flies
        return rng.uniform(0.1, 1.0, 3) * rng.choice([-1.0, 1.0], 3) + slow(float(kind.split('_')[-1]))
    if kind == 'alternating':
        # +-a under a slow envelope: the content sits next to the Nyquist bin, not on it (a pure +-a of even length is
        # all Nyquist bin, which the metric excludes)
        env = 1.0 + 0.5 * np.sin(2 * np.pi * k / 50.0 + rng.uniform(0, 2 * np.pi, 3))
        return rng.uniform(0.05, 0.3, 3) * np.where(k % 2 == 0, 1.0, -1.0) * env
    if kind == 'impulse':
        y = np.zeros((n, 3))
        if n:
            y[rng.randint(0, n, 3), np.arange(3)] = rng.uniform(0.1, 1.0, 3)
        return y
    if kind == 'zeros':
        return np.zeros((n, 3))
    if kind == 'scales':                      # channels 1 : 1e-4 : 1e-2
        return (0.05 + slow(0.1) + 0.01 * rng.randn(n, 3)) * np.array([1.0, 1e-4, 1e-2])
    raise ValueError(kind)


def batch(horizon, lengths, kinds, rng):
    """[len(lengths), horizon, 3] fp32 with trajectory i = signal(kinds[i]) over its first lengths[i] steps and NaN after
    them: a step past N that reached the metric would poison it"""
    a = np.full((len(lengths), horizon, 3), np.nan, dtype=np.float32)
    for i, (n, kind) in enumerate(zip(lengths, kinds)):
        a[i, :n] = signal(kind, n, rng)
    return a, np.asarray(lengths, dtype=np.int32)


def k6(a, steps, dt=0.01):
    return rollout.smoothness(torch.as_tensor(a, device=DEV), torch.as_tensor(steps, device=DEV), dt).cpu().numpy()


def path_of(horizon):
    return 'fft' if horizon <= FFT_MAX_HORIZON else 'direct'


def check(got, a, steps, dt, horizon, kinds=None):
    w = WORST[path_of(horizon)]
    for i, n in enumerate(steps):
        ref = calc_smoothness(a[i, :n].astype(np.float64), dt=dt)
        what = (horizon, dt, int(n), kinds[i] if kinds else i, got[i], ref)
        if n // 2 - 1 <= 0:
            assert got[i] == 0.0 and np.signbit(got[i]), what          # -0.0, as the reference
            continue
        assert np.isfinite(got[i]), what
        err = abs(got[i] - ref)
        assert err <= REL * abs(ref) + ABS, what
        if kinds and kinds[i] in ZERO_KINDS:
            w['abs_at_zero'] = max(w['abs_at_zero'], err)
        else:
            assert ref < 0, what
            w['rel'] = max(w['rel'], err / abs(ref))


def fft_lengths(h):
    ns = {0, 1, 2, 3, 4, 5, (2 * h) // 3 | 1, (h // 2) & ~1, h - 1, h}      # none, one bin, odd, even, the two longest
    if h == FFT_MAX_HORIZON:
        ns |= {1024, 1025, 2047, 2048}
    return sorted(n for n in ns if n <= h)


def direct_lengths(h):
    return sorted(n for n in {0, 1, 2, 3, 4, 5, 1001, 2047, 2048, 2049, 2050, (h + 2049) // 2 | 1, h - 1, h} if n <= h)


CASES = [(h, dt) for h in FFT_HORIZONS + DIRECT_HORIZONS for dt in DTS]


@pytest.mark.parametrize('horizon,dt', CASES, ids=['h%d-dt%g' % c for c in CASES])
def test_k6_matches_the_float64_formula(horizon, dt):
    """every length class x every signal, all in one launch per (horizon, dt)"""
    lens = fft_lengths(horizon) if horizon <= FFT_MAX_HORIZON else direct_lengths(horizon)
    lengths = [n for n in lens for _ in KINDS]
    kinds = [kind for _ in lens for kind in KINDS]
    a, steps = batch(horizon, lengths, kinds, np.random.RandomState(horizon * 3 + DTS.index(dt)))
    check(k6(a, steps, dt), a, steps, dt, horizon, kinds)


def test_the_direct_path_holds_dc_dominated_histories():
    """the cases a direct DFT without mean removal gets wrong: a constant deflection (the float64 metric is ~0) and a trim
    with a 1e-4 ripple, 8001 steps (the 80 s evaluation episode) and the longest accepted horizon"""
    for horizon in (8001, DIRECT_MAX_HORIZON):
        kinds = ['constant', 'saturated', 'trim_ripple_1e-4', 'trim_ripple_1e-3'] * 2
        a, steps = batch(horizon, [horizon] * 4 + [horizon - 1] * 4, kinds, np.random.RandomState(5))
        got = k6(a, steps)
        check(got, a, steps, 0.01, horizon, kinds)
        assert np.abs(got[[0, 1, 4, 5]]).max() <= ABS


def rollout_histories(horizon, t_max=None):
    """deflection records of K1 (h = 72: two trained actors, two untrained ones that crash) and K1-TC ([256] * 4, relu)
    on three flight conditions: [n, horizon, 3] fp32 and their executed steps"""
    torch.manual_seed(7)
    k1 = np.concatenate([ACT['serl10_pop_h72_tanh'][:2], np.stack([OA.flatten(OA.Actor(hidden=72)) for _ in range(2)])])
    tc = np.stack([OA.flatten(OA.Actor(hidden=256, activation='relu')) for _ in range(2)]).astype(np.float32)
    kw = {} if t_max is None else dict(t_max=t_max, smooth_width=refsig.widths(t_max)[1])
    lv, st = refsig.make_ref_params(3, seed_base=17, **({} if t_max is None else dict(t_max=int(t_max))))
    md = torch.tensor([rollout.mode_code(m) for m in ('nominal', 'be', 'ice')], dtype=torch.int32, device=DEV)
    acts, steps = [], []
    for w, shape in ((k1, rollout.actor_shape(72)), (tc, rollout.actor_shape(256, 3, 'relu'))):
        r = rollout.population_rollout(torch.as_tensor(w, device=DEV), shape, torch.as_tensor(lv, device=DEV),
                                       torch.as_tensor(st, device=DEV), md, horizon=horizon, actions=True, fitness=False, **kw)
        torch.cuda.synchronize()
        r.check()
        acts.append(r.actions.reshape(-1, horizon, 3).cpu().numpy())
        steps.append(r.steps.reshape(-1).cpu().numpy())
    return np.concatenate(acts), np.concatenate(steps).astype(np.int32)


@pytest.mark.parametrize('horizon,t_max', [(1000, None), (2001, None), (FFT_MAX_HORIZON + 1, 80.0), (8001, 80.0)])
def test_k6_matches_the_float64_formula_on_rollout_histories(horizon, t_max):
    """the records as flown, next to the same records cut short (an early termination as K6 sees one), in one launch"""
    a, steps = rollout_histories(horizon, t_max)
    print('\nhorizon %d: executed steps %s' % (horizon, sorted(steps.tolist())))
    assert (steps == horizon).any() and (steps < horizon).any()         # full-length and crashed flights side by side
    assert (steps > 5).all() and np.isfinite(np.concatenate([a[i, :n] for i, n in enumerate(steps)])).all()
    a = np.concatenate([a, a])
    steps = np.concatenate([steps, np.maximum(steps * 2 // 3, 4)]).astype(np.int32)
    for dt in DTS:
        check(k6(a, steps, dt), a, steps, dt, horizon)


def bits(x):
    return np.ascontiguousarray(x).view(np.int64)


@pytest.mark.parametrize('horizon', [2001, FFT_MAX_HORIZON, 8001])
def test_a_trajectory_gets_the_same_bits_in_any_batch(horizon):
    """position, batch order, n_traj and the lengths of the other trajectories of the launch change no bit; nor does a
    second launch"""
    rng = np.random.RandomState(horizon)
    lengths = [horizon, 7, horizon, 1000, 3, horizon - 1, 4, 1500, horizon]
    kinds = ['mix', 'trim_ripple_1e-4', 'alternating', 'mix', 'mix', 'impulse', 'scales', 'trim_ripple_1e-3', 'constant']
    a, steps = batch(horizon, lengths, kinds, rng)
    got = k6(a, steps)
    check(got, a, steps, 0.01, horizon, kinds)
    assert np.array_equal(bits(k6(a, steps)), bits(got))
    assert np.array_equal(bits(k6(a[::-1].copy(), steps[::-1].copy())), bits(got[::-1]))
    for i in range(len(lengths)):
        assert np.array_equal(bits(k6(a[i:i + 1], steps[i:i + 1])), bits(got[i:i + 1])), i
    assert np.array_equal(bits(k6(np.concatenate([a] * 3), np.concatenate([steps] * 3))), bits(np.concatenate([got] * 3)))
    # the other trajectories of the launch run other lengths (full-length ones included: the precomputed chirp)
    other = steps.copy()
    other[1::2] = [horizon, 2, horizon - 3, 901]
    a2 = a.copy()
    for i in range(1, len(lengths), 2):
        a2[i, :other[i]] = signal('mix', other[i], rng)
    assert np.array_equal(bits(k6(a2, other)[0::2]), bits(got[0::2]))


def test_launches_on_two_streams_give_the_same_bits():
    """each stream keeps its own K6 tables: launches of different horizons queued on two streams without a wait between
    them give what the same launches give one after the other"""
    rng = np.random.RandomState(2)
    jobs = []
    for horizon in (2001, 1000, 8001):
        lengths = [horizon, horizon // 2 | 1, horizon, 17, horizon - 1, 5]
        kinds = ['mix', 'trim_ripple_1e-3', 'alternating', 'impulse', 'scales', 'mix']
        a, steps = batch(horizon, lengths, kinds, rng)
        jobs.append((torch.as_tensor(a, device=DEV), torch.as_tensor(steps, device=DEV)))
    want = [rollout.smoothness(a, s).cpu().numpy() for a, s in jobs]
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(DEV), torch.cuda.Stream(DEV)
    outs = {}
    for name, stream, order in (('s1', s1, (0, 1, 2)), ('s2', s2, (1, 2, 0)), ('s1b', s1, (2, 0, 1)), ('s2b', s2, (0, 2, 1))):
        with torch.cuda.stream(stream):
            outs[name] = {j: rollout.smoothness(*jobs[j]) for j in order}
    torch.cuda.synchronize()
    for name, res in outs.items():
        for j, out in res.items():
            assert np.array_equal(bits(out.cpu().numpy()), bits(want[j])), (name, j)


def test_smooth_fitness_is_return_plus_the_smoothness_of_the_flown_actions():
    """Parameters.smooth_fitness: an episode's fitness (Agent.evaluate) and an actor's population fitness (one
    generation's population evaluation, agent.py:229-245) add calc_smoothness of the deflections that were flown"""
    from serl_b200.core import agent as agent_mod
    from serl_b200.envs import config
    from test_boundary_gpu import make_args
    args = make_args(pop=4, hidden=72, smooth_fitness=True)
    assert args.smooth_fitness
    env = config.select_env('PHlab_attitude_nominal')
    torch.manual_seed(7); np.random.seed(7); random.seed(7)
    ag = agent_mod.Agent(args, env)
    w = np.concatenate([ACT['serl10_pop_h72_tanh'][:2], np.stack([OA.flatten(OA.Actor(hidden=72)) for _ in range(2)])])
    ag.pop.genomes.copy_(torch.as_tensor(w))
    ag.gen_frames = 0
    for i in range(4):
        ep = ag.evaluate(ag.pop[i], is_action_noise=False, store_transition=False)
        u = np.asarray(ep.actions, dtype=np.float32).astype(np.float64)           # the fp32 record K6 reads
        ref = calc_smoothness(u)
        ret = float(np.sum(ep.reward_lst))
        assert abs(ep.smoothness - ref) <= REL * abs(ref) + ABS, (i, ep.smoothness, ref)
        assert abs((ep.fitness - ret) - ref) <= REL * abs(ref) + ABS + 1e-12 * abs(ret), (i, ep.fitness, ret, ref)
    # the population's fitness: the mean over its envs of return + smoothness
    draws = ag._draw_population()
    launched = ag._launch_population(draws=draws)
    r = launched[0]
    fit, _, rec = ag._finish_population(launched)
    lv, st, md = launched[2]
    again = rollout.population_rollout(ag.pop.genomes, ag.shape, lv, st, md, horizon=ag._horizon(), actions=True, fitness=False,
                                       **ag._eval_kw())
    torch.cuda.synchronize()
    steps = again.steps.cpu().numpy()
    assert np.array_equal(steps, r.steps.cpu().numpy())
    acts, returns = again.actions.cpu().numpy(), r.returns.cpu().numpy()
    for p in range(4):
        sm = np.array([calc_smoothness(acts[p, e, :steps[p, e]].astype(np.float64)) for e in range(steps.shape[1])])
        assert abs((fit[p] - returns[p].mean()) - sm.mean()) <= REL * np.abs(sm).mean() + ABS + 1e-12 * abs(fit[p]), (p, fit[p], sm)
        assert abs(rec[p, 4] - sm.sum()) <= REL * np.abs(sm).sum() + ABS, (p, rec[p, 4], sm)


def test_evaluation_suite_smoothness_is_that_of_the_zeroed_history():
    """evaluate_population zeroes the last recorded deflection of each trajectory (validate_agent's history is the
    deflection BEFORE each step); on one 8001-step flight its smoothness is calc_smoothness of that same zeroed record"""
    g = ACT['serl10_elite_h72_tanh'][None]
    shape = rollout.actor_shape(72)
    np.random.seed(5)
    refs = evaluation.eval_refs(0)
    res = evaluation.evaluate_population(g, shape, ['nominal'], refs, 0)
    env = evaluation.condition_env('nominal')
    lv, st = evaluation._ref_arrays(refs)
    md = torch.tensor([env.mode_code], dtype=torch.int32, device=DEV)
    r = rollout.population_rollout(torch.as_tensor(g, device=DEV), shape, torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV),
                                   md, horizon=8001, t_max=float(env.t_max), smooth_width=float(refs[0][0].smooth_width),
                                   env_order=rollout.variant_sorted_order(md), fitness=False, actions=True)
    torch.cuda.synchronize()
    r.check()
    n = int(r.steps[0, 0])
    assert n == 8001
    u = r.actions[0, 0, :n].cpu().numpy().astype(np.float64)
    u[n - 1] = 0.0
    ref = calc_smoothness(u)
    got = float(res.sm_trials[0, 0, 0])
    assert abs(got - ref) <= REL * abs(ref) + ABS, (got, ref)
    WORST['direct']['rel'] = max(WORST['direct']['rel'], abs(got - ref) / abs(ref))
