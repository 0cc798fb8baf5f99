"""K1-TC (csrc/rollout_tc.cu) across the whole width-list domain it accepts: every depth from 2 to 9 widths, w0 up to 1024,
hidden widths on and off both paddings (8 and 64), the lists at the shared-memory edge, and every kernel instantiation.

Genomes are random WideActors whose LayerNorm parameters differ from layer to layer (test_k1_tc_domain.genome): a kernel
that read another layer's gamma or beta, or a wrong per-layer or per-actor offset into the small block or the tile block,
changes the actions.  The tensor cores' accumulation order cannot be restated on a CPU, so the bars are:
  - forward pass: max |tc - f64| <= max(4 * max |torch f32 - f64|, 5e-6) against the float64 reference forward64, or
    4x the error of a float64 model of the kernel's own rounding where that is larger (forward_check); |tc - torch f32|
    <= 2e-5 at scale 1 where w0 <= 321;
  - closed loop: identical termination steps and returns within 1e-4 relative of the C episode port;
  - launches that must agree (tracking on / off, per-actor refs that repeat the shared ones, an actor flown in a population
    or alone): bit for bit."""
import numpy as np
import pytest
import torch

from oracle import actor as A, fast, refsig
from test_k1_tc_domain import (EDGE_1024_W, EDGE_1024_WW, EDGE_UNIFORM, EDGE_W0_320, edge_lists, forward64, forward_3xtf32, genome,
                               largest_accepted, width_grid)

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
REL_TOL = 1e-4
ACTS = ('tanh', 'elu', 'relu')
MODES = ['nominal', 'ice', 'be', 'cg', 'sa', 'jr']


def observations(n, seed):
    """n rows cycling through flight-like, N(0, 1), x30 (saturating) and zero rows"""
    rs = np.random.RandomState(seed)
    kinds = np.stack([rs.randn(n, 7) * [0.05, 0.05, 0.01, 0.02, 0.02, 0.02, 0.05], rs.randn(n, 7), rs.randn(n, 7) * 30.0, np.zeros((n, 7))])
    return kinds[np.arange(n) % 4, np.arange(n)].astype(np.float32)


def forward_check(widths, activation, scale, obs, seed):
    """the device forward pass of one genome against forward64 and torch fp32; returns the device actions.
    The float64 bar is 4x float32's own error, or 4x the error of forward_3xtf32 (the kernel's TF32 split with the tensor
    cores' truncating accumulation) where that is larger: it grows with a layer's input width, to several times float32's
    at w0 = 1024.  The torch fp32 bar holds with margin up to w0 = 321 (the largest K of a layer <= 328)."""
    from serl_b200 import rollout
    g = genome(widths, activation, seed, scale=scale)
    got = rollout.actor_forward_wide(torch.as_tensor(g, device=DEV), widths, activation, torch.as_tensor(obs, device=DEV)).cpu().numpy()
    ref64 = forward64(g, widths, activation, obs)
    with torch.no_grad():
        ref32 = A.unflatten_wide(g, widths, activation)(torch.as_tensor(obs)).numpy()
    err, base, d32 = np.abs(got - ref64).max(), np.abs(ref32 - ref64).max(), np.abs(got - ref32).max()
    model = np.abs(forward_3xtf32(g, widths, activation, obs) - ref64).max() if err > max(4 * base, 5e-6) else float('nan')
    print('%s %s x%g n=%d: max |tc - f64| %.2e  max |torch f32 - f64| %.2e  max |3xtf32 model - f64| %.2e  max |tc - torch f32| %.2e'
          % (widths, activation, scale, obs.shape[0], err, base, model, d32))
    assert err <= max(4 * base, 5e-6) or err <= 4 * model, (widths, activation, scale, err, base, model)
    if scale == 1.0 and widths[0] <= 321:
        assert d32 <= 2e-5, (widths, activation, d32)
    return got


def refs(n, seed):
    lv, st = refsig.make_ref_params(n, seed_base=seed)
    return lv, st, torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV)


def modes_tensor(modes):
    from serl_b200 import rollout
    return torch.as_tensor(np.array([rollout.mode_code(m) for m in modes], dtype=np.int32), device=DEV)


def fly(w, widths, activation, modes, seed, horizon, **kw):
    """population_rollout of genomes w [pop, P] (numpy) on K1-TC -> (result, ref levels, ref starts)"""
    from serl_b200 import rollout
    lv, st, dlv, dst = refs(len(modes), seed)
    r = rollout.population_rollout(torch.as_tensor(w, device=DEV), rollout.actor_shape(72, 3, activation), dlv, dst, modes_tensor(modes),
                                   horizon=horizon, widths=widths, **kw)
    torch.cuda.synchronize()
    r.check()
    return r, lv, st


def against_port(r, w, widths, activation, modes, lv, st, horizon, what):
    oret, ostp = fast.evaluate_population_wide(w, widths, lv, st, modes, activation=activation, horizon=horizon)
    ret, stp = r.returns.cpu().numpy(), r.steps.cpu().numpy()
    assert np.array_equal(stp, ostp), (what, stp, ostp)
    rel = np.abs(ret - oret) / np.abs(oret)
    print(what, 'max rel return diff %.2e' % rel.max())
    assert rel.max() <= REL_TOL, (what, rel.max())
    return stp


def closed_loop(widths, activation, seed, gains=(0.2, 0.3), modes=('nominal', 'ice', 'be', 'cg'), horizon=300, **kw):
    w = np.stack([genome(widths, activation, seed + k, out_gain=g) for k, g in enumerate(gains)])
    r, lv, st = fly(w, widths, activation, list(modes), seed, horizon, **kw)
    return against_port(r, w, widths, activation, list(modes), lv, st, horizon, (widths, activation))


# ---- 1. the forward pass over the whole grid ----------------------------------------------------------------------------
@pytest.mark.parametrize('widths,activation', width_grid())
def test_forward_matches_float64_over_the_grid(widths, activation):
    """scale 1, and the same genome x3 to drive the activations into saturation"""
    obs = observations(3301, len(widths) + widths[-1])
    for scale in (1.0, 3.0):
        forward_check(widths, activation, scale, obs, 100 * len(widths) + widths[0])


# ---- 2. observation counts: partial groups, n = 1, and a grid that strides -----------------------------------------------
@pytest.mark.parametrize('widths,activation', [([321, 257], 'tanh'), ([129, 65, 127, 63], 'elu')])
def test_observation_counts(widths, activation):
    """The grid is min(ceil(n / 256), SMs) CTAs of two 128-row groups, so past 2 * SMs * 256 rows it strides.  At
    2 * SMs * 256 + 65 group 0 of CTA 0 runs three trips (the last one on 65 rows) and group 1 two; at + 129 group 1 runs a
    third trip on one row.  Every row's action is the one it gets in any other launch, bit for bit."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    big = 2 * sms * 256
    obs = observations(big + 129, 7)
    full = forward_check(widths, activation, 1.0, obs, 31)
    for n in (1, 63, 64, 65, 255, 256, 257, big + 65):
        got = forward_check(widths, activation, 1.0, obs[:n], 31)
        assert np.array_equal(got.view(np.uint32), full[:n].view(np.uint32)), (widths, n)


# ---- 3. the shared-memory edge ---------------------------------------------------------------------------------------------
def _forward_accepts(widths):
    from serl_b200 import _native, rollout
    g = torch.zeros(rollout.num_params_wide(widths), dtype=torch.float32, device=DEV)
    try:
        rollout.actor_forward_wide(g, widths, 'tanh', torch.zeros((5, 7), dtype=torch.float32, device=DEV))
    except _native.NativeError as e:
        assert '(-3)' in str(e), str(e)
        return False
    return True


def test_the_largest_accepted_lists_are_the_pinned_edge():
    """searched with real serl_actor_forward_wide calls (a refused list launches nothing)"""
    for n in range(2, 10):
        assert largest_accepted(_forward_accepts, lambda x: [x] * n, hi=320) == EDGE_UNIFORM[n], n
    assert largest_accepted(_forward_accepts, lambda x: [1024, x], hi=320) == EDGE_1024_W
    assert largest_accepted(_forward_accepts, lambda x: [1024, x, x], hi=320) == EDGE_1024_WW
    assert largest_accepted(_forward_accepts, lambda x: [x, 320]) == EDGE_W0_320
    torch.cuda.synchronize()


@pytest.mark.parametrize('good,bad', edge_lists() + [([320, 320], [320, 321])])
def test_edge_lists_fly_and_the_next_width_up_is_refused(good, bad):
    from serl_b200 import _native, rollout
    act = ACTS[len(good) % 3]
    forward_check(good, act, 1.0, observations(1001, 3), 17)
    forward_check(good, act, 3.0, observations(1001, 3), 17)
    closed_loop(good, act, 40 + len(good), horizon=200)
    lib = _native.lib()
    w = torch.zeros((2, rollout.num_params_wide(bad)), dtype=torch.float32, device=DEV)
    _, _, dlv, dst = refs(2, 3)
    torch.cuda.synchronize()
    before = lib.serl_launch_count()
    with pytest.raises(_native.NativeError, match=r'\(-3\)'):
        rollout.population_rollout(w, rollout.actor_shape(72), dlv, dst, modes_tensor(['nominal', 'ice']), horizon=50, widths=bad)
    with pytest.raises(_native.NativeError, match=r'\(-3\)'):
        rollout.actor_forward_wide(w[0].contiguous(), bad, 'tanh', torch.zeros((5, 7), dtype=torch.float32, device=DEV))
    assert lib.serl_launch_count() == before, bad


# ---- 4. the closed loop against the C episode port ---------------------------------------------------------------------
@pytest.mark.parametrize('widths,activation', width_grid()[:24])
def test_closed_loop_at_every_depth_and_activation(widths, activation):
    """three lists per depth from 2 to 9 widths, one per activation (w0 = 1024 among them)"""
    closed_loop(widths, activation, 7 * len(widths) + widths[-1])


FULL = {2: [129, 65], 3: [96, 257, 64], 4: [63, 127, 65, 320], 5: [128] * 5, 6: [128] * 6, 7: [9, 65, 63, 64, 15, 127, 129],
        8: [100] * 8, 9: [64] * 9}


@pytest.mark.parametrize('n', sorted(FULL))
def test_strict_parity_at_full_horizon(n):
    """gentle output gains fly most episodes to the end, the larger ones end some early"""
    stp = closed_loop(FULL[n], 'tanh', 900 + n, gains=(0.2, 0.3, 1.0, 3.0), modes=('nominal', 'se', 'ice', 'cg'), horizon=2001)
    assert (stp == 2001).any() and (stp < 2001).any(), stp          # full episodes and early terminations


# ---- 5. every kernel instantiation -----------------------------------------------------------------------------------------
def host_track_sums(r, modes):
    """the tracking-error sums rebuilt from the trace (as test_eval_suite_population_gpu.host_sums, noiseless)"""
    from serl_b200 import evaluation, rollout
    steps, trace = r.steps.cpu().numpy(), r.trace.cpu().numpy()
    out = np.zeros(steps.shape + (4,))
    for a in range(steps.shape[0]):
        for j in range(steps.shape[1]):
            k = int(steps[a, j])
            tr = trace[a, j, :k]
            x_after = tr[:, rollout.TRACE_X]
            ref = tr[:, rollout.TRACE_ERR] + x_after[:, [7, 6, 5]]
            x0 = evaluation.reset_state(rollout.initial_state(rollout.mode_variant(rollout.mode_code(modes[j]))), None)
            e = ref - np.vstack((x0[None], x_after[:-1]))[:, [7, 6, 5]]
            out[a, j] = [np.abs(e[:, 0]).sum(), np.abs(e[:, 1]).sum(), np.abs(e[:, 2]).sum(), e[:, 2].sum()]
    return out


@pytest.mark.parametrize('activation', ACTS)
@pytest.mark.parametrize('widths', [[129, 65], [65, 129, 63]], ids=['two', 'deep'])
def test_every_rollout_instantiation(widths, activation):
    """kernels[act][gust][deep], track_kernels[act][deep] and per_actor_kernels[act][gust][deep] of rollout_tc_impl"""
    from serl_b200 import rollout
    horizon, seed = 300, 60 + len(widths)
    w = np.stack([genome(widths, activation, seed + k, out_gain=g) for k, g in enumerate((0.2, 0.3))])
    sh = rollout.actor_shape(72, 3, activation)
    modes = MODES
    lv, st, dlv, dst = refs(len(modes), seed)
    md = modes_tensor(modes)
    dw = torch.as_tensor(w, device=DEV)
    run = lambda *a, **kw: rollout.population_rollout(dw, sh, *a, horizon=horizon, widths=widths, **kw)
    shared = {gust: run(dlv, dst, md, gust=gust) for gust in (False, True)}
    pop = w.shape[0]
    per = {gust: run(dlv[None].repeat(pop, 1, 1, 1).contiguous(), dst[None].repeat(pop, 1, 1, 1).contiguous(), md[None].repeat(pop, 1).contiguous(),
                     gust=gust) for gust in (False, True)}
    tracked = run(dlv, dst, md, gust=True, track=True, trace=True)
    torch.cuda.synchronize()
    for r in list(shared.values()) + list(per.values()) + [tracked]:
        r.check()
    for gust in (False, True):
        against_port(shared[gust], w, widths, activation, modes, lv, st, horizon, (widths, activation, 'gust' if gust else 'plain'))
        assert torch.equal(per[gust].returns, shared[gust].returns) and torch.equal(per[gust].steps, shared[gust].steps), gust
    # tracking (and the trace) does not perturb the trajectories, and its sums are the trace's
    assert torch.equal(tracked.returns, shared[True].returns) and torch.equal(tracked.steps, shared[True].steps)
    got, want = tracked.track.cpu().numpy(), host_track_sums(tracked, modes)
    assert np.all(np.abs(got - want) <= 1e-12 * np.abs(want) + 1e-300), np.abs(got - want).max()


@pytest.mark.parametrize('activation', ACTS)
@pytest.mark.parametrize('widths', [[129, 65], [65, 129, 63]], ids=['two', 'deep'])
def test_every_forward_instantiation(widths, activation):
    """actor_forward_tc_kernel[act][deep] on a genome with per-layer LayerNorm parameters"""
    forward_check(widths, activation, 1.0, observations(515, 5), 3)


# ---- 6. per-actor offsets ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('widths,activation', [([129, 65], 'tanh'), ([200, 72], 'relu'), ([65, 129, 63, 15], 'elu')])
def test_each_actor_of_a_population_flies_as_it_flies_alone(widths, activation):
    """Distinct genomes, each with its own LayerNorm parameters, and 129 envs: an actor's second chunk holds one env.  Actor a
    in the population must give the bits it gives alone, so the per-actor small_floats and tile_floats strides are right
    (small_floats is 4 mod 32 for every list)."""
    pop, n_envs, horizon = 5, 129, 200
    w = np.stack([genome(widths, activation, 500 + a, out_gain=0.3) for a in range(pop)])
    modes = [MODES[i % len(MODES)] for i in range(n_envs)]
    both = fly(w, widths, activation, modes, 21, horizon, actions=True)[0]
    for a in range(pop):
        alone = fly(w[a:a + 1], widths, activation, modes, 21, horizon, actions=True)[0]
        assert torch.equal(both.steps[a], alone.steps[0]), a
        assert torch.equal(both.returns[a], alone.returns[0]), a
        flown = torch.arange(horizon, device=DEV)[None] < alone.steps[0][:, None]          # the actions past a trajectory's end are not written
        assert torch.equal(both.actions[a][flown], alone.actions[0][flown]), a
    # the genomes really differ, so a wrong stride would show
    assert not torch.equal(both.returns[0], both.returns[1])
