"""BASELINE config 5: wide two-hidden-layer actors ([400,300], [128,128]) on the tensor-core rollout kernel
(csrc/rollout_tc.cu: wgmma .tf32 as 3xTF32, register accumulators, TMA-streamed weight slabs).

The tensor core's accumulation order cannot be restated on a CPU, so this path is compared with the torch fp32 oracle
(oracle/actor.py WideActor = the reference's Actor form with a width list) within a tolerance:
  * forward pass: |action - torch fp32| <= 2e-5 and not worse than 4x the float32 forward pass's own distance from float64;
  * closed loop: termination step identical and return within 1e-4 relative on gentle (small output gain) policies."""
import os

import numpy as np
import pytest
import torch

from oracle import actor as A, fast, refsig

pytestmark = pytest.mark.gpu


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


@pytest.mark.parametrize('widths,activation', [([128, 128], 'tanh'), ([400, 300], 'tanh'), ([64, 48], 'relu'), ([256, 200], 'elu'),
                                               ([8, 16], 'tanh')])
def test_tensor_core_forward_matches_torch_fp32(widths, activation):
    from serl_b200 import rollout
    dev = torch.device('cuda:0')
    g = wide_genomes(1, widths, activation, 3)[0]
    assert g.size == rollout.num_params_wide(widths)
    rs = np.random.RandomState(5)
    obs = np.concatenate([rs.randn(700, 7) * [0.05, 0.05, 0.01, 0.02, 0.02, 0.02, 0.05], rs.randn(300, 7), np.zeros((1, 7))]).astype(np.float32)
    got = rollout.actor_forward_wide(torch.as_tensor(g, device=dev), widths, activation, torch.as_tensor(obs, device=dev)).cpu().numpy()
    net = A.unflatten_wide(g, widths, activation)
    ref32 = net(torch.as_tensor(obs)).detach().numpy()
    ref64 = net.double()(torch.as_tensor(obs, dtype=torch.float64)).detach().numpy()
    err = np.abs(got - ref64).max()
    base = np.abs(ref32 - ref64).max()
    print('widths', widths, activation, 'max |tc - f64| %.2e   max |torch f32 - f64| %.2e' % (err, base))
    assert np.abs(got - ref32).max() <= 2e-5
    assert err <= max(4 * base, 5e-6)


@pytest.mark.parametrize('widths', [[128, 128], [400, 300]])
def test_wide_closed_loop_against_the_c_episode_port(widths):
    from serl_b200 import rollout
    dev = torch.device('cuda:0')
    w = wide_genomes(4, widths, 'tanh', 11, out_gain=0.2)
    modes = ['nominal', 'ice', 'be', 'cg', 'sa', 'nominal']
    lv, st = refsig.make_ref_params(len(modes), seed_base=505)
    md = torch.as_tensor(np.array([rollout.mode_code(m) for m in modes], dtype=np.int32), device=dev)
    r = rollout.population_rollout(torch.as_tensor(w, device=dev), rollout.actor_shape(72), torch.as_tensor(lv, device=dev),
                                   torch.as_tensor(st, device=dev), md, horizon=600, widths=widths)
    torch.cuda.synchronize()
    r.check()
    oret, ostp = fast.evaluate_population_wide(w, widths, lv, st, modes, horizon=600)
    ret, stp = r.returns.cpu().numpy(), r.steps.cpu().numpy()
    assert np.array_equal(stp, ostp), (stp, ostp)
    rel = np.abs(ret - oret) / np.abs(oret)
    assert rel.max() <= 1e-4, rel.max()
    assert np.allclose(r.fitness.cpu().numpy(), oret.mean(1), rtol=1e-4)


def test_config5_shape_many_ctas_deterministic():
    """pop x 256 envs: two 128-env chunks per actor, more CTAs than resident slots, identical genomes -> identical bits
    (the two groups of a CTA take turns on the shared weight ring)."""
    from serl_b200 import rollout
    dev = torch.device('cuda:0')
    for widths in ([400, 300], [128, 128]):
        g = wide_genomes(3, widths, 'tanh', 21, out_gain=0.3)
        w = np.tile(g, (120, 1))
        lv, st = refsig.make_ref_params(256, seed_base=9)
        md = torch.zeros(256, dtype=torch.int32, device=dev)
        r = rollout.population_rollout(torch.as_tensor(w, device=dev), rollout.actor_shape(72), torch.as_tensor(lv, device=dev),
                                       torch.as_tensor(st, device=dev), md, horizon=40, widths=widths)
        torch.cuda.synchronize()
        r.check()
        ret = r.returns.cpu().numpy()
        assert np.isfinite(ret).all() and (r.steps.cpu().numpy() == 40).all()
        for a in range(3, 360):
            assert np.array_equal(ret[a], ret[a % 3]), a


def test_gust_schedule_of_the_tensor_core_kernel_matches_k1():
    """K1-TC takes the gust instantiation from the launch's flag, as K1 does.  A [128, 128] genome has the parameters() layout of
    K1's hidden = 128, num_layers = 1 actor; with zero output weights both kernels emit the same constant action am_tanh1(bo), and
    the env / plant code they share must then give the same bits through the 20-23 s pulse."""
    from serl_b200 import rollout
    dev = torch.device('cuda:0')
    g = wide_genomes(1, [128, 128], 'tanh', 3)[0]
    g[-3 - 3 * 128:-3] = 0.0
    g[-3:] = [0.02, -0.01, 0.01]
    w = torch.as_tensor(g[None], device=dev)
    modes = ['gust', 'test', 'nominal', 'cg-timed', 'gust', 'nominal']
    lv, st = refsig.make_ref_params(len(modes), seed_base=77, t_max=25)
    lv, st = torch.as_tensor(lv, device=dev), torch.as_tensor(st, device=dev)
    md = torch.as_tensor(np.array([rollout.mode_code(m) for m in modes], dtype=np.int32), device=dev)
    run = lambda shape, widths, gust: rollout.population_rollout(w, shape, lv, st, md, horizon=2501, t_max=25.0, widths=widths, gust=gust)
    k1 = run(rollout.actor_shape(128, 1, 'tanh'), None, True)
    tc = run(rollout.actor_shape(72), [128, 128], True)
    torch.cuda.synchronize()
    k1.check()
    tc.check()
    assert torch.equal(tc.steps, k1.steps), (tc.steps, k1.steps)
    assert torch.equal(tc.returns, k1.returns), (tc.returns, k1.returns)
    steps, ret = tc.steps.cpu().numpy()[0], tc.returns.cpu().numpy()[0]
    gust = np.array([m in ('gust', 'test') for m in modes])
    assert (steps[gust] > 2301).all(), steps                     # flown through the whole pulse
    # without the flag the gust envs fly the nominal dynamics, and that is reported
    nominal = run(rollout.actor_shape(72), [128, 128], False)
    torch.cuda.synchronize()
    assert (ret[gust] != nominal.returns.cpu().numpy()[0][gust]).all()      # the pulse was really on
    with pytest.raises(Exception, match='gust'):
        nominal.check()
