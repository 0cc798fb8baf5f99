"""K7, the fused TD3 learner (csrc/td3.cu, serl_b200/td3_fused.py), against a float64 reference across the inputs
serl_td3_learn accepts.

Every case runs K7 with its draws recorded (batch rows, clipped target-policy noise, CAPS uniforms) and replays them on the
CPU through the fp32 oracle (oracle/td3.py, bit-exact against TD3.update_parameters) and through its float64 copy
(oracle.td3.as_float64).  Then all eight blocks of the learner state (actor θ, actor target, actor Adam m, actor Adam v, the
same four for the critic) are compared per tensor, and the loss series as a whole, against an error budget:

    ||K7 - f64|| <= C * ||torch32 - f64|| + FLOOR * scale

where scale is the float64 displacement from the start of the run for parameters and targets and ||f64|| for Adam moments
and losses.  A tensor that the float64 update leaves bit-unchanged (the actor on critic-only iterations, the actor target
under a champion target, both targets between actor iterations) must be bit-unchanged in K7 too.  Cases: every hidden
width and layer count up to 5, batches 1..128 (n_valid == batch included), gradient clipping of the critic alone and of
both nets (the oracle's pre-clip norms prove that the clip fired), warm Adam moments at iteration 1000 with the critic's
and the actor's own step counts, the CAPS term combinations, a strided replay with NaN rows past n_valid, and 300-step
runs.  Apart from the state, the draws are judged on their own (distribution, independence, reproducibility) and the
status words are checked.

Budget: C = 4 (as tests/test_wide_actor_gpu.py); FLOOR = 1e-4 for parameters and targets, 4e-6 for Adam moments, 1e-6
for the losses.  Measured on an H100 80GB HBM3 (700 W) over all 61 replayed cases:
  * per block, K7's largest distance from float64 is within a few times torch32's: one step, parameters 5e-5..3.5e-4 of
    the displacement (torch32 the same), moments <= 1e-6 of their norm; 300 steps on flight rows, actor 1.7e-4 / critic
    3.9e-5 of the displacement (torch32 identical to two digits), moments <= 5.6e-6 (torch32 4.9e-6); td loss <= 2.1e-7,
    pg <= 3.6e-7 relative (torch32 is often luckier: down to 1e-9);
  * per tensor, no parameter or target tensor is beyond C x torch32.  Up to 6 moment tensors per case are (ratio up to
    466), all tiny tensors whose torch32 moment rounds almost exactly: the critic heads' output weight / bias, the actor's
    output bias, LayerNorm vectors.  The largest of them is 1.6e-6 of ||f64||, under the 4e-6 floor.
  * the parameter floor covers the one tail seen: under other draws one 64 x 64 critic weight at Adam's first step was
    7.8x torch32 (1.1e-4 of the displacement).  At t = 1 Adam's update is lr * g / (|g| + 1e-8), so an element whose
    gradient is within rounding of zero moves by an amount set by that rounding, in either fp32 order.
Each of these edits to csrc/td3.cu fails tests here: the norm's last partial chunk dropped (the clipping cases), beta2 =
0.99 in the v update, the critic's step count in the actor's bias correction, noise * noise_sd^2 (the noise
distribution), Floyd keeping a repeated draw (n_valid == batch)."""
import os
import types

import numpy as np
import pytest
import torch

from oracle import td3 as O

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
C, THETA_FLOOR, MOMENT_FLOOR, LOSS_FLOOR = 4.0, 1e-4, 4e-6, 1e-6
BLOCKS = ('actor', 'actor_target', 'actor_m', 'actor_v', 'critic', 'critic_target', 'critic_m', 'critic_v')
LR = 0.00018643512599969097
NOISE_SD = 0.2962183114680794


def td3_args(hidden=72, num_layers=3, activation='tanh', use_caps=True, batch_size=86, policy_update_freq=3, noise_sd=NOISE_SD):
    return types.SimpleNamespace(device=DEV, individual_bs=100, hidden_size=hidden, num_layers=num_layers,
                                 activation_actor=activation, state_dim=7, action_dim=3, lr=LR, gamma=0.98, tau=0.005,
                                 noise_sd=noise_sd, noise_clip=0.5, policy_update_freq=policy_update_freq, use_caps=use_caps,
                                 batch_size=batch_size, seed=7)


def synthetic_rows(n, seed=0, reward_scale=1.0):
    g = torch.Generator().manual_seed(seed)
    rows = torch.randn((n, 19), generator=g) * 0.3
    rows[:, 7:10] = torch.rand((n, 3), generator=g) * 2 - 1
    rows[:, 17] = -torch.rand(n, generator=g) * reward_scale
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


def fused(args, seed=7):
    from serl_b200.td3_fused import FusedTD3
    torch.manual_seed(11)
    return FusedTD3(args, seed=seed)


def torch_learner(f):
    """a CPU TD3 holding the weights (and caps_dict) of the FusedTD3 f, fresh Adam state"""
    from serl_b200.core.td3 import TD3
    t = TD3(types.SimpleNamespace(**dict(vars(f.args), device=torch.device('cpu'))))
    for mf, mo in ((f.actor, t.actor), (f.actor_target, t.actor_target), (f.critic, t.critic), (f.critic_target, t.critic_target)):
        for pf, po in zip(mf.parameters(), mo.parameters()):
            po.data.copy_(pf.data.cpu())
    t.caps_dict = None if f.caps_dict is None else dict(f.caps_dict)
    return t


def k7_blocks(f):
    """K7's state as the eight blocks, each a list of float64 CPU tensors in parameters() order"""
    st = f.state.detach().cpu().double()
    shapes = [[p.shape for p in m.parameters()] for m in (f.actor, f.critic)]
    out, off = [], 0
    for b in range(8):
        blk = []
        for s in shapes[b // 4]:
            k = int(np.prod(s))
            blk.append(st[off:off + k].view(s))
            off += k
        out.append(blk)
    assert off == st.numel()
    return out


def torch_blocks(t):
    out = []
    for mods, opt in (((t.actor, t.actor_target), t.actor_optim), ((t.critic, t.critic_target), t.critic_optim)):
        out += [[p.detach().double().clone() for p in m.parameters()] for m in mods]
        out += [[opt.state[p][key].double().clone() if p in opt.state else torch.zeros(p.shape, dtype=torch.float64)
                 for p in mods[0].parameters()] for key in ('exp_avg', 'exp_avg_sq')]
    return out


class Reference:
    """the fp32 oracle and its float64 copy of a FusedTD3, and the state they start from"""

    def __init__(self, f):
        self.t32 = torch_learner(f)
        self.start_from(f)

    def start_from(self, f):
        self.t64 = O.as_float64(self.t32)
        self.start = torch_blocks(self.t32)
        assert all(torch.equal(a, b) for x, y in zip(self.start, k7_blocks(f)) for a, b in zip(x, y))

    def replay(self, rows_cpu, launch, first_iteration, champion=False):
        """the recorded draws through both; returns fp32 and fp64 losses [n, 2] (td, pg) and the pre-clip norms per step"""
        idx, noise, caps = launch.indices.cpu().long(), launch.noise.cpu(), launch.caps.cpu()
        use_caps = self.t32.caps_dict is not None
        l32, l64, norms = [], [], []
        for k in range(idx.shape[0]):
            it, nk = first_iteration + k, []
            rows = rows_cpu[idx[k]]
            pg, td = O.update_parameters(self.t32, rows, it, noise[k], caps[k] if use_caps else None, champion, norms=nk)
            pg6, td6 = O.update_parameters(self.t64, rows.double(), it, noise[k].double(), caps[k].double() if use_caps else None, champion)
            l32.append((float(td), float('nan') if pg is None else float(pg)))
            l64.append((float(td6), float('nan') if pg6 is None else float(pg6)))
            norms.append(nk)
        return np.array(l32), np.array(l64), norms

    def check(self, f, launch, l32, l64, label):
        """the error budget on every tensor of the eight blocks and on the td / pg series"""
        K, T, D = k7_blocks(f), torch_blocks(self.t32), torch_blocks(self.t64)
        bad, report, ratio, floored, count = [], [], 0.0, [], 0
        for b, name in enumerate(BLOCKS):
            wk = wt = 0.0
            floor = THETA_FLOOR if b % 4 < 2 else MOMENT_FLOOR
            for j, (k, t, d, s) in enumerate(zip(K[b], T[b], D[b], self.start[b])):
                if torch.equal(d, s):                 # untouched by the update: untouched by K7
                    if not torch.equal(k, s):
                        bad.append((name, j, 'changed'))
                    continue
                scale = float((d - s).norm()) if b % 4 < 2 else float(d.norm())
                ek, et = float((k - d).norm()) / scale, float((t - d).norm()) / scale
                wk, wt = max(wk, ek), max(wt, et)
                ratio, count = max(ratio, ek / max(et, 1e-30)), count + 1
                if ek > C * et:
                    floored.append('%s[%d]%s %.1e/%.1e' % (name, j, tuple(k.shape), ek, et))
                if not ek <= C * et + floor:
                    bad.append((name, j, tuple(k.shape), '%.2e vs torch32 %.2e' % (ek, et)))
            report.append('%s %.1e/%.1e' % (name, wk, wt))
        got = launch.losses.cpu().double().numpy()
        for c, name in ((0, 'td'), (1, 'pg')):
            on = ~np.isnan(l64[:, c])
            assert np.array_equal(np.isnan(got[:, c]), ~on) and np.array_equal(np.isnan(l32[:, c]), ~on), name
            if on.any():
                scale = np.linalg.norm(l64[on, c])
                ek, et = np.linalg.norm(got[on, c] - l64[on, c]) / scale, np.linalg.norm(l32[on, c] - l64[on, c]) / scale
                report.append('%s %.1e/%.1e' % (name, ek, et))
                if not ek <= C * et + LOSS_FLOOR:
                    bad.append((name, '%.2e vs torch32 %.2e' % (ek, et)))
        print('\n[%s] K7/torch32 vs f64: %s; max ratio %.1f, %d of %d tensors beyond C: %s'
              % (label, ', '.join(report), ratio, len(floored), count, ' '.join(floored)))
        assert not bad, (label, bad)


def run_and_check(f, ref, rows, n, first_iteration, label, champion=False, n_valid=None):
    """n steps of K7 on device rows (a [N, >= 19] view), replayed; returns the launch and the oracle's pre-clip norms"""
    n_valid = rows.shape[0] if n_valid is None else n_valid
    r = f.run(rows, n_valid, n, first_iteration, champion, record=True)
    r.check()
    rows_cpu = rows[:n_valid, :19].cpu()
    l32, l64, norms = ref.replay(rows_cpu, r, first_iteration, champion)
    ref.check(f, r, l32, l64, label)
    return r, norms


# ---- shapes, batches ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('hidden,num_layers', [(32, 2), (64, 1), (64, 2), (96, 1), (96, 4), (128, 5)])
@pytest.mark.parametrize('activation', ['tanh', 'elu', 'relu'])
@pytest.mark.parametrize('iteration', [1, 3])
def test_every_shape_matches_float64(hidden, num_layers, activation, iteration):
    f = fused(td3_args(hidden, num_layers, activation))
    ref = Reference(f)
    rows = synthetic_rows(3000, seed=hidden + num_layers).to(DEV)
    run_and_check(f, ref, rows, 1, iteration, 'h%d L%d %s it%d' % (hidden, num_layers, activation, iteration))


@pytest.mark.parametrize('batch', [1, 2, 31, 32, 33, 64, 127, 128])
def test_every_batch_matches_float64(batch):
    f = fused(td3_args(batch_size=batch))
    ref = Reference(f)
    rows = synthetic_rows(3000, seed=batch).to(DEV)
    run_and_check(f, ref, rows, 3, 1, 'B%d' % batch)


@pytest.mark.parametrize('batch', [1, 33, 128])
def test_batch_equal_to_the_valid_rows_takes_every_row(batch):
    f = fused(td3_args(batch_size=batch))
    ref = Reference(f)
    rows = synthetic_rows(batch, seed=batch).to(DEV)
    r, _ = run_and_check(f, ref, rows, 3, 1, 'B%d = n_valid' % batch)
    for step in r.indices.cpu().numpy():
        assert np.array_equal(np.sort(step), np.arange(batch))


# ---- gradient clipping ---------------------------------------------------------------------------------------------------

def test_clipped_critic_matches_float64():
    f = fused(td3_args())
    ref = Reference(f)
    rows = synthetic_rows(3000, seed=5, reward_scale=30.0).to(DEV)
    _, norms = run_and_check(f, ref, rows, 3, 1, 'critic clipped')
    assert all(n[0] > 10 for n in norms), norms             # every critic step clipped (measured ~156)
    assert norms[2][1] < 10, norms                           # the actor step not


def test_clipped_critic_and_actor_match_float64():
    f = fused(td3_args())
    with torch.no_grad():
        f.critic.q1[4].weight.mul_(300.0)                    # the critic's, not the target's
    ref = Reference(f)
    rows = synthetic_rows(3000, seed=5).to(DEV)
    _, norms = run_and_check(f, ref, rows, 3, 1, 'both clipped')
    assert all(n[0] > 10 for n in norms) and norms[2][1] > 10, norms      # measured ~654 and ~108


# ---- Adam past its first steps --------------------------------------------------------------------------------------------

def warm_adam(f, ref, critic_steps, actor_steps, seed=3):
    """random moments (v >= 0) in K7's state and in both torch optimisers, with the given step counts"""
    g = torch.Generator().manual_seed(seed)
    pa = sum(p.numel() for p in f.actor.parameters())
    pc = sum(p.numel() for p in f.critic.parameters())
    for mod, opt, off, count, steps in ((ref.t32.actor, ref.t32.actor_optim, 2 * pa, pa, actor_steps),
                                        (ref.t32.critic, ref.t32.critic_optim, 4 * pa + 2 * pc, pc, critic_steps)):
        m = torch.randn(count, generator=g) * 0.02
        v = m * m + torch.rand(count, generator=g) * 1e-4
        f.state[off:off + count].copy_(m)
        f.state[off + count:off + 2 * count].copy_(v)
        o = 0
        for p in mod.parameters():
            k = p.numel()
            opt.state[p] = {'step': torch.tensor(float(steps)), 'exp_avg': m[o:o + k].view(p.shape).clone(),
                            'exp_avg_sq': v[o:o + k].view(p.shape).clone()}
            o += k
    f.critic_steps, f.actor_steps = critic_steps, actor_steps
    ref.start_from(f)


@pytest.mark.parametrize('freq', [1, 2, 3])
@pytest.mark.parametrize('champion', [False, True])
def test_warm_adam_at_iteration_1000_matches_float64(freq, champion):
    f = fused(td3_args(policy_update_freq=freq))
    ref = Reference(f)
    warm_adam(f, ref, 999, 999 // freq)                      # what a run over iterations 1..999 leaves
    rows = synthetic_rows(3000, seed=freq).to(DEV)
    run_and_check(f, ref, rows, 4, 1000, 'warm Adam freq %d champion %d' % (freq, champion), champion=champion)
    step = lambda opt: int(next(iter(opt.state.values()))['step'])
    assert (f.critic_steps, f.actor_steps) == (step(ref.t32.critic_optim), step(ref.t32.actor_optim)) == \
        (1003, 999 // freq + sum(1 for it in range(1000, 1004) if it % freq == 0))


# ---- CAPS terms ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('lambda_t,lambda_s', [(0.1, 0.5), (0.0, 0.0), (0.1, 0.0)])
def test_caps_terms_match_float64(lambda_t, lambda_s):
    f = fused(td3_args())
    f.caps_dict = {'lambda_t': lambda_t, 'lambda_s': lambda_s, 'eps_sd': 0.05}
    ref = Reference(f)
    rows = synthetic_rows(3000, seed=8).to(DEV)
    run_and_check(f, ref, rows, 3, 1, 'CAPS lt %g ls %g' % (lambda_t, lambda_s))


# ---- replay layout -----------------------------------------------------------------------------------------------------------

def test_strided_replay_never_reads_past_n_valid():
    """K1's 20-column replay rows as a [:, :19] view (row stride 20); rows past n_valid and the 20th column are NaN, so a
    row or a column read outside the transitions shows as a NaN loss and a status bit"""
    n = 2000
    f = fused(td3_args())
    ref = Reference(f)
    buf = torch.full((n + 300, 20), float('nan'))
    buf[:n, :19] = synthetic_rows(n, seed=12)
    rows = buf.to(DEV)[:, :19]
    assert rows.stride(0) == 20
    r, _ = run_and_check(f, ref, rows, 6, 1, 'strided replay', n_valid=n)
    assert int(r.status.item()) == 0 and torch.isfinite(r.losses[:, 0]).all()
    assert int(r.indices.max()) < n


# ---- long runs -------------------------------------------------------------------------------------------------------------

def test_300_steps_on_flight_rows_match_float64():
    f = fused(td3_args())
    ref = Reference(f)
    run_and_check(f, ref, flight_rows(), 300, 1, '300 steps, flight rows')


def test_300_steps_with_both_clips_match_float64():
    f = fused(td3_args())
    with torch.no_grad():
        f.critic.q1[4].weight.mul_(300.0)
    ref = Reference(f)
    rows = synthetic_rows(3000, seed=0, reward_scale=30.0).to(DEV)
    _, norms = run_and_check(f, ref, rows, 300, 1, '300 steps, both clipped')
    actor = [n[1] for n in norms if len(n) > 1]
    assert len(actor) == 100 and all(n[0] > 10 for n in norms), min(n[0] for n in norms)
    assert all(a > 10 for a in actor[:10]), actor[:10]     # the actor's norm decays below the clip after ~18 actor steps


# ---- the draws on their own ------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def draws():
    """2000 steps x 86 rows of recorded draws at two noise_sd (the second wider than the clip)"""
    rows = synthetic_rows(5000, seed=9).to(DEV)
    out = {}
    for sd in (NOISE_SD, 0.6):
        f = fused(td3_args(hidden=32, num_layers=1, noise_sd=sd))
        r = f.run(rows, rows.shape[0], 2000, 1, record=True)
        out[sd] = (r.noise.cpu().double().numpy(), r.caps.cpu().double().numpy(), r.indices.cpu().numpy())
    return out


@pytest.mark.parametrize('sd', [NOISE_SD, 0.6])
def test_target_noise_is_a_clipped_normal(draws, sd):
    from scipy import stats
    noise = draws[sd][0].reshape(-1)
    clip, n = 0.5, noise.size
    assert np.abs(noise).max() == clip
    p = 2 * stats.norm.cdf(-clip / np.float32(sd))
    for k, q in ((np.sum(np.abs(noise) == clip), p), (np.sum(noise == clip), p / 2), (np.sum(noise == -clip), p / 2)):
        assert abs(k - n * q) <= 5 * np.sqrt(n * q * (1 - q)), (sd, k, n * q)
    inner = noise[np.abs(noise) < clip]
    lo, hi = stats.norm.cdf(-clip / sd), stats.norm.cdf(clip / sd)
    ks = stats.kstest(inner, lambda x: (stats.norm.cdf(x / sd) - lo) / (hi - lo))
    assert ks.pvalue > 1e-3, (sd, ks)


def test_caps_draws_are_uniform(draws):
    from scipy import stats
    u = draws[NOISE_SD][1].reshape(-1)
    assert u.min() >= 0.0 and u.max() < 1.0
    ks = stats.kstest(u, 'uniform')
    assert ks.pvalue > 1e-3, ks


def test_draws_are_uncorrelated(draws):
    """noise channels (0, 1 are the two outputs of one Box-Muller draw; also their squares), CAPS channels, noise against
    CAPS, adjacent rows and adjacent steps: |corr| < 5 / sqrt(n)"""
    noise, caps, _ = draws[NOISE_SD]
    pairs = [(noise[..., 0], noise[..., 1]), (noise[..., 0] ** 2, noise[..., 1] ** 2), (noise[..., 0], noise[..., 2]),
             (noise[..., 1], noise[..., 2]), (noise[..., 0], caps[..., 0]), (noise[..., 2], caps[..., 6])]
    pairs += [(caps[..., i], caps[..., i + 1]) for i in range(6)]
    for x in (noise[..., 0], noise[..., 2], caps[..., 0], caps[..., 4]):
        pairs += [(x[:, :-1], x[:, 1:]), (x[:-1], x[1:])]               # adjacent rows, adjacent steps
    for k, (a, b) in enumerate(pairs):
        a, b = a.reshape(-1), b.reshape(-1)
        r = np.corrcoef(a, b)[0, 1]
        assert abs(r) < 5 / np.sqrt(a.size), (k, r)


def test_draws_depend_on_seed_and_iteration_not_on_the_launch():
    rows = synthetic_rows(3000, seed=4).to(DEV)
    args = td3_args(hidden=32, num_layers=1)
    a, b = fused(args, seed=7), fused(args, seed=8)
    long_ = a.run(rows, 3000, 6, 20, record=True)
    one = a.run(rows, 3000, 1, 23, record=True)                # step 23 alone, after six more steps of training
    other = b.run(rows, 3000, 6, 20, record=True)
    for x, y, z in ((long_.indices, one.indices, other.indices), (long_.noise, one.noise, other.noise), (long_.caps, one.caps, other.caps)):
        assert torch.equal(x[3], y[0])
        assert not torch.equal(x[3], z[3]) and not torch.equal(x, z)


# ---- status words -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('bad', [-1, 'n_valid'])
def test_given_index_outside_the_rows_sets_the_index_status(bad):
    from serl_b200 import _native
    n = 1000
    f = fused(td3_args())
    rows = synthetic_rows(n, seed=6).to(DEV)
    given = torch.as_tensor(np.stack([np.random.RandomState(k).permutation(n)[:86] for k in range(3)]), dtype=torch.int32, device=DEV)
    given[1, 5] = -1 if bad == -1 else n
    s0, steps = f.state.clone(), (f.critic_steps, f.actor_steps)
    r = f.run(rows, n, 3, 1, indices=given)
    assert int(r.status.item()) == _native.TD3_STATUS_INDEX
    with pytest.raises(_native.NativeError, match='outside'):
        r.check()
    got, s_bad = r.losses.clone(), f.state.clone()
    f.state.copy_(s0)
    f.critic_steps, f.actor_steps = steps
    given[1, 5] = 0
    r0 = f.run(rows, n, 3, 1, indices=given)
    r0.check()
    assert torch.equal(got.nan_to_num(7.0), r0.losses.nan_to_num(7.0)) and torch.equal(s_bad, f.state)


def test_nan_reward_sets_the_nonfinite_status():
    from serl_b200 import _native
    n = 1000
    f = fused(td3_args(hidden=32, num_layers=1))                # throwaway: its weights end up NaN
    rows = synthetic_rows(n, seed=6)
    rows[17, 17] = float('nan')
    given = torch.arange(86, dtype=torch.int32, device=DEV).reshape(1, 86)
    r = f.run(rows.to(DEV), n, 1, 1, indices=given)
    assert int(r.status.item()) == _native.STATUS_NONFINITE and torch.isnan(r.losses[0, 0])
    with pytest.raises(_native.NativeError, match='NaN'):
        r.check()
