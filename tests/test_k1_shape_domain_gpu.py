"""K1 (csrc/rollout.cu) across the whole uniform-actor domain it accepts: every hidden size 2 <= h <= 256 and depth L that
K1 keeps rather than hand to K1-TC (rollout.tc_widths is None), not only the L = 3 actors of the rest of the suite.

Genomes are random reference Actors whose LayerNorm parameters differ from layer to layer (gamma ~ U(0.5, 1.5),
beta ~ N(0, 0.1)): a kernel that read another layer's gamma or beta, or walked the genome with a wrong per-layer stride,
changes the bits.  Bars:
  - the actor's forward pass is bit-identical with the kernel-order oracle (oracle/plant/actor_kernel_order.c), and within
    4x the float32 torch forward pass's own distance from float64 (catches a bug the two share);
  - closed loop: identical termination steps, returns within 1e-4 relative of the C episode port with the kernel-order actor;
  - the warp kernel and the one-thread-per-env kernel give identical bits;
  - shapes K1 hands on fly on K1-TC, and shapes no kernel holds are refused before any launch."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import actor as A, fast, refsig

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')
HERE = os.path.dirname(os.path.abspath(__file__))
WARP = (32, 64, 72, 96, 128)                  # the hidden sizes the warp actor is instantiated for
SIMPLE = (2, 3, 5, 7, 8, 31, 33, 50, 100, 101, 127, 129, 141)
ACTS = ('tanh', 'elu', 'relu')
REL_TOL = 1e-4
SMEM_OPTIN = 227 * 1024


def genome(hidden, num_layers, activation, seed, scale=1.0, out_gain=1.0):
    """flat genome of a random Actor with per-layer LayerNorm parameters; out_gain scales the output layer, scale the whole genome"""
    torch.manual_seed(seed)
    m = A.Actor(hidden=hidden, num_layers=num_layers, activation=activation)
    with torch.no_grad():
        for mod in m.net:
            if isinstance(mod, A.LayerNorm):
                mod.gamma.uniform_(0.5, 1.5)
                mod.beta.normal_(0.0, 0.1)
        m.net[-2].weight.mul_(out_gain)
        m.net[-2].bias.mul_(out_gain)
    return A.flatten(m) * np.float32(scale)


def k1_deepest(h):
    """the deepest L that K1 flies at hidden size h (tc_widths is None from L = 0 up to it)"""
    from serl_b200 import rollout
    keeps = lambda L: rollout.tc_widths(rollout.actor_shape(h, L)) is None
    lo, hi = 0, 1
    while keeps(hi):
        lo, hi = hi, hi * 2
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if keeps(mid) else (lo, mid)
    return lo


def forward_deepest(h):
    """the deepest L serl_actor_forward holds at hidden size h: the warp kernel needs the genome and the exchange buffers of
    4 warps (h/4 x 32 floats each) in shared memory, the one-thread-per-env kernel the genome and 2 x h x 128 floats"""
    from serl_b200 import rollout
    p4 = lambda L: (rollout.num_params(rollout.actor_shape(h, L)) + 3) // 4 * 4 * 4
    need = (lambda L: p4(L) + 4 * (h // 4) * 32 * 4) if h in WARP else (lambda L: p4(L) + 2 * h * 128 * 4)
    L = -1
    while need(L + 1) <= SMEM_OPTIN:
        L += 1
    return L


def observations(seed):
    """3301 rows (not a multiple of 128): flight-like, N(0, 1), x30 (saturating) and a zero row"""
    rs = np.random.RandomState(seed)
    return np.concatenate([rs.randn(2000, 7) * [0.05, 0.05, 0.01, 0.02, 0.02, 0.02, 0.05], rs.randn(1000, 7), rs.randn(300, 7) * 30.0,
                           np.zeros((1, 7))]).astype(np.float32)


def refs(n, seed):
    lv, st = refsig.make_ref_params(n, seed_base=seed)
    return lv, st, torch.as_tensor(lv, device=DEV), torch.as_tensor(st, device=DEV)


def modes_tensor(modes):
    from serl_b200 import rollout
    return torch.as_tensor(np.array([rollout.mode_code(m) for m in modes], dtype=np.int32), device=DEV)


def fly(w, h, L, activation, modes, seed, horizon):
    """population_rollout of genomes w [pop, P] (numpy) through K1 -> (returns, steps) and the kernel-order oracle's"""
    from serl_b200 import rollout
    sh = rollout.actor_shape(h, L, activation)
    assert rollout.tc_widths(sh) is None, (h, L)
    lv, st, dlv, dst = refs(len(modes), seed)
    r = rollout.population_rollout(torch.as_tensor(w, device=DEV), sh, dlv, dst, modes_tensor(modes), horizon=horizon)
    torch.cuda.synchronize()
    r.check()
    oret, ostp = fast.evaluate_population(w, h, lv, st, modes, num_layers=L, activation=activation, horizon=horizon, actor_order='kernel')
    return r.returns.cpu().numpy(), r.steps.cpu().numpy(), oret, ostp


def strict(ret, stp, oret, ostp, what):
    assert np.array_equal(stp, ostp), (what, stp, ostp)
    rel = np.abs(ret - oret) / np.abs(oret)
    assert rel.max() <= REL_TOL, (what, rel.max())


# ---- a. the forward pass, bit for bit, at every depth the kernels hold -------------------------------------------------
def _forward_case(h, L, activation, scale):
    from serl_b200 import rollout
    L = {'k1': k1_deepest(h), 'fwd': forward_deepest(h)}.get(L, L)
    sh = rollout.actor_shape(h, L, activation)
    g = genome(h, L, activation, 1000 * h + L, scale=scale)
    obs = observations(h + L)
    for o in (obs[:1], obs):
        got = rollout.actor_forward(torch.as_tensor(g, device=DEV), sh, torch.as_tensor(o, device=DEV)).cpu().numpy()
        want = fast.actor_forward_kernel_order(g, o, h, L, activation)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (h, L, activation, o.shape[0], np.abs(got - want).max())
    with torch.no_grad():
        net = A.unflatten(g, hidden=h, num_layers=L, activation=activation)
        ref32 = net(torch.as_tensor(obs)).numpy()
        ref64 = net.double()(torch.as_tensor(obs, dtype=torch.float64)).numpy()
    err, base = np.abs(got - ref64).max(), np.abs(ref32 - ref64).max()
    assert err <= max(4 * base, 5e-6), (h, L, activation, err, base)


@pytest.mark.parametrize('h,L', [(h, L) for h in WARP for L in (0, 1, 2, 4, 'k1', 'fwd') if not (h == 128 and L == 4)] +
                         [(h, L) for h in SIMPLE for L in (0, 1, 'k1')] + [(200, 0)])
def test_forward_is_bit_exact_with_the_kernel_order_oracle_at_every_depth(h, L):
    """tanh, and the same genome x3 to drive the activations into saturation; L = 'k1': the deepest L the rollout keeps,
    'fwd': the deepest the forward kernel holds"""
    _forward_case(h, L, 'tanh', 1.0)
    _forward_case(h, L, 'tanh', 3.0)


@pytest.mark.parametrize('activation', ['elu', 'relu'])
@pytest.mark.parametrize('h,L', [(32, 'k1'), (64, 2), (72, 4), (96, 'k1'), (128, 'k1'), (3, 1), (50, 'k1'), (141, 1)])
def test_forward_other_activations_at_every_depth(h, L, activation):
    _forward_case(h, L, activation, 1.0)


# ---- b. every shape K1 claims, on a short horizon ---------------------------------------------------------------------
def _short_flights(h, depths):
    for L in depths:
        act = ACTS[L % 3]
        w = np.stack([genome(h, L, act, 7 * h + L + k, out_gain=0.3) for k in range(2)])
        ret, stp, oret, ostp = fly(w, h, L, act, ['nominal', 'be', 'ice', 'cg', 'sa'], 300 + L, 60)
        strict(ret, stp, oret, ostp, (h, L, act))


@pytest.mark.parametrize('h', WARP)
def test_every_depth_k1_keeps_flies_at_a_warp_size(h):
    """L = 0 up to the deepest L that tc_widths leaves to K1: past the warp kernel's limit, the one-thread-per-env kernel"""
    _short_flights(h, range(k1_deepest(h) + 1))


@pytest.mark.parametrize('h', SIMPLE + (142, 200))
def test_sampled_depths_k1_keeps_fly_at_other_sizes(h):
    d = k1_deepest(h)
    _short_flights(h, sorted({0, min(1, d), d // 2, d}))


# ---- c. the closed loop at full horizon ----------------------------------------------------------------------------------
@pytest.mark.parametrize('h,L', [(h, L) for h in WARP for L in (1, 2, 'k1')] + [(3, 1), (33, 1), (127, 1), (141, 1)])
def test_strict_parity_at_full_horizon(h, L):
    """h = 128: L = 2 keeps the plant tables in shared memory, L = 3 reads them from global memory"""
    L = k1_deepest(h) if L == 'k1' else L
    # gentle output gains fly most episodes to the end, the larger ones end some early
    w = np.stack([genome(h, L, 'tanh', 50 * h + L + k, out_gain=g) for k, g in enumerate((0.2, 0.3, 1.0, 3.0))])
    ret, stp, oret, ostp = fly(w, h, L, 'tanh', ['nominal', 'se', 'ice', 'cg'], 700 + h, 2001)
    strict(ret, stp, oret, ostp, (h, L))
    assert (stp == 2001).any() and (stp < 2001).any(), stp          # full episodes and early terminations


# ---- d. the warp kernel and the one-thread-per-env kernel give the same bits --------------------------------------------
BOTH_KERNELS = [(h, L) for h in (32, 64, 72) for L in (0, 1, 2, 4)] + [(96, 0), (96, 1), (96, 2), (128, 0), (128, 1)]


def run_both_kernel_shapes(path):
    """(in a subprocess whose SERL_ROLLOUT_IMPL picks the kernel) rollouts and forward passes at BOTH_KERNELS into `path`"""
    from serl_b200 import rollout
    out = {}
    modes = ['nominal', 'be', 'ice', 'cg', 'jr']
    _, _, dlv, dst = refs(len(modes), 41)
    obs = torch.as_tensor(observations(3), device=DEV)
    for h, L in BOTH_KERNELS:
        act = ACTS[(h + L) % 3]
        sh = rollout.actor_shape(h, L, act)
        assert rollout.tc_widths(sh) is None, (h, L)
        w = torch.as_tensor(np.stack([genome(h, L, act, 11 * h + L + k, out_gain=0.3) for k in range(3)]), device=DEV)
        r = rollout.population_rollout(w, sh, dlv, dst, modes_tensor(modes), horizon=400)
        a = rollout.actor_forward(w[0].contiguous(), sh, obs)
        torch.cuda.synchronize()
        r.check()
        out['%d_%d' % (h, L)] = [r.returns.cpu().numpy().view(np.uint64).tolist(), r.steps.cpu().tolist(),
                                 a.cpu().numpy().view(np.uint32).tolist()]
    with open(path, 'w') as f:
        json.dump(out, f)


def test_warp_and_simple_kernels_give_identical_bits(tmp_path):
    """SERL_ROLLOUT_IMPL=simple is read once per process, so each kernel flies in its own"""
    outs = []
    for impl in ('gemm', 'simple'):
        path = str(tmp_path / ('%s.json' % impl))
        code = ('import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_k1_shape_domain_gpu as T; '
                'T.run_both_kernel_shapes(%r)') % (os.path.dirname(HERE), HERE, path)
        p = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, env=dict(os.environ, SERL_ROLLOUT_IMPL=impl),
                           timeout=900)
        assert p.returncode == 0, p.stderr
        with open(path) as f:
            outs.append(json.load(f))
    for h, L in BOTH_KERNELS:
        k = '%d_%d' % (h, L)
        warp, simple = outs[0][k], outs[1][k]
        assert warp[1] == simple[1], (h, L, 'steps')
        assert warp[0] == simple[0], (h, L, 'returns')
        assert warp[2] == simple[2], (h, L, 'actions')


# ---- e. what K1 hands on -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('h,L', [(96, 5), (72, 8)])
def test_shapes_past_the_warp_kernel_fly_on_k1_tc(h, L):
    """K7 trains these shapes; their genome fits next to the exchange buffers but not next to the plant tables"""
    from serl_b200 import rollout
    sh = rollout.actor_shape(h, L, 'tanh')
    widths = rollout.tc_widths(sh)
    assert widths == [h] * (L + 1)
    w = np.stack([genome(h, L, 'tanh', 90 + k, out_gain=0.2) for k in range(3)])
    modes = ['nominal', 'ice', 'be', 'cg', 'sa', 'jr']
    lv, st, dlv, dst = refs(len(modes), 505)
    r = rollout.population_rollout(torch.as_tensor(w, device=DEV), sh, dlv, dst, modes_tensor(modes), horizon=600)
    torch.cuda.synchronize()
    r.check()
    oret, ostp = fast.evaluate_population_wide(w, widths, lv, st, modes, horizon=600)
    strict(r.returns.cpu().numpy(), r.steps.cpu().numpy(), oret, ostp, (h, L))


def test_shapes_no_kernel_holds_are_refused_before_any_launch():
    from serl_b200 import _native, rollout
    lib = _native.lib()
    modes = ['nominal', 'ice']
    _, _, dlv, dst = refs(len(modes), 3)
    for h, L in ((64, 10), (256, 0), (32, 45)):        # [64] * 11 and [32] * 46: more widths than K1-TC takes
        sh = rollout.actor_shape(h, L)
        w = torch.zeros((2, rollout.num_params(sh)), dtype=torch.float32, device=DEV)
        torch.cuda.synchronize()
        before = lib.serl_launch_count()
        with pytest.raises(_native.NativeError, match=r'\(-3\)'):
            rollout.population_rollout(w, sh, dlv, dst, modes_tensor(modes), horizon=50)
        assert lib.serl_launch_count() == before, (h, L)
    obs = torch.zeros((5, 7), dtype=torch.float32, device=DEV)
    for h, L in ((96, 6), (64, 13), (32, 51), (128, 4), (256, 0)):    # one layer past forward_deepest
        assert L == forward_deepest(h) + 1
        sh = rollout.actor_shape(h, L)
        g = torch.zeros(rollout.num_params(sh), dtype=torch.float32, device=DEV)
        before = lib.serl_launch_count()
        with pytest.raises(_native.NativeError, match=r'\(-3\)'):
            rollout.actor_forward(g, sh, obs)
        assert lib.serl_launch_count() == before, (h, L)
