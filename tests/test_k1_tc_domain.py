"""K1-TC (csrc/rollout_tc.cu) across the whole width-list domain it accepts, without a GPU: the float64 reference forward
pass the GPU tests hold the kernel to, the width-list grid they fly, and tc_prepare's envelope (2 to 9 widths,
8 <= w0 <= 1024, 8 <= w_i <= 320, shared memory) pinned at every boundary before any CUDA call.

Genomes are random WideActors whose LayerNorm parameters differ from layer to layer (gamma ~ U(0.5, 1.5), beta ~ N(0, 0.1)):
a kernel that read another layer's gamma or beta, or stepped through the small block with a wrong per-layer offset, changes
the actions."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import actor as A

ACTS = ('tanh', 'elu', 'relu')
W0S = (8, 9, 63, 65, 320, 321, 640, 1024)
# hidden widths w_i (i >= 1): residues of the padding to 8 (K-slabs) and to 64 (accumulator columns)
WIS = (8, 9, 15, 63, 64, 65, 127, 129, 257, 319, 320)
WLAST = (8, 320)
# hidden widths before the last layer: a deep list's activation buffer holds at most EDGE_UNIFORM[3] columns
MID = tuple(w for w in WIS if w <= 257)
# the shared-memory edge: n_widths -> the largest accepted uniform width [w] * n_widths (the next width up is refused)
EDGE_UNIFORM = {2: 320, 3: 264, 4: 264, 5: 264, 6: 264, 7: 264, 8: 264, 9: 264}
EDGE_1024_W = 256          # [1024, w]: the largest accepted w
EDGE_1024_WW = 264         # [1024, w, w]
EDGE_W0_320 = 856          # [w0, 320]: the largest accepted w0 (two widths keep both small blocks in shared memory)


def genome(widths, activation, seed, scale=1.0, out_gain=1.0):
    """flat genome (parameters() order) of a random WideActor with per-layer LayerNorm parameters; out_gain scales the output
    layer, scale the whole genome"""
    torch.manual_seed(seed)
    m = A.WideActor(widths, activation=activation)
    with torch.no_grad():
        for mod in m.net:
            if isinstance(mod, A.LayerNorm):
                mod.gamma.uniform_(0.5, 1.5)
                mod.beta.normal_(0.0, 0.1)
        m.net[-2].weight.mul_(out_gain)
        m.net[-2].bias.mul_(out_gain)
    return A.flatten(m) * np.float32(scale)


def _act64(name, x):
    if name == 'tanh':
        return np.tanh(x)
    if name == 'elu':
        return np.where(x > 0, x, np.expm1(np.minimum(x, 0.0)))
    return np.where(x >= 0, x, 0.01 * x)                     # LeakyReLU, the reference's 'relu'


def forward64(g, widths, activation, obs):
    """the actor's forward pass in float64, read straight from the flat genome: Linear(7, w0), act, per layer
    Linear(w_{l-1}, w_l), LayerNorm (unbiased std, eps added to the std), act, then Linear(w_last, 3), tanh"""
    g = np.asarray(g, dtype=np.float64)
    x = np.asarray(obs, dtype=np.float64)
    off = 0

    def take(*shape):
        nonlocal off
        n = int(np.prod(shape))
        v = g[off:off + n].reshape(shape)
        off += n
        return v
    W, b = take(widths[0], 7), take(widths[0])
    x = _act64(activation, x @ W.T + b)
    for a, c in zip(widths[:-1], widths[1:]):
        W, b, gamma, beta = take(c, a), take(c), take(c), take(c)
        y = x @ W.T + b
        mean = y.mean(-1, keepdims=True)
        std = np.sqrt(((y - mean) ** 2).sum(-1, keepdims=True) / (c - 1))
        x = _act64(activation, gamma * (y - mean) / (std + 1e-6) + beta)
    W, b = take(3, widths[-1]), take(3)
    assert off == g.size
    return np.tanh(x @ W.T + b)


def _tf32(x):
    """round float32 to TF32 (10-bit mantissa), ties away: rn_tf32 of csrc/rollout_tc.cu"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def _to_f32(x, truncate):
    """x (float64) to the nearest float32, or to the float32 next to it toward zero"""
    f = x.astype(np.float32)
    if truncate:
        over = np.abs(f.astype(np.float64)) > np.abs(x)
        f[over] = np.nextafter(f[over], np.float32(0))
    return f.astype(np.float64)


def forward_3xtf32(g, widths, activation, obs, truncate=True):
    """a model of K1-TC's arithmetic: every tensor-core layer splits its float32 input and weights into TF32 hi + lo parts,
    and each MMA (8 K values of one of the products hi.hi, hi.lo, lo.hi, in the kernel's order) adds exactly into a float32
    accumulator that is rounded once, toward zero when `truncate` (the tensor cores' fp32 accumulation), else to nearest.
    Everything else is float64, with the activations rounded to float32 where the kernel stores them."""
    g = np.asarray(g, dtype=np.float64)
    off = 0

    def take(*shape):
        nonlocal off
        n = int(np.prod(shape))
        v = g[off:off + n].reshape(shape)
        off += n
        return v
    W, b = take(widths[0], 7), take(widths[0])
    x = _act64(activation, np.asarray(obs, dtype=np.float64) @ W.T + b).astype(np.float32)
    for a, c in zip(widths[:-1], widths[1:]):
        W, b, gamma, beta = take(c, a), take(c), take(c), take(c)
        wh = _tf32(W.astype(np.float32))
        wl = _tf32(W.astype(np.float32) - wh)
        xh = _tf32(x)
        xl = _tf32(x - xh)
        acc = np.zeros((x.shape[0], c))
        for s in range(0, a, 8):
            k = slice(s, s + 8)
            for p, q in ((xh, wh), (xh, wl), (xl, wh)):
                acc = _to_f32(acc + p[:, k].astype(np.float64) @ q[:, k].T.astype(np.float64), truncate)
        y = acc + b
        mean = y.mean(-1, keepdims=True)
        std = np.sqrt(((y - mean) ** 2).sum(-1, keepdims=True) / (c - 1))
        x = _act64(activation, gamma * (y - mean) / (std + 1e-6) + beta).astype(np.float32)
    W, b = take(3, widths[-1]), take(3)
    return np.tanh(x.astype(np.float64) @ W.T + b)


def width_grid():
    """(widths, activation) lists the GPU tests fly: three lists at every depth, one per activation, that walk w0 through
    W0S, the hidden widths through MID and the last width through WLAST + WIS, then a few hand-picked lists"""
    grid = []
    lasts = WLAST + WIS
    for n in range(2, 10):
        for k, act in enumerate(ACTS):
            i = 3 * n + k
            mids = [MID[(i + 5 * j) % len(MID)] for j in range(n - 2)]
            w0, last = W0S[i % len(W0S)], lasts[i % len(lasts)]
            if n == 2 and w0 == 1024:
                last = min(last, EDGE_1024_W)
            grid.append(([w0] + mids + [last], act))
    grid += [([1024, 64, 320], 'relu'), ([9, 257, 8], 'tanh'), ([640, 129, 15, 65, 8], 'elu'), ([63] + [8] * 8, 'relu'),
             ([65] * 9, 'tanh'), ([200] * 9, 'elu'), ([256] * 9, 'relu')]
    return grid


def test_the_grid_covers_the_domain():
    grid = width_grid()
    assert {len(w) for w, _ in grid} == set(range(2, 10))
    for n in range(2, 10):
        assert {a for w, a in grid if len(w) == n} == set(ACTS), n
    assert {w[0] for w, _ in grid} >= set(W0S)
    assert {x for w, _ in grid for x in w[1:]} >= set(WIS)
    assert {w[-1] for w, _ in grid} >= set(WLAST)
    # both paddings: widths already on the 8 / 64 grid, one past it and one short of it
    hid = {x for w, _ in grid for x in w[1:]}
    assert {x % 8 for x in hid} >= {0, 1, 7} and {x % 64 for x in hid} >= {0, 1, 63}
    assert len(grid) == len({(tuple(w), a) for w, a in grid})


@pytest.mark.parametrize('widths,activation', [([8, 16], 'tanh'), ([65, 9, 129], 'elu'), ([320, 257, 63, 8], 'relu'),
                                               ([9] + [15] * 8, 'tanh'), ([1024, 320], 'elu')])
def test_the_float64_reference_is_the_wide_actor(widths, activation):
    """forward64 against oracle.actor.WideActor in float64 on the same genome (per-layer LayerNorm, x3 to saturate)"""
    g = genome(widths, activation, len(widths) + widths[0], scale=3.0)
    assert g.size == A.num_params_wide(widths)
    rs = np.random.RandomState(1)
    obs = np.concatenate([rs.randn(50, 7) * 0.05, rs.randn(50, 7), rs.randn(20, 7) * 30.0, np.zeros((1, 7))])
    with torch.no_grad():
        want = A.unflatten_wide(g, widths, activation).double()(torch.as_tensor(obs)).numpy()
    got = forward64(g, widths, activation, obs)
    assert np.abs(got - want).max() <= 1e-12, np.abs(got - want).max()
    # the genome's LayerNorm parameters are not the defaults, and differ from layer to layer
    net = A.unflatten_wide(g, widths, activation)
    lns = [m for m in net.net if isinstance(m, A.LayerNorm)]
    assert all((m.gamma != 1).all() and (m.beta != 0).any() for m in lns)
    if len(lns) > 1:
        assert not torch.equal(lns[0].gamma[:8], lns[1].gamma[:8])


def test_truncating_accumulation_is_what_grows_with_the_layer_input_width():
    """The model with round-to-nearest accumulation is as close to float64 as torch's float32 forward pass; with truncation
    its error grows with the number of MMAs of a layer (3 per 8 inputs), several times float32's at w0 = 1024.  The GPU
    tests hold K1-TC to 4x the larger of the two errors."""
    rs = np.random.RandomState(2)
    obs = np.concatenate([rs.randn(200, 7) * 0.05, rs.randn(200, 7)]).astype(np.float32)
    for widths, activation, scale in (([1024, 65], 'elu', 3.0), ([64, 65, 63], 'tanh', 1.0)):
        g = genome(widths, activation, 5, scale=scale)
        ref64 = forward64(g, widths, activation, obs)
        with torch.no_grad():
            base = np.abs(A.unflatten_wide(g, widths, activation)(torch.as_tensor(obs)).numpy() - ref64).max()
        rn = np.abs(forward_3xtf32(g, widths, activation, obs, truncate=False) - ref64).max()
        rz = np.abs(forward_3xtf32(g, widths, activation, obs) - ref64).max()
        assert rn <= 2 * base, (widths, rn, base)
        assert rz <= 1e-4, (widths, rz)
        if widths[0] == 1024:
            assert rz > 4 * base, (widths, rz, base)


def _lib():
    from serl_b200 import _native, build
    build.build()
    return _native.lib()


def rollout_run(widths):
    """serl_rollout_run of a width list with fake device pointers (never dereferenced when the call is refused first)"""
    from serl_b200 import _native, rollout
    lib = _lib()
    warr = (ctypes.c_int32 * len(widths))(*widths)
    d = _native.RolloutDesc()
    fake = iter(range(0x10000, 0x100000, 0x1000))
    for f in ('d_weights', 'd_ref_levels', 'd_ref_starts', 'd_env_mode', 'd_returns', 'd_steps', 'd_fitness', 'd_status'):
        setattr(d, f, next(fake))
    d.pop, d.shape, d.n_envs, d.horizon = 4, rollout.actor_shape(72), 8, 100
    d.widths, d.n_widths = ctypes.cast(warr, ctypes.c_void_p), len(widths)
    before = lib.serl_launch_count()
    rc = lib.serl_rollout_run(ctypes.byref(d), None)
    assert lib.serl_launch_count() == before
    return rc, lib.serl_last_error().decode()


def forward_run(widths):
    """serl_actor_forward_wide with fake device pointers"""
    lib = _lib()
    warr = (ctypes.c_int32 * len(widths))(*widths)
    before = lib.serl_launch_count()
    rc = lib.serl_actor_forward_wide(0x10000, warr, len(widths), 0, 0x20000, 5, 0x30000, None)
    assert lib.serl_launch_count() == before
    return rc, lib.serl_last_error().decode()


def largest_accepted(accepts, make, lo=8, hi=1024):
    """the largest w in [lo, hi] with accepts(make(w)), given that acceptance is monotone in w and accepts(make(lo))"""
    assert accepts(make(lo))
    if accepts(make(hi)):
        return hi
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if accepts(make(mid)) else (lo, mid)
    return lo


def edge_lists():
    """(largest accepted list, the next one up) at the shared-memory edge"""
    out = [([w] * n, [w + 1] * n) for n, w in EDGE_UNIFORM.items() if n > 2]      # [320, 320] is the w_i <= 320 boundary
    return out + [([EDGE_W0_320, 320], [EDGE_W0_320 + 1, 320]), ([1024, EDGE_1024_W], [1024, EDGE_1024_W + 1]), ([1024, EDGE_1024_WW, EDGE_1024_WW], [1024, EDGE_1024_WW + 1, EDGE_1024_WW + 1])]


no_device = pytest.mark.skipif(torch.cuda.is_available(), reason='the fake pointers must not reach a device')


@no_device
@pytest.mark.parametrize('widths,activation', width_grid())
def test_every_grid_list_passes_every_check(widths, activation):
    """Without a GPU, a list that passes the checks stops at the first CUDA call (SERL_ERR_CUDA), not at SERL_ERR_UNSUPPORTED"""
    assert rollout_run(widths)[0] == -2, widths
    assert forward_run(widths)[0] == -2, widths


@no_device
def test_the_shared_memory_edge_is_where_the_table_says():
    ok = lambda ws: rollout_run(ws)[0] == -2
    for n, w in EDGE_UNIFORM.items():
        assert largest_accepted(ok, lambda x: [x] * n, hi=320) == w, n
    assert largest_accepted(ok, lambda x: [1024, x], hi=320) == EDGE_1024_W
    assert largest_accepted(ok, lambda x: [1024, x, x], hi=320) == EDGE_1024_WW
    assert largest_accepted(ok, lambda x: [x, 320]) == EDGE_W0_320
    for good, bad in edge_lists():
        assert rollout_run(good)[0] == -2 and forward_run(good)[0] == -2, good
        for run in (rollout_run, forward_run):
            rc, msg = run(bad)
            assert rc == -3 and 'shared memory' in msg, (bad, rc, msg)


@pytest.mark.parametrize('widths,what', [([1025, 64], 'w0 <= 1024'), ([1025, 64, 64], 'w0 <= 1024'), ([7, 64], 'w0 <= 1024'),
                                         ([64, 321], 'w_i <= 320'), ([64, 64, 321, 64], 'w_i <= 320'), ([64] * 8 + [321], 'w_i <= 320'),
                                         ([64, 7], 'w_i <= 320'), ([64] * 10, '2 to 9 widths'), ([8] * 10, '2 to 9 widths'),
                                         ([64], '2 to 9 widths')])
def test_each_boundary_is_refused_with_its_message_before_any_cuda_call(widths, what):
    for run in (rollout_run, forward_run):
        rc, msg = run(widths)
        assert rc == -3 and what in msg, (widths, rc, msg)


@no_device
@pytest.mark.parametrize('widths', [[1024, 64], [1024, 64, 64], [64, 320], [64, 64, 64, 320], [64] * 8 + [320], [EDGE_UNIFORM[3]] * 2 + [320], [8] * 9, [8, 8]])
def test_the_last_accepted_value_at_each_boundary_passes_every_check(widths):
    assert rollout_run(widths)[0] == -2, widths
    assert forward_run(widths)[0] == -2, widths
