"""K6 (csrc/smoothness.cu, serl_smoothness) without a GPU: the horizon limits of its two paths pinned against the source,
the C-ABI's refusals before any CUDA call, and the host calc_smoothness (base/core/utils.py:82-120) held to a plain
O(N^2) float64 DFT at the small lengths where the bin count is 0 or 1.  tests/test_k6_domain_gpu.py relies on all three."""
import ctypes
import math
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, 'serl_b200', 'csrc', 'smoothness.cu')

# Bluestein FFT of size FM = 4096: the circular convolution needs 2 * horizon - 1 <= FM
FFT_MAX_HORIZON = 2048
# direct DFT: twiddles (float2) + three fp32 channels = 20 bytes per step in at most 200 KB of shared memory
DIRECT_MAX_HORIZON = 10240
ERR_ARG, ERR_UNSUPPORTED = -1, -3           # SERL_ERR_ARG, SERL_ERR_UNSUPPORTED (include/serl_b200.h)


def test_path_limits_match_the_source():
    src = open(SRC).read()
    fm = int(re.search(r'^#define FM (\d+)$', src, re.M).group(1))
    assert 'if (2 * horizon - 1 <= FM) {' in src
    assert (fm + 1) // 2 == FFT_MAX_HORIZON
    per_step = re.search(r'const size_t smem = \(size_t\)horizon \* \((\d+) \+ (\d+)\);', src)
    cap = re.search(r'if \(smem > (\d+) \* 1024\) return serl_fail\(SERL_ERR_UNSUPPORTED', src)
    assert per_step and cap
    assert int(cap.group(1)) * 1024 // (int(per_step.group(1)) + int(per_step.group(2))) == DIRECT_MAX_HORIZON


def test_refusals_launch_nothing():
    """null pointers, n_traj <= 0, horizon <= 0: SERL_ERR_ARG; a horizon past the direct DFT's shared memory:
    SERL_ERR_UNSUPPORTED.  The (fake, non-null) device pointers are never read and no kernel is launched."""
    from serl_b200 import build, _native
    build.build()
    L = _native.lib()
    fake = ctypes.c_void_p(256)
    ok = dict(d_actions=fake, d_steps=fake, n_traj=4, horizon=2001, dt=0.01, d_out=fake)
    cases = [(dict(d_actions=None), ERR_ARG), (dict(d_steps=None), ERR_ARG), (dict(d_out=None), ERR_ARG),
             (dict(n_traj=0), ERR_ARG), (dict(n_traj=-1), ERR_ARG), (dict(horizon=0), ERR_ARG), (dict(horizon=-5), ERR_ARG),
             (dict(horizon=DIRECT_MAX_HORIZON + 1), ERR_UNSUPPORTED), (dict(horizon=1 << 20), ERR_UNSUPPORTED)]
    for kw, want in cases:
        a = dict(ok, **kw)
        launches = L.serl_launch_count()
        rc = L.serl_smoothness(a['d_actions'], a['d_steps'], a['n_traj'], a['horizon'], a['dt'], a['d_out'], None)
        msg = L.serl_last_error().decode()
        assert rc == want, (kw, rc, msg)
        assert L.serl_launch_count() == launches, kw
        assert msg.startswith('serl_smoothness'), (kw, msg)
        if want == ERR_UNSUPPORTED:
            assert 'horizon too long' in msg, msg


def plain_dft_smoothness(y, dt):
    """the metric from its definition: Y_i[k] = sum_n y_i[n] exp(-2 pi i k n / N) for k = 1 .. N/2 - 1, each bin weighted by
    f_k = dt + (k - 1) * (1/(2 dt) - dt) / (M - 1) (the kernels' form of linspace(dt, 1/(2 dt), M); f_1 = dt when M = 1)"""
    N = y.shape[0]
    M = N // 2 - 1
    if M <= 0:
        return -0.0
    fstep = (1.0 / (2.0 * dt) - dt) / (M - 1) if M > 1 else 0.0
    S = 0.0
    for k in range(1, M + 1):
        f = dt + (k - 1) * fstep
        for c in range(y.shape[1]):
            re = sum(y[n, c] * math.cos(2 * math.pi * k * n / N) for n in range(N))
            im = -sum(y[n, c] * math.sin(2 * math.pi * k * n / N) for n in range(N))
            S += f * (re * re + im * im)
    S *= dt * 2.0 / N
    return -(math.sqrt(S) * 100.0 * (80.0 / (N * dt)))


@pytest.mark.parametrize('dt', [0.01, 0.02, 0.005])
def test_calc_smoothness_matches_a_plain_dft_at_small_lengths(dt):
    from serl_b200.core.utils import calc_smoothness
    rng = np.random.RandomState(11)
    for N in range(4):                     # no bin: -0.0, as the reference returns it
        got = calc_smoothness(rng.uniform(-1, 1, (N, 3)), dt=dt)
        assert got == 0.0 and math.copysign(1.0, got) < 0, (N, got)
    for N in (4, 5, 6, 7, 16, 33):
        y = rng.uniform(-1, 1, (N, 3)) + np.array([0.3, -0.7, 0.0])
        want = plain_dft_smoothness(y, dt)
        assert want < 0
        assert calc_smoothness(y, dt=dt) == pytest.approx(want, rel=1e-12), (N, dt)
    # one bin (N = 4, 5): only k = 1 counts, with f = dt
    y = np.array([[1.0, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]])
    assert calc_smoothness(y, dt=dt) == pytest.approx(-math.sqrt(dt * 1.0 * dt * 2 / 4) * 100 * 80 / (4 * dt), rel=1e-14)
