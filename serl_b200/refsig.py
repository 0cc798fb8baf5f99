"""Reference-signal parameter generator (host side of the product; oracle/refsig.py is the checker's own copy).

The reference builds its tracking references with the third-party package `signals==0.0.1`
(envs/phlabenv.py:303-345: RandomizedCosineStepSequence(t_max=20, ampl_max=30|20, block_width=4,
smooth_width=3, n_levels=10, vary_timings=0.04) + Const(theta_trim)), whose source is not in the reference
tree -> PARITY UNPINNED for its RNG stream.  The shape below is the one recovered from the 15 logged episodes
(cols 0-2 of logs/wandb/*/files/*statehistory*.txt): 4 s blocks, first level 0, levels on
linspace(-A, A, 10), raised-cosine transitions of width 3 s that start at 4k +- 0.04 s.
The rollout kernel evaluates the signal on device from the arrays returned here (csrc/rollout.cu: ref_deg).
"""
import numpy as np

N_BLOCKS = 6          # block k starts at ~4k s; k = 5 starts at ~20 s (only reachable by jitter)
BLOCK_W = 4.0
SMOOTH_W = 3.0
JITTER = 0.04
N_LEVELS = 10
AMPL = (30.0, 20.0)   # theta, phi [deg]


def widths(t_max=20, symmetric=False):
    """(block width, smooth width, timing jitter) of init_ref (envs/phlabenv.py:321-335) for an episode of t_max seconds.
    symmetric=True: the theta-only reference of symmetric control (:304-313), smooth width t_max // 6.7 (2 s at 20 s, 11 s at
    80 s) and jitter t_max // 500, a floor division that is 0 for any episode shorter than 500 s."""
    if symmetric:
        return float(t_max // 5), float(t_max // 6.7), float(t_max // 500)
    return float(t_max // 5), float(t_max // 6), t_max / 500.


def make_ref_params(n_envs, seed_base=7_000_000, t_max=20, symmetric=False):
    """levels[n_envs, 2, N_BLOCKS] (deg, without the theta trim offset), starts[n_envs, 2, N_BLOCKS] (s).
    symmetric=True draws the theta channel alone (symmetric control's parameters); the phi channel stays zero."""
    block_w, _, jitter = widths(t_max, symmetric)
    levels = np.zeros((n_envs, 2, N_BLOCKS))
    starts = np.zeros((n_envs, 2, N_BLOCKS))
    for e in range(n_envs):
        rs = np.random.RandomState(seed_base + e)
        for c in range(1 if symmetric else 2):
            grid = np.linspace(-AMPL[c], AMPL[c], N_LEVELS)
            lv = grid[rs.randint(0, N_LEVELS, size=N_BLOCKS)]
            lv[0] = 0.0
            st = block_w * np.arange(N_BLOCKS) + rs.uniform(-jitter, jitter, size=N_BLOCKS)
            st[0] = 0.0
            levels[e, c] = lv
            starts[e, c] = st
    return levels, starts


def ref_value_deg(levels, starts, t, offset=0.0, smooth_w=SMOOTH_W, t_end=None):
    """value [deg] of one channel at time t. levels/starts: [N_BLOCKS].  `offset` is the reference's
    `+ signals.Const(0., t_max, theta_trim)` (envs/phlabenv.py:344): a constant that exists on [0, t_max] only — the last
    row of every logged episode (t = 20.01 s) shows the step sequence without it, and so does the final step of an
    episode, whose accumulated time is 20.000000000000327 s."""
    if t_end is not None and t > t_end:
        offset = 0.0
    k = 0
    for j in range(1, N_BLOCKS):
        if t >= starts[j]:
            k = j
    if k == 0:
        return offset + levels[0]
    x = (t - starts[k]) / smooth_w
    if x >= 1.0:
        return offset + levels[k]
    return offset + (levels[k - 1] + (levels[k] - levels[k - 1]) * (0.5 * (1.0 - np.cos(np.pi * x))))
