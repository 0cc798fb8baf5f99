"""Record what the reference's own plant binaries compute, for the tests that compare against them: run once where the
binaries exist (oracle/build.py copies them to oracle/_ref), output tests/golden/refbin_kat.npz.

  plant_<key>          the binary's 12 outputs at every SAMPLE-th step of two logged episodes replayed through it (h2000_v90)
  variant_<v>          the outputs at every SAMPLE-th of 300 steps of seeded random commands (ice, cg, h2000_v150)
  timed_<b>_X0/_X1     the binary's state before / after each native call of the gust-pulse windows (gust, test builds)
  lookup_index / lookup2d / lookup1d   the binary's rt_GetLookupIndex / rt_Lookup2D_Normal / rt_Lookup on the probes of
                       tests/test_lifter_reference.py, in the order the test makes them
  env_<m>_rows/_x/...  one closed-loop episode of the oracle env on the binary (cg_timed 40 s, gust 30 s): a sample of the
                       live state rows (every 25th step and both edges of the pulse / trigger), return and length
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from oracle import build as obuild, phlab, plant as P, refsig  # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'refbin_kat.npz')
SAMPLE = 10                 # stored rows: every SAMPLE-th step (the file stays small; every row is still compared)
LIVE = [0, 1, 2, 3, 4, 5, 6, 7, 9]
TIMED_WINDOW = [k for k in range(2306) if 1996 <= k <= 2003 or 2296 <= k <= 2303 or k == 2150]


def replay(pl, a):
    X = pl.initial_state()
    _, X = pl.step(X, np.zeros(10))
    outs = []
    for k in range(a.shape[0]):
        cmd = np.zeros(10)
        cmd[:3] = a[k, 3:6]
        out, X = pl.step(X, cmd)
        outs.append(out)
    return np.array(outs)


def env_rows(k):
    return sorted(set(range(0, k + 1, 25)) | set(range(1990, min(2010, k + 1))) | set(range(2290, min(2310, k + 1))))


def main():
    obuild.build()
    assert obuild.have_ref(), 'the reference binaries are not under oracle/_ref'
    out = {}
    traj = np.load(os.path.join(ROOT, 'tests', 'golden', 'plant_traj_kat.npz'))
    for key in ['ERL10_rl_statehistory_episode209', 'l_TD3_rl_statehistory_episode575']:
        out['plant_' + key] = replay(P.RefPlant('h2000_v90'), traj[key])[::SAMPLE]
    for v in ['ice', 'cg', 'h2000_v150']:
        b = P.RefPlant(v)
        X = b.initial_state()
        rng = np.random.RandomState(1)
        outs = []
        for k in range(300):
            cmd = np.zeros(10)
            cmd[:3] = 0.05 * rng.uniform(-1, 1, 3)
            o, X = b.step(X, cmd)
            outs.append(o)
        out['variant_' + v] = np.array(outs)[::SAMPLE]
    for build in ['gust', 'test']:
        pl = P.RefPlant(build)
        X = pl.initial_state()
        x0, x1 = [], []
        for k in range(2306):
            cmd = 0.02 * np.sin(0.01 * k + np.arange(3))
            if k in TIMED_WINDOW:
                x0.append(X.copy())
            _, X = pl.step(X, np.concatenate([cmd, np.zeros(7)]))
            if k in TIMED_WINDOW:
                x1.append(X.copy())
        out['timed_%s_X0' % build], out['timed_%s_X1' % build] = np.array(x0), np.array(x1)
    from test_eval_suite_gpu import ACT, KOActor
    g = ACT['serl10_elite_h72_tanh']
    for mode, seed, t_max, sw in [('cg-timed', 40, 40, 6.0), ('gust', 41, 30, 4.5)]:
        lv, st = refsig.make_ref_params(1, seed_base=seed, t_max=t_max)
        env = phlab.CitationEnv(mode, 'ref', t_max=t_max)
        env.smooth_w = sw
        obs = env.reset(lv[0], st[0])
        tot, xs = 0.0, []
        for k in range(100 * t_max + 1):
            obs, rew, done, _ = env.step(KOActor(g).select_action(obs))
            xs.append(env.x.copy())
            tot += rew
            if done:
                break
        rows = env_rows(k)
        name = mode.replace('-', '_')
        out['env_%s_rows' % name] = np.array(rows, dtype=np.int16)
        out['env_%s_x' % name] = np.asarray(xs)[rows][:, LIVE]
        out['env_%s_return' % name] = np.array(tot)
        out['env_%s_steps' % name] = np.array(k + 1)
    import test_lifter_reference as TL
    L = TL.load_binary_lookups(os.path.join(obuild.HERE, '_ref', 'citation_h2000_v90.so'))
    out['lookup_index'] = np.array([r for _, _, r in TL.index_cases(L)], dtype=np.int8)
    both = list(TL.formula_cases(L))
    out['lookup2d'] = np.array([b[0] for b in both])
    out['lookup1d'] = np.array([b[1] for b in both])
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
