"""Run the REFERENCE SSNE (base/core/mod_neuro_evo.py, imported from /root/reference) with the exclusive-index shim of
make_golden_ea.py over the actor shapes, populations and operator settings the engine evolves, on seeded genomes with
planted edge values (tests/ssne_domain_cases.py), and record what one epoch computed. Runs only where the reference tree
exists; output tests/golden/ssne_domain_kat.npz (data only). Regenerating reproduces the file byte for byte.

Per case <name>_*: seed, shape, pop, planted, elite_fraction, mutation_prob, mutation_mag, fitness (pairwise distinct),
elite, written (per row, how many elements the point mutations wrote) and either `after` (whole genomes) or, for large
populations x P, per-row SHA-256 `digest`s of `after` plus `after` at the seeded columns `cols` (`sample`). Digests are
taken over the bits with NaNs at written elements made canonical (the comparison rule of ssne_domain_cases.py).
"""
import io
import os
import random
import sys
import tempfile
import types
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests')]
sys.path.insert(0, '/root/reference/base')
os.chdir(tempfile.mkdtemp())                     # the reference's Parameters writes ./tmp/
from core import mod_neuro_evo as ne, genetic_agent          # noqa: E402
from parameters import Parameters                             # noqa: E402
import ssne_domain_cases as D                                 # noqa: E402

IDX_LINES = {51, 76, 79, 89, 92, 357, 358, 517}
FULL_LIMIT = 40000          # pop * P up to which the whole `after` is stored
DEFAULT_MAG = 0.0247682869654


class Shim:
    def __getattr__(self, k):
        return getattr(random, k)

    def randint(self, a, b):
        if sys._getframe(1).f_lineno in IDX_LINES:
            return random.randrange(a, b)
        return random.randint(a, b)


ne.random = Shim()
WRITTEN = []                                     # data_ptr of every element regularize_weight clamps (one per point mutation)
_regularize = ne.SSNE.regularize_weight


def _recording_regularize(self, weight, mag):
    WRITTEN.append(weight.data_ptr())
    return _regularize(self, weight, mag)


ne.SSNE.regularize_weight = _recording_regularize


def cases():
    """(seed, pop, shape, planted, elite_fraction, mutation_prob, mutation_mag, fitness kind)"""
    shapes = [(7, 3, h, L) for L in (1, 2, 3, 4, 8) for h in (8, 72, 257)]
    shapes += [(10, 3, h, 3) for h in (8, 72, 257)] + [(2, 1, h, 3) for h in (8, 72, 257)] + [(7, 3, 320, 1), (7, 3, 264, 2)]
    out = []
    for k, shape in enumerate(shapes):
        P = D.param_table(*shape)[1]
        pops = [2, 3, 4, 5, 6, 8] if P > 200000 else [3, 5, 8, 12, 17] if P > 20000 else [2, 6, 10, 16, 24, 33, 64]
        out.append((100 + k, pops[k % len(pops)], shape, k % 4 != 3, (0.2, 0.5)[k % 2], (0.9, 1.0)[(k // 2) % 2],
                    (DEFAULT_MAG, 0.01, 0.2)[(k + k // 3) % 3], 'distinct'))
    # small populations at elite fraction 0.5 (unselects run out: the elitism takes from the offsprings), the fitness
    # edge case, and more populations at the small shapes
    for k, (pop, shape, ef) in enumerate([(2, (7, 3, 8, 1), 0.5), (3, (7, 3, 8, 2), 0.5), (4, (2, 1, 8, 3), 0.5),
                                          (5, (10, 3, 8, 3), 0.5), (6, (7, 3, 8, 3), 0.5), (7, (7, 3, 72, 1), 0.5),
                                          (40, (7, 3, 8, 3), 0.2), (64, (2, 1, 8, 3), 0.2), (48, (7, 3, 8, 1), 0.5)]):
        out.append((200 + k, pop, shape, k % 2 == 0, ef, (1.0, 0.9)[k % 2], (0.2, DEFAULT_MAG, 0.01)[k % 3],
                    'nan_ninf' if k == 6 else 'distinct'))
    return out


def fitness(seed, pop, kind):
    fit = np.random.RandomState(seed + 777).uniform(-3000, -50, pop)
    if kind == 'nan_ninf':
        fit[1], fit[pop // 2] = np.nan, -np.inf
    assert len(np.unique(fit[np.isfinite(fit)])) == np.isfinite(fit).sum()       # no ties: the reference sorts unstably
    return fit


def run_case(seed, pop, shape, planted, ef, mprob, mag, fkind):
    cla = types.SimpleNamespace(disable_cuda=True, env='phlab_attitude_nominal', seed=7, pop_size=pop, mut_type='normal')
    args = Parameters(cla)
    args.state_dim, args.action_dim, args.hidden_size, args.num_layers = shape
    args.distil_crossover = False
    args.elite_fraction, args.mutation_prob, args.mutation_mag = ef, mprob, mag
    table, P = D.param_table(*shape)
    torch.manual_seed(seed)
    agents = [genetic_agent.GeneticAgent(args) for _ in range(pop)]
    before = D.genomes(seed, pop, shape, planted)
    where = []                                    # (first byte, last byte, actor, genome offset) of every parameter
    for a, g in enumerate(agents):
        params = list(g.actor.parameters())
        assert len(params) == len(table)
        for p, (off, r, c) in zip(params, table):
            assert p.numel() == r * max(c, 1)
            p.data.copy_(torch.from_numpy(before[a, off:off + p.numel()].reshape(p.shape)))
            where.append((p.data_ptr(), p.data_ptr() + 4 * p.numel(), a, off))
    flat = lambda: np.stack([torch.cat([p.data.reshape(-1) for p in g.actor.parameters()]).numpy().copy() for g in agents])
    assert np.array_equal(flat().view(np.uint32), before.view(np.uint32))
    fit = fitness(seed, pop, fkind)
    ev = ne.SSNE(args, None, None)
    WRITTEN.clear()
    np.random.seed(seed + 1); random.seed(seed + 2)
    elite = ev.epoch(agents, fit)
    after = flat()
    written = np.zeros((pop, P), bool)
    for ptr in WRITTEN:
        lo, hi, a, off = next(w for w in where if w[0] <= ptr < w[1])
        written[a, off + (ptr - lo) // 4] = True
    c = dict(seed=np.int64(seed), shape=np.array(shape, np.int64), pop=np.int64(pop), planted=np.bool_(planted),
             elite_fraction=np.float64(ef), mutation_prob=np.float64(mprob), mutation_mag=np.float64(mag), fitness=fit,
             elite=np.int64(elite), written=written.sum(1).astype(np.int64))
    if pop * P <= FULL_LIMIT:
        c['after'] = after
    else:
        cols = D.sample_cols(seed, P)
        c['cols'], c['sample'], c['digest'] = cols, after[:, cols].copy(), D.row_digests(after, written)
    return c


def save(path, arrays):
    """np.savez_compressed with fixed zip timestamps, so that regenerating reproduces the file byte for byte"""
    with zipfile.ZipFile(path, 'w', compression=zipfile.ZIP_DEFLATED) as z:
        for name in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[name]), allow_pickle=False)
            info = zipfile.ZipInfo(name + '.npy', date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


if __name__ == '__main__':
    out = {}
    for k, case in enumerate(cases()):
        c = run_case(*case)
        for name, v in c.items():
            out['d%02d_%s' % (k, name)] = v
        print(k, case[:7], 'elite', int(c['elite']), 'written', int(c['written'].sum()), 'full' if 'after' in c else 'digest')
    save(os.path.join(HERE, 'ssne_domain_kat.npz'), out)
