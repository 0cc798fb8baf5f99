"""K2-K5 on the device across the actor shapes, populations and operator settings the engine evolves: one epoch against
the reference module's (tests/golden/ssne_domain_kat.npz), two fed-forward epochs against the oracle at engine scale,
and each kernel on its own against its model (K2: numpy's stable argsort; K3/K4/K5: tests/ssne_domain_cases.py) on
hand-built op lists. Every comparison follows the rule of ssne_domain_cases.py; every launch must leave the rows it was
not told to write untouched, which the whole-matrix comparisons check."""
import os
import random
import types

import numpy as np
import pytest
import torch

from oracle import ssne as OS
import ssne_domain_cases as D

pytestmark = pytest.mark.gpu
KAT = D.load_cases(np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ssne_domain_kat.npz')))
DEV = 'cuda:0'


def i32(a):
    return torch.as_tensor(np.ascontiguousarray(np.asarray(a, dtype=np.int32)), device=DEV)


def random_bits(rng, pop, P):
    """fp32 matrix of arbitrary bit patterns: every NaN payload, signaling NaNs, subnormals, infinities"""
    return rng.randint(0, 2 ** 32, size=(pop, P), dtype=np.uint64).astype(np.uint32).view(np.float32)


@pytest.mark.parametrize('case', sorted(KAT))
def test_device_epoch_equals_reference_module_across_the_domain(case):
    from serl_b200 import evo
    c = KAT[case]
    seed, pop, shape, planted, ef, mprob, mag = D.case_params(c)
    W = torch.as_tensor(D.genomes(seed, pop, shape, planted), device=DEV)
    np.random.seed(seed + 1)
    random.seed(seed + 2)
    elite, plan = evo.epoch_flat(W, c['fitness'], shape, elite_fraction=ef, mutation_prob=mprob, mutation_mag=mag)
    assert elite == int(c['elite'])
    D.assert_case(W.cpu().numpy(), c, D.written_mask(plan, pop, W.shape[1]), case)


@pytest.mark.parametrize('pop,shape,fit_kind', [
    (512, (7, 3, 72, 3), 'ties_nan'), (1025, (7, 3, 16, 2), 'ties'), (4096, (7, 3, 8, 2), 'ties_nan'),
    (16384, (7, 3, 8, 1), 'ties_nan'), (64, (2, 1, 64, 3), 'distinct'), (64, (10, 3, 72, 3), 'ties_nan'),
    (24, (7, 3, 257, 1), 'ties'), (20, (7, 3, 320, 1), 'distinct'), (32, (7, 3, 64, 8), 'ties_nan')])
def test_two_device_epochs_equal_the_oracle_at_engine_scale(pop, shape, fit_kind):
    from serl_b200 import evo
    rng = np.random.RandomState(pop + shape[2])
    before = rng.normal(0, 0.2, (pop, OS.param_table(*shape)[1])).astype(np.float32)
    for gen in range(2):
        fit = rng.uniform(-3000, -50, pop)
        if fit_kind != 'distinct':
            fit = np.round(fit, -2)                      # many exact ties
        if fit_kind == 'ties_nan':
            fit[rng.randint(pop, size=3)] = np.nan
        np.random.seed(11 + gen); random.seed(13 + gen)
        Wo = before.copy()
        elite_o = OS.SSNE(pop, shape).epoch(Wo, fit)
        np.random.seed(11 + gen); random.seed(13 + gen)
        W = torch.as_tensor(before, device=DEV)
        elite, plan = evo.epoch_flat(W, torch.as_tensor(fit, device=DEV), shape)
        assert elite == elite_o
        D.assert_same(W.cpu().numpy(), Wo, D.written_mask(plan, pop, W.shape[1]), 'pop %d %s gen %d' % (pop, shape, gen))
        before = Wo


def _fitness(kind, pop, rng):
    if kind == 'equal':
        return np.full(pop, -7.5)
    if kind == 'nan':
        return np.full(pop, np.nan)
    if kind == 'mixed':
        pool = np.array([np.inf, -np.inf, np.nan, 0.0, -0.0, 5e-324, -5e-324, 2.2e-308, 1.0, -1.0])
        return pool[rng.randint(len(pool), size=pop)]
    return rng.uniform(-3000, -50, pop)


@pytest.mark.parametrize('pop', [1, 2, 1023, 1024, 1025, 12288, 12289, 16384])
@pytest.mark.parametrize('kind', ['distinct', 'equal', 'nan', 'mixed'])
def test_select_kernel_against_numpy_stable_argsort(pop, kind):
    """K2: rank = argsort(kind='stable')[::-1] (NaN first, equal values larger index first), offsprings =
    rank[min of each slot's three draws]; pop > 1024 strides one thread over several i, pop > 12288 needs more than the
    default 48 KB of dynamic shared memory"""
    from serl_b200 import evo
    fit = _fitness(kind, pop, np.random.RandomState(pop))
    for ne in sorted({1, max(pop // 5, 1), pop}):                    # ne == pop: n_off = 0
        np.random.seed(pop + ne)
        rank, offs = evo.select_device(torch.as_tensor(fit, device=DEV), ne)
        want = np.argsort(fit, kind='stable')[::-1]
        assert np.array_equal(rank, want)
        np.random.seed(pop + ne)
        draws = np.stack([np.random.randint(pop, size=3) for _ in range(pop - ne)]) if pop > ne else np.zeros((0, 3), int)
        assert np.array_equal(offs, want[draws.min(1)]) and offs.shape == (pop - ne,)


def _clone(W, pairs):
    from serl_b200 import _native
    Wd = torch.tensor(W, device=DEV)
    _native.call('serl_ssne_clone', Wd, W.shape[0], W.shape[1], i32(pairs), len(pairs))
    torch.cuda.synchronize()
    return Wd.cpu().numpy()


@pytest.mark.parametrize('P', [1, 255, 8193, 8 * 1024 * 3 + 5])
def test_clone_kernel_copies_rows_bit_for_bit(P):
    """K3: grid.x strides P in 1024-element chunks up to 8 blocks, so P = 8*1024*3+5 makes each thread copy several chunks"""
    rng = np.random.RandomState(P)
    W = random_bits(rng, 12, P)
    pairs = [(0, 5), (3, 3), (1, 7), (0, 8), (11, 2)]                # src == dst is a no-op; one source, two targets
    want = W.copy()
    for s, d in pairs:
        want[d] = W[s]
    got = _clone(W, pairs)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_clone_kernel_wave_of_thousands_of_pairs():
    rng = np.random.RandomState(3)
    pop, P = 8000, 37
    W = random_bits(rng, pop, P)
    src = rng.randint(0, 3000, size=4500)
    dst = 3000 + rng.permutation(pop - 3000)[:4500]
    want = W.copy()
    want[dst] = W[src]
    got = _clone(W, np.stack([src, dst], 1))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def _crossover(W, desc, ops):
    """K4 on W through the C-ABI, and the model's result"""
    from serl_b200 import _native
    desc, ops = np.asarray(desc, np.int32).reshape(-1, 6), np.asarray(ops, np.int32).reshape(-1, 3)
    Wd = torch.tensor(W, device=DEV)
    _native.call('serl_ssne_crossover', Wd, W.shape[0], W.shape[1], i32(desc), desc.shape[0], i32(ops))
    torch.cuda.synchronize()
    want = W.copy()
    empty = np.zeros(0, np.int32)
    D.interpret(want, types.SimpleNamespace(clone_waves=[], cross_waves=[(desc, ops)], mut_seg=np.zeros((0, 3), np.int32),
                                            mut_off=empty, mut_kind=empty, mut_z=empty.astype(np.float32)), 0.0)
    return Wd.cpu().numpy(), want


def _assert_bits(got, want):
    bad = np.argwhere(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, '%d elements differ, first %s' % (len(bad), bad[0].tolist())


def _row_ops(rng, layout, n):
    """n crossover ops as crossover_inplace makes them: a whole row (offset base + r*cols, length cols) of one of the
    parameters layout = [(base, rows, cols)], random dir. Ops touching an element all have its row's offset and length,
    which is what K4's ordering without barriers relies on."""
    ops = []
    for _ in range(n):
        base, rows, cols = layout[rng.randint(len(layout))]
        ops.append((base + rng.randint(rows) * cols, cols, rng.randint(2)))
    return ops


@pytest.mark.parametrize('length', [1, 255, 256, 257, 320, 513])
def test_crossover_kernel_op_lengths(length):
    """K4 runs 256 threads: from length 257 on, a thread owns two (513: three) columns of a row op"""
    rng = np.random.RandomState(length)
    layout = [(3, 3, length), (3 + 3 * length, 5, 1)]
    W = random_bits(rng, 6, 3 + 3 * length + 5 + 2)
    ops = _row_ops(rng, layout, 40)
    got, want = _crossover(W, [(1, 2, 4, 5, 0, len(ops))], ops)
    _assert_bits(got, want)


def test_crossover_kernel_keeps_op_order_on_one_row():
    """one row copied back and forth with alternating dir, between ops on other rows: only the ordered result matches"""
    rng = np.random.RandomState(5)
    layout = [(5, 4, 257), (5 + 4 * 257, 6, 1)]
    W = random_bits(rng, 4, 5 + 4 * 257 + 6)
    ops = []
    for k in range(24):
        ops.append((5 + 2 * 257, 257, k % 2))
        ops += _row_ops(rng, layout, 2)
    got, want = _crossover(W, [(0, 1, 2, 3, 0, len(ops))], ops)
    _assert_bits(got, want)
    # the same ops in reverse order give another matrix, so the comparison above decides the order
    _, rev = _crossover(W, [(0, 1, 2, 3, 0, len(ops))], ops[::-1])
    assert not np.array_equal(rev.view(np.uint32), want.view(np.uint32))


def test_crossover_kernel_duplicate_pair_and_self_sources():
    rng = np.random.RandomState(6)
    W = random_bits(rng, 10, 610)
    ops = [(0, 300, 0), (605, 1, 1), (300, 300, 1)]                  # rows of a [2, 300] matrix, one element of a vector
    # padded duplicate pair g1 == g2 with two different sources: the second clone wins, the ops copy the row onto itself
    got, want = _crossover(W, [(4, 4, 1, 2, 0, 3)], ops)
    _assert_bits(got, want)
    assert np.array_equal(got[4].view(np.uint32), W[2].view(np.uint32))
    # s == g: no clone of that slot, the ops act on the slot's own row
    got, want = _crossover(W, [(5, 6, 5, 9, 0, 3), (7, 8, 0, 8, 1, 2)], ops)
    _assert_bits(got, want)


def test_crossover_kernel_many_pairs_per_launch():
    rng = np.random.RandomState(7)
    layout = [(0, 4, 72), (288, 12, 1), (300, 2, 257)]
    pop, P = 1500, 300 + 2 * 257
    W = random_bits(rng, pop, P)
    desc, ops = [], []
    for p in range(500):
        begin = len(ops)
        ops += _row_ops(rng, layout, rng.randint(0, 12))
        desc.append((500 + 2 * p, 501 + 2 * p, rng.randint(500), rng.randint(500), begin, len(ops) - begin))
    got, want = _crossover(W, desc, ops)
    _assert_bits(got, want)


def _mutate(W, seg, off, kind, z, mag):
    from serl_b200 import _native
    Wd = torch.tensor(W, device=DEV)
    z = np.asarray(z, np.float32)
    _native.call('serl_ssne_mutate', Wd, W.shape[0], W.shape[1], i32(seg), len(seg), i32(off), i32(kind),
                 torch.as_tensor(z, device=DEV), float(np.float32(mag)), float(np.float32(10 * mag)))
    torch.cuda.synchronize()
    want = W.copy()
    D.mutate(want, np.asarray(seg), np.asarray(off), np.asarray(kind), z, mag)
    written = np.zeros(W.shape, bool)
    for a, b, n in seg:
        written[a, np.asarray(off)[b:b + n]] = True
    return Wd.cpu().numpy(), want, written


@pytest.mark.parametrize('mag', [0.0, 0.0247682869654, 0.2, 3.0e4])
def test_mutate_kernel_on_every_edge_value(mag):
    """K5 on each planted edge value, every kind, z = +-0 and large |z|; segments of several actors in one launch, some
    offsets mutated several times within a segment. -0.0 weights come out +0.0, NaN stays NaN, +-inf - inf is NaN."""
    E = len(D.EDGE)
    zs = np.array([0.0, -0.0, 1.5, -1.5, 1e-3, -40.0, 1e30], np.float32)
    pop, P = 9, 3 * E * len(zs) + 11
    rng = np.random.RandomState(int(mag * 10) + 1)
    W = rng.normal(0, 0.2, (pop, P)).astype(np.float32)
    seg, off, kind, z = [], [], [], []
    for a in (0, 2, 3, 7):                          # rows 1, 4, 5, 6, 8 are not told to mutate
        begin = len(off)
        for k in range(3):
            for e in range(E):
                for q in range(len(zs)):
                    col = (k * E + e) * len(zs) + q
                    W[a, col] = D.EDGE[e]
                    off.append(col); kind.append(k); z.append(zs[(q + a) % len(zs)])
        for rep in range(6):                        # repeated offsets: the order of the ops decides the result
            off.append(P - 1 - rep % 3); kind.append(rep % 3); z.append(zs[rep % len(zs)])
        seg.append((a, begin, len(off) - begin))
    got, want, written = _mutate(W, seg, off, kind, z, mag)
    D.assert_same(got, want, written, 'mag %g' % mag)
    if mag == 0.0247682869654:
        added = written & (np.arange(P) < 2 * E * len(zs))[None, :]          # kinds 0 and 1 add an increment
        neg0 = (W == 0) & np.signbit(W) & added
        assert neg0.any() and not np.signbit(got[neg0]).any()
        nan_in = np.isnan(W) & added
        assert nan_in.any() and np.isnan(got[nan_in]).all()


def test_apply_plan_phases_pre_then_mut_equal_all():
    from serl_b200 import evo
    c = KAT[sorted(k for k in KAT if KAT[k]['planted'] and int(KAT[k]['pop']) >= 16)[0]]
    seed, pop, shape, planted, ef, mprob, mag = D.case_params(c)
    W0 = D.genomes(seed, pop, shape, planted)
    np.random.seed(seed + 1); random.seed(seed + 2)
    ne = max(int(ef * pop), 1)
    rank, offs = evo.select_device(torch.as_tensor(c['fitness'], device=DEV), ne)
    plan = evo.plan_epoch(rank, offs, evo.param_table(*shape)[0], pop, ne, mprob, native=True)
    assert plan.mut_seg.shape[0] and plan.cross_waves and plan.clone_waves
    Wa = torch.tensor(W0, device=DEV)
    evo.apply_plan(Wa, plan, mag, phase='all')
    Wp = torch.tensor(W0, device=DEV)
    evo.apply_plan(Wp, plan, mag, phase='pre')
    pre = Wp.cpu().numpy().copy()
    evo.apply_plan(Wp, plan, mag, phase='mut')
    assert np.array_equal(Wp.cpu().numpy().view(np.uint32), Wa.cpu().numpy().view(np.uint32))
    want = W0.copy()
    D.interpret(want, types.SimpleNamespace(clone_waves=plan.clone_waves, cross_waves=plan.cross_waves,
                                            mut_seg=np.zeros((0, 3), np.int32), mut_off=None, mut_kind=None, mut_z=None), mag)
    assert np.array_equal(pre.view(np.uint32), want.view(np.uint32))         # 'pre' makes no point mutation
