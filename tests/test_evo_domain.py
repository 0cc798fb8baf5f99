"""K2-K5's models across the actor shapes, populations and operator settings the engine evolves (CPU): the oracle and the
planner + the numpy model of K3/K4/K5 against the reference module's epochs in tests/golden/ssne_domain_kat.npz
(tests/golden/make_golden_ea_domain.py), the C planner against the Python planner, and the C-ABI's refusals."""
import ctypes
import os
import random

import numpy as np
import pytest

from oracle import ssne as OS
from serl_b200 import evo
import ssne_domain_cases as D

# planted NaN / inf / 1e6 weights make the models' fp32 arithmetic overflow and produce NaN on purpose
pytestmark = pytest.mark.filterwarnings('ignore:invalid value:RuntimeWarning', 'ignore:overflow:RuntimeWarning')
KAT = D.load_cases(np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ssne_domain_kat.npz')))
CASES = sorted(KAT)


def plan_case(c, native):
    """the fixture case's genomes before the epoch and the planner's plan for it, seeded as the generator seeded the reference"""
    seed, pop, shape, planted, ef, mprob, mag = D.case_params(c)
    ne = max(int(ef * pop), 1)
    np.random.seed(seed + 1); random.seed(seed + 2)
    rank, offs = D.host_select(c['fitness'], ne)
    plan = evo.plan_epoch(rank, offs, evo.param_table(*shape)[0], pop, ne, mprob, native=native)
    return D.genomes(seed, pop, shape, planted), plan


def test_fixture_covers_the_domain():
    """the shapes, settings and edge paths the fixture was made to reach are in it"""
    shapes = {tuple(int(x) for x in KAT[k]['shape']) for k in CASES}
    for L in (1, 2, 3, 4, 8):
        for h in (8, 72, 257):
            assert (7, 3, h, L) in shapes
    assert {(10, 3, h, 3) for h in (8, 72, 257)} <= shapes and {(2, 1, h, 3) for h in (8, 72, 257)} <= shapes
    assert (7, 3, 320, 1) in shapes and (7, 3, 264, 2) in shapes
    par = [D.case_params(KAT[k]) for k in CASES]
    assert {p[4] for p in par} == {0.2, 0.5} and {p[5] for p in par} == {0.9, 1.0}
    assert {p[6] for p in par} == {0.0247682869654, 0.01, 0.2}
    assert any(p[3] for p in par) and not all(p[3] for p in par)
    assert max(p[1] for p in par) >= 64 and min(p[1] for p in par) == 2
    assert any(p[3] and p[2][2] >= 257 for p in par)
    assert sum(np.isnan(KAT[k]['fitness']).any() for k in CASES) == 1
    # the elitism takes from the offsprings once the unselects run out (`except: offsprings.pop(0)`)
    short = 0
    for k in CASES:
        seed, pop, shape, planted, ef, mprob, mag = D.case_params(KAT[k])
        ne = max(int(ef * pop), 1)
        np.random.seed(seed + 1)
        rank, offs = D.host_select(KAT[k]['fitness'], ne)
        short += pop - len(set(offs.tolist()) | set(rank[:ne].tolist())) < ne
    assert short >= 2


def test_planted_genomes_reach_every_edge_value_in_a_mutated_element():
    """K5's signed-zero and NaN rules are exercised: every planted edge value sits at an element the reference mutated"""
    hit = set()
    for k in CASES:
        c = KAT[k]
        if not c['planted']:
            continue
        W, plan = plan_case(c, native=True)
        m = D.written_mask(plan, W.shape[0], W.shape[1])
        hit |= set(W[m].view(np.uint32).tolist()) & set(D.EDGE.view(np.uint32).tolist())
    assert hit == set(D.EDGE.view(np.uint32).tolist())


@pytest.mark.parametrize('case', CASES)
def test_oracle_reproduces_reference_epoch(case):
    c = KAT[case]
    seed, pop, shape, planted, ef, mprob, mag = D.case_params(c)
    W, plan = plan_case(c, native=True)
    written = D.written_mask(plan, pop, W.shape[1])
    np.random.seed(seed + 1); random.seed(seed + 2)
    elite = OS.SSNE(pop, shape, ef, mprob, mag).epoch(W, c['fitness'])
    assert elite == int(c['elite'])
    D.assert_case(W, c, written, case)


@pytest.mark.parametrize('native', [False, True])
@pytest.mark.parametrize('case', CASES)
def test_plan_and_interpreter_reproduce_reference_epoch(case, native):
    c = KAT[case]
    W, plan = plan_case(c, native)
    D.interpret(W, plan, D.case_params(c)[6])
    assert plan.elite == int(c['elite'])
    D.assert_case(W, c, D.written_mask(plan, W.shape[0], W.shape[1]), case)


def test_mutation_of_signed_zero_gives_positive_zero():
    """the reference's increment random.gauss(0, s*w) is 0 + z*(s*w): -0.0 mutates to +0.0 for either sign of z; NaN and
    inf - inf stay NaN through the clamp, +inf and super-mutated 9.9e5 clamp to 1e6"""
    W = np.full((1, 4), -0.0, np.float32)
    D.mutate(W, np.array([[0, 0, 4]]), np.array([0, 1, 2, 3]), np.array([0, 0, 1, 1]),
             np.array([0.5, -0.5, 1.5, -1.5], np.float32), 0.1)
    assert W.view(np.uint32).tolist() == [[0] * 4]
    W = np.array([[np.nan, np.inf, np.inf, 9.9e5]], np.float32)
    D.mutate(W, np.array([[0, 0, 4]]), np.array([0, 1, 2, 3]), np.array([0, 0, 0, 1]), np.array([1, 1, -1, 2], np.float32), 0.1)
    assert np.isnan(W[0, 0]) and W[0, 1] == np.float32(1e6) and np.isnan(W[0, 2]) and W[0, 3] == np.float32(1e6)


def _plan_and_states(shape, pop, mprob, seed, native):
    table = evo.param_table(*shape)[0]
    ne = max(int(0.2 * pop), 1)
    np.random.seed(seed); random.seed(seed)
    random.gauss(0, 1)                            # leave a cached second variate in the stream
    fit = np.random.uniform(-3000, -50, pop)
    rank, offs = D.host_select(fit, ne)
    plan = evo.plan_epoch(rank, offs, table, pop, ne, mprob, native=native)
    return plan, random.getstate(), np.random.get_state(), random.random(), random.gauss(0, 1), np.random.rand()


@pytest.mark.parametrize('shape,pop,mprob', [((2, 1, 64, 3), 33, 0.9), ((10, 3, 72, 3), 20, 0.9), ((7, 3, 257, 1), 9, 1.0),
                                             ((7, 3, 320, 1), 6, 0.9), ((7, 3, 264, 2), 5, 0.0), ((7, 3, 64, 8), 12, 1.0),
                                             ((7, 3, 8, 1), 4096, 0.9), ((7, 3, 8, 2), 4096, 1.0), ((7, 3, 8, 1), 300, 0.0)])
def test_native_planner_equals_python_planner_across_the_domain(shape, pop, mprob):
    """csrc/evo_plan.cpp against evo.py: identical op lists, identical stdlib / np.random states afterwards"""
    a, b = (_plan_and_states(shape, pop, mprob, pop + shape[2], native) for native in (False, True))
    pa, pb = a[0], b[0]
    for x, y in ((pa.mut_seg, pb.mut_seg), (pa.mut_off, pb.mut_off), (pa.mut_kind, pb.mut_kind), (pa.mut_z, pb.mut_z)):
        assert np.array_equal(x, y)
    assert (pa.mut_seg.shape[0] == 0) == (mprob == 0)
    assert len(pa.cross_waves) == len(pb.cross_waves)
    for (d1, o1), (d2, o2) in zip(pa.cross_waves, pb.cross_waves):
        assert np.array_equal(d1, d2) and np.array_equal(o1, o2)
    for w1, w2 in zip(pa.clone_waves, pb.clone_waves):
        assert np.array_equal(w1, w2)
    assert a[1] == b[1]
    assert np.array_equal(a[2][1], b[2][1]) and a[2][2:] == b[2][2:]
    assert a[3:] == b[3:]


def test_evo_entry_points_refuse_bad_arguments_before_any_cuda_call():
    """every refusal returns SERL_ERR_ARG with the entry point's name; the pointers are never dereferenced"""
    from serl_b200 import build, _native
    build.build()
    L = _native.lib()
    p = ctypes.c_void_p(0x10000)          # non-null, never read
    msg = lambda: L.serl_last_error().decode()

    def refused(rc, name):
        return rc == -1 and name in msg()
    sel = lambda fit=p, pop=4, draws=p, n_off=3, rank=p, offs=p: L.serl_ssne_select(fit, pop, draws, n_off, rank, offs, None)
    for kw in ({'pop': 0}, {'pop': 16385}, {'pop': -1}, {'n_off': -1}, {'fit': None}, {'rank': None}, {'draws': None},
               {'offs': None}):
        assert refused(sel(**kw), 'serl_ssne_select'), kw
    clone = lambda W=p, pop=4, P=10, pairs=p, n=2: L.serl_ssne_clone(W, pop, P, pairs, n, None)
    for kw in ({'W': None}, {'pairs': None}, {'pop': 0}, {'P': 0}, {'n': -1}):
        assert refused(clone(**kw), 'serl_ssne_clone'), kw
    assert clone(W=None, pairs=None, n=0) == 0
    cross = lambda W=p, pop=4, P=10, desc=p, n=2, ops=p: L.serl_ssne_crossover(W, pop, P, desc, n, ops, None)
    for kw in ({'W': None}, {'desc': None}, {'ops': None}, {'pop': 0}, {'P': -3}, {'n': -1}):
        assert refused(cross(**kw), 'serl_ssne_crossover'), kw
    assert cross(W=None, desc=None, ops=None, n=0) == 0
    mut = lambda W=p, pop=4, P=10, seg=p, n=2, off=p, kind=p, z=p: L.serl_ssne_mutate(W, pop, P, seg, n, off, kind, z, 0.1, 1.0, None)
    for kw in ({'W': None}, {'seg': None}, {'off': None}, {'kind': None}, {'z': None}, {'pop': 0}, {'P': 0}, {'n': -1}):
        assert refused(mut(**kw), 'serl_ssne_mutate'), kw
    assert mut(W=None, seg=None, off=None, kind=None, z=None, n=0) == 0
