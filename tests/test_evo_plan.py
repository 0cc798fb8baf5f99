"""CPU tests of the neuro-evolution planner (serl_b200/evo.py): the op lists it emits, applied by the numpy model of
K3/K4/K5 (tests/ssne_domain_cases.py), must reproduce the genomes recorded from the reference module (tests/golden/ssne_kat.npz)."""
import os
import random

import numpy as np
import pytest

from serl_b200 import evo
from oracle import ssne as OS
from ssne_domain_cases import host_select, interpret

KAT = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'ssne_kat.npz'))
CASES = sorted({k.split('_')[0] for k in KAT.files})


@pytest.mark.parametrize('native', [False, True])
@pytest.mark.parametrize('case', CASES)
def test_plan_reproduces_reference_epoch(case, native):
    before, fit, after = KAT[case + '_before'], KAT[case + '_fitness'], KAT[case + '_after']
    seed = int(KAT[case + '_seed'])
    shape = tuple(int(x) for x in KAT[case + '_shape'])
    table, P = evo.param_table(*shape)
    assert table == OS.param_table(*shape)[0]
    pop = before.shape[0]
    ne = max(int(0.2 * pop), 1)
    np.random.seed(seed + 1)
    random.seed(seed + 2)
    rank, offs = host_select(fit, ne)
    plan = evo.plan_epoch(rank, offs, table, pop, ne, 0.9, native=native)
    W = before.copy()
    interpret(W, plan, 0.0247682869654)
    assert plan.elite == int(KAT[case + '_elite'])
    assert np.array_equal(W.view(np.uint32), after.view(np.uint32))


def test_hazard_waves():
    w = evo._waves([(0, 5), (1, 6), (5, 7), (2, 6)], lambda c: (c[0],), lambda c: (c[1],))
    assert w == [[(0, 5), (1, 6)], [(5, 7), (2, 6)]]


@pytest.mark.parametrize('seed', range(8))
def test_plan_matches_oracle_with_ties_and_odd_sizes(seed):
    """fitness ties, odd unselect counts (padded duplicate pair), tiny populations."""
    rng = np.random.RandomState(seed)
    pop = int(rng.choice([3, 5, 6, 9, 11, 24]))
    shape = (7, 3, 8, int(rng.choice([1, 2, 3])))
    table, P = evo.param_table(*shape)
    before = rng.normal(0, 0.3, (pop, P)).astype(np.float32)
    fit = np.round(rng.uniform(-10, 0, pop))            # many exact ties
    ne = max(int(0.2 * pop), 1)
    np.random.seed(seed); random.seed(seed)
    ev = OS.SSNE(pop, shape)
    Wo = before.copy()
    elite_o = ev.epoch(Wo, fit)
    np.random.seed(seed); random.seed(seed)
    rank, offs = host_select(fit, ne)
    plan = evo.plan_epoch(rank, offs, table, pop, ne, 0.9)
    W = before.copy()
    interpret(W, plan, 0.0247682869654)
    assert plan.elite == elite_o
    assert np.array_equal(W.view(np.uint32), Wo.view(np.uint32))


@pytest.mark.parametrize('pop,seed', [(512, 1), (33, 2), (6, 3)])
def test_native_planner_equals_python_planner_and_leaves_identical_rng_states(pop, seed):
    """csrc/evo_plan.cpp re-implements CPython's random (MT19937, _randbelow, gauss cache) and NumPy's legacy uniform."""
    table, P = evo.param_table(7, 3, 72, 3)
    ne = max(int(0.2 * pop), 1)
    out = []
    for native in (False, True):
        np.random.seed(seed); random.seed(seed)
        random.gauss(0, 1)                       # leave a cached second variate in the stream
        fit = np.random.uniform(-3000, -50, pop)
        rank, offs = host_select(fit, ne)
        plan = evo.plan_epoch(rank, offs, table, pop, ne, 0.9, native=native)
        out.append((plan, random.getstate(), np.random.get_state(), random.random(), random.gauss(0, 1), np.random.rand()))
    a, b = out[0][0], out[1][0]
    for x, y in ((a.mut_seg, b.mut_seg), (a.mut_off, b.mut_off), (a.mut_kind, b.mut_kind), (a.mut_z, b.mut_z)):
        assert np.array_equal(x, y)
    assert len(a.cross_waves) == len(b.cross_waves)
    for (d1, o1), (d2, o2) in zip(a.cross_waves, b.cross_waves):
        assert np.array_equal(d1, d2) and np.array_equal(o1, o2)
    assert out[0][1] == out[1][1]
    assert np.array_equal(out[0][2][1], out[1][2][1]) and out[0][2][2:] == out[1][2][2:]
    assert out[0][3:] == out[1][3:]
