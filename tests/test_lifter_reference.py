"""The lifter's hand-restated helper semantics against the exported functions of the reference binary
(rt_GetLookupIndex @0xf470, rt_Lookup @0xf530, rt_Lookup2D_Normal @0xf590), including exact ties, and the branch-free
breakpoint count the generated code uses.  The binary's answers are stored in tests/golden/refbin_kat.npz
(make_golden_refbin.py calls load_binary_lookups / index_cases / formula_cases below on the binary)."""
import ctypes
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools', 'lift'))
D = ctypes.c_double
KAT = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'refbin_kat.npz'))


def load_binary_lookups(so):
    p = os.path.join(tempfile.mkdtemp(), 'c.so')
    shutil.copy(so, p)
    L = ctypes.CDLL(p)
    L.rt_GetLookupIndex.restype = ctypes.c_int
    L.rt_GetLookupIndex.argtypes = [ctypes.POINTER(D), ctypes.c_int, D]
    L.rt_Lookup.restype = D
    L.rt_Lookup.argtypes = [ctypes.POINTER(D), ctypes.c_int, D, ctypes.POINTER(D)]
    L.rt_Lookup2D_Normal.restype = D
    L.rt_Lookup2D_Normal.argtypes = [ctypes.POINTER(D), ctypes.c_int, ctypes.POINTER(D), ctypes.c_int, ctypes.POINTER(D), D, D]
    return L


def axes(rng):
    for n in (2, 3, 4, 6, 9, 11, 17, 22):
        for lo in (-0.3, 0.0, 0.2):
            yield np.sort(lo + np.cumsum(rng.uniform(0.01, 0.3, n)))
        yield np.linspace(-1.0, 1.0, n)          # has an exact 0.0 breakpoint for odd n


def probes(x, rng):
    u = list(rng.uniform(x[0] - 0.5, x[-1] + 0.5, 40)) + list(x) + [0.0, -0.0, x[0] - 1, x[-1] + 1]
    u += list((x[:-1] + x[1:]) / 2)
    return u


def count_rule(x, u):
    """the generated code's index: number of interior breakpoints below u, `<=` for negative breakpoints (codegen.index_of)."""
    return sum((xj <= u) if xj < 0 else (xj < u) for xj in x[1:-1])


def index_cases(lib=None):
    """(breakpoints, probe, the binary's index or None) in a fixed order"""
    rng = np.random.RandomState(0)
    for x in axes(rng):
        arr = (D * len(x))(*x)
        for u in probes(x, rng):
            yield x, u, (lib.rt_GetLookupIndex(arr, len(x), float(u)) if lib else None)


def formula_cases(lib=None):
    """(the binary's 2-D lookup, its 1-D lookup, my 2-D value, my 1-D value) in a fixed order"""
    import symtrace as S
    rng = np.random.RandomState(1)
    li = S.Tracer.lookup_index
    for _ in range(30):
        nx, ny = rng.randint(2, 12), rng.randint(2, 12)
        xs = np.sort(rng.uniform(-1, 1, nx)); ys = np.sort(rng.uniform(-1, 1, ny)); zs = rng.normal(0, 1, nx * ny)
        X, Y, Z = (D * nx)(*xs), (D * ny)(*ys), (D * (nx * ny))(*zs)
        for _ in range(20):
            x, y = rng.uniform(-1.3, 1.3), rng.uniform(-1.3, 1.3)
            ix, iy = li(list(xs), x), li(list(ys), y)
            dx, ux = xs[ix + 1] - xs[ix], x - xs[ix]
            a = (zs[ix + 1 + nx * iy] - zs[ix + nx * iy]) / dx * ux + zs[ix + nx * iy]
            b = (zs[ix + 1 + nx * (iy + 1)] - zs[ix + nx * (iy + 1)]) / dx * ux + zs[ix + nx * (iy + 1)]
            mine = (b - a) / (ys[iy + 1] - ys[iy]) * (y - ys[iy]) + a
            i = li(list(xs), x)
            zz = zs[:nx]
            mine1 = (zz[i + 1] - zz[i]) / (xs[i + 1] - xs[i]) * (x - xs[i]) + zz[i]
            ref2 = lib.rt_Lookup2D_Normal(X, nx, Y, ny, Z, x, y) if lib else None
            ref1 = lib.rt_Lookup(X, nx, x, (D * nx)(*zz)) if lib else None
            yield ref2, ref1, mine, mine1


def test_lookup_index_restatements_equal_the_binary():
    import symtrace as S
    cases = list(index_cases())
    assert len(cases) == len(KAT['lookup_index'])
    for (x, u, _), ref in zip(cases, KAT['lookup_index']):
        assert S.Tracer.lookup_index(list(x), float(u)) == ref, (list(x), u)
        assert count_rule(x, u) == ref, (list(x), u)


def test_lookup_formulas_equal_the_binary():
    cases = list(formula_cases())
    assert len(cases) == len(KAT['lookup2d'])
    for (_, _, mine, mine1), ref2, ref1 in zip(cases, KAT['lookup2d'], KAT['lookup1d']):
        assert mine == ref2           # bit-exact
        assert mine1 == ref1
