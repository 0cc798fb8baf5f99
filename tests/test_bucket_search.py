"""The bucketed breakpoint searches of the generated device plant (serl_b200/csrc/gen/plant_rhs_common.h, plant_bucket in
plant_support.h) give the counted search's index for every input: read from the committed text and tables, evaluated both
in exact arithmetic (the fma rounded once, as the hardware does) and through plant_support.h compiled with gcc, at every
breakpoint and both neighbouring doubles, at every cell boundary, at NaN, +-0, +-inf and far out of range, and at random
points.  The whole right-hand side with the bucketed searches (PLANT_SEARCH picking them, as K1's shared-memory instance
does) is bit-identical to the counted one on the recorded and perturbed states.  Also: the generator's certificate
(tools/lift/bucket.py) accepts every emitted table and rejects a corrupted one."""
import ctypes
import math
import os
import re
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEN = os.path.join(ROOT, 'serl_b200', 'csrc', 'gen')
HEX = r'-?0x[0-9a-f.]+p[+-]\d+'
LIT = r'(?:PLANT_K\(\d+\)|%s)' % HEX
CALL = re.compile(r'const int (i\d+) = PLANT_SEARCH\(plant_bucket\((plant_tie_up\()?(\w+)\)?, (%s), (%s), (\d+), PLANT_BKT\((\w+)\), PLANT_TAB\((\w+)\)\), '
                  % (LIT, LIT))


def _val(tok):
    tok = tok.strip()
    return {'(0.0/0.0)': math.nan, '(1.0/0.0)': math.inf, '(-1.0/0.0)': -math.inf}.get(tok) if tok.startswith('(') else float.fromhex(tok)


def _committed():
    blob = open(os.path.join(GEN, 'plant_tables_blob.h')).read()
    offs = {m.group(1): int(m.group(2)) for m in re.finditer(r'PT_OFF_(\w+) = (\d+)', blob)}
    words = [_val(t) for t in re.search(r'plant_tables_blob\[PT_TOTAL\] = \{(.*?)\};', blob, re.S).group(1).split(',') if t.strip()]
    boffs = {m.group(1): int(m.group(2)) for m in re.finditer(r'PB_OFF_(\w+) = (\d+)', blob)}
    bbytes = [int(t) for t in re.sub(r'/\*.*?\*/', '', re.search(r'plant_bucket_blob\[PB_TOTAL\] = \{(.*?)\};', blob, re.S).group(1)).split(',')
              if t.strip()]
    consts = [_val(t) for t in re.search(r'PLANT_CONSTS\(\d+\) = \{(.*?)\};', open(os.path.join(GEN, 'plant_consts.h')).read(),
                                         re.S).group(1).split(',') if t.strip()]

    def lit(tok):
        m = re.match(r'PLANT_K\((\d+)\)', tok)
        return consts[int(m.group(1))] if m else float.fromhex(tok)

    def table(name):
        n = int(re.match(r'[A-Z](\d+)_', name).group(1))
        return words[offs[name]:offs[name] + n]
    out = []
    for m in CALL.finditer(open(os.path.join(GEN, 'plant_rhs_common.h')).read()):
        iv, tie, x, s, o, nb, bk, ax = m.groups()
        bkt = bbytes[boffs[bk]:boffs[bk] + int(nb)]
        out.append(dict(name=iv, tie=tie is not None, s=lit(s), o=lit(o), nb=int(nb), bkt=bkt, xs=table(ax), axis=ax))
    return out


SEARCHES = _committed()


def counted(xs, x):
    """the counted search the generator replaced (codegen.Emitter.index_of): interior breakpoints, '<=' for negative ones"""
    return sum(1 for b in xs[1:-1] if ((b <= x) if b < 0 else (b < x)))


def bucketed(sr, x):
    """plant_bucket on the device: exact fma, floor, clamp to [0, nb-1], NaN -> cell 0"""
    y = math.nextafter(x, math.inf) if (sr['tie'] and x < 0) else x
    nb = sr['nb']
    if y != y:
        c = 0
    elif math.isinf(y):
        c = nb - 1 if y > 0 else 0
    else:
        v = Fraction(y) * Fraction(sr['s']) + Fraction(sr['o'])
        c = 0 if v < -2 else nb - 1 if v > nb + 2 else min(max(math.floor(float(v)), 0), nb - 1)
    n0 = sr['bkt'][c]
    return n0 + (1 if sr['xs'][n0 + 1] < y else 0)


def probe_points(sr):
    pts = [math.nan, 0.0, -0.0, 5e-324, -5e-324, math.inf, -math.inf, 1.7976931348623157e308, -1.7976931348623157e308, 1e300, -1e300,
           1e30, -1e30]
    for b in sr['xs']:
        pts += [math.nextafter(b, -math.inf), b, math.nextafter(b, math.inf)]
    # cell boundaries: the doubles around (k - o) / s for every cell edge k
    for k in range(sr['nb'] + 1):
        e = (k - sr['o']) / sr['s']
        for _ in range(3):
            pts.append(e)
            e = math.nextafter(e, math.inf)
        e = (k - sr['o']) / sr['s']
        for _ in range(3):
            e = math.nextafter(e, -math.inf)
            pts.append(e)
    rng = np.random.default_rng(0)
    lo, hi = sr['xs'][0], sr['xs'][-1]
    w = hi - lo
    pts += list(rng.uniform(lo - 0.25 * w, hi + 0.25 * w, 2000))
    return pts


def test_every_long_search_is_bucketed():
    """the fast device plant has no counted search of 7 or more breakpoints left, and at least the 14 it had"""
    text = open(os.path.join(GEN, 'plant_rhs_common.h')).read()
    assert len(SEARCHES) >= 14
    for m in re.finditer(r'const int i\d+ = (\(.*?\));', text):
        assert m.group(1).count(' + ') + 1 < 7, m.group(0)[:120]


@pytest.mark.parametrize('k', range(len(SEARCHES)), ids=[s['name'] for s in SEARCHES])
def test_bucketed_index_is_the_counted_index(k):
    sr = SEARCHES[k]
    assert all(a < b for a, b in zip(sr['xs'], sr['xs'][1:]))
    assert sr['tie'] == any(b < 0 for b in sr['xs'][1:-1])
    for x in probe_points(sr):
        assert bucketed(sr, x) == (0 if x != x else counted(sr['xs'], x)), (sr['name'], x)


HARNESS = r'''
#include <math.h>
typedef double real;
#define PLANT_FN static
#include "%s"
int bucket_index(double x, int tie, double s, double o, int nb, const unsigned char* bkt, const double* xs)
{
    return plant_bucket(tie ? plant_tie_up(x) : x, s, o, nb, bkt, xs);
}
'''


@pytest.fixture(scope='module')
def clib(tmp_path_factory):
    d = tmp_path_factory.mktemp('bucket')
    (d / 'h.c').write_text(HARNESS % os.path.join(ROOT, 'serl_b200', 'csrc', 'plant_support.h'))
    subprocess.check_call(['gcc', '-O2', '-ffp-contract=off', '-fPIC', '-shared', '-o', str(d / 'h.so'), str(d / 'h.c'), '-lm'])
    lib = ctypes.CDLL(str(d / 'h.so'))
    D = ctypes.c_double
    lib.bucket_index.argtypes = [D, ctypes.c_int, D, D, ctypes.c_int, ctypes.c_char_p, ctypes.POINTER(D)]
    return lib


@pytest.mark.parametrize('k', range(len(SEARCHES)), ids=[s['name'] for s in SEARCHES])
def test_plant_support_bucket_matches_on_the_host(clib, k):
    sr = SEARCHES[k]
    D = ctypes.c_double
    bw = bytes(sr['bkt'])
    xs = (D * len(sr['xs']))(*sr['xs'])
    for x in probe_points(sr):
        got = clib.bucket_index(x, int(sr['tie']), sr['s'], sr['o'], sr['nb'], bw, xs)
        assert got == (0 if x != x else counted(sr['xs'], x)), (sr['name'], x)


def test_generator_certificate_accepts_the_committed_tables_and_rejects_a_corrupted_one():
    sys.path.insert(0, os.path.join(ROOT, 'tools', 'lift'))
    try:
        import bucket as B
    finally:
        sys.path.pop(0)
    for sr in SEARCHES:
        p = B.plan(sr['xs'])
        assert p is not None and (p.s, p.o, p.nb, p.tie, p.bkt) == (sr['s'], sr['o'], sr['nb'], sr['tie'], sr['bkt'])
        starts = [B._first_at_least(j, p.s, p.o, p.nb, p.tie) for j in range(1, p.nb)]
        assert B.certify(p, starts)
        m = len(sr['xs']) - 2
        for c in range(p.nb):
            bad = B.Plan(p.xs, p.s, p.o, p.nb, p.tie, list(p.bkt))
            bad.bkt[c] = (bad.bkt[c] + 1) % m
            assert not B.certify(bad, starts), (sr['name'], c)


def test_right_hand_side_with_bucketed_searches_is_bit_identical_to_the_counted_one(tmp_path):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    try:
        import test_generated_plant as G
    finally:
        sys.path.pop(0)
    libs = {}
    for form, extra in (('counted', ''), ('bucketed', '#define PLANT_SEARCH(bucketed, counted) (bucketed)\n'
                                                      '#define PLANT_BKT(name) (plant_bucket_blob + PB_OFF_##name)\n')):
        src = tmp_path / (form + '.c')
        text = G.HARNESS % {'support': os.path.join(ROOT, 'serl_b200', 'csrc', 'plant_support.h'), 'gen': GEN, 'real': 'double', 'sfx': ''}
        src.write_text(extra + text)
        so = tmp_path / (form + '.so')
        subprocess.check_call(['gcc', '-O1', '-ffp-contract=off', '-fPIC', '-shared', '-o', str(so), str(src), '-lm'])
        libs[form] = ctypes.CDLL(str(so))
    D = ctypes.c_double
    rng = np.random.default_rng(1)
    n = 0
    for v, name in enumerate(G.VARIANTS):
        for x, u in zip(G.KAT[name + '_X'], G.KAT[name + '_U']):
            for scale in (0.0, 1e-3, 1e-1, 1.0):
                xx = x * (1 + scale * rng.standard_normal(19))
                out = {}
                for form, lib in libs.items():
                    o = (D * 19)()
                    lib.dev_rhs(v, (D * 19)(*xx), (D * 4)(*u, 0.0), o)
                    out[form] = np.array(o[:])
                assert np.array_equal(out['counted'].view(np.int64), out['bucketed'].view(np.int64)), (name, xx)
                n += 1
    assert n >= 4000
