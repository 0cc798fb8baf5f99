"""Bucketed breakpoint searches: the counted search of codegen.Emitter.index_of in O(1), exact by construction.

counted (the reference's rt_GetLookupIndex tie rule, one compare per interior breakpoint):
    i = #{1 <= j <= n-2 : xs[j] op_j x},    op_j = '<=' if xs[j] < 0 else '<'
bucketed (plant_bucket / plant_tie_up in serl_b200/csrc/plant_support.h):
    y  = next double above x if x < 0 and some interior breakpoint is negative, else x
         (b <= x  <=>  b < nextup(x): every op_j becomes '<')
    c  = floor(fma(y, s, o)) clamped to [0, nb - 1]; NaN -> 0
    n0 = bkt[c]                                   (one byte per cell, global memory: plant_bucket_blob)
    i  = n0 + (xs[n0 + 1] < y)

plan(xs) picks s, o and nb (the fewest cells that work) and proves bucketed(x) == counted(x) for EVERY double x and NaN, in
exact arithmetic: the fma is evaluated on fractions and rounded once, as the hardware does.  The proof: both sides are
monotone step functions of x.  counted changes only between a breakpoint and its neighbour double; bucketed only where the
cell changes (the boundaries are found by bisection over the ordered doubles, so both doubles around each are known) or
where a compare xs[k] < y changes (between xs[k] and a neighbour).  Every such pair of adjacent doubles is in the set of
critical points the certificate evaluates, so the two functions are constant between consecutive critical points and
agree everywhere once they agree at each of them."""
import math
import struct
from fractions import Fraction

MIN_TERMS = 7        # fewer interior breakpoints: the counted form issues no more than the bucketed one
MAX_NB = 255
_INF = float('inf')


def _bits(x):
    return struct.unpack('<q', struct.pack('<d', x))[0]


def _key(x):
    """strictly increasing integer key of a non-NaN double (-0.0 just below +0.0)"""
    i = _bits(x)
    return i if i >= 0 else -1 - (i & 0x7fffffffffffffff)


def _unkey(k):
    i = k if k >= 0 else (-1 - k) | -0x8000000000000000
    return struct.unpack('<d', struct.pack('<q', i))[0]


def tie_up(x, tie):
    return math.nextafter(x, _INF) if tie and x < 0 else x


def cell(y, s, o, nb):
    """clamp(floor(fma(y, s, o)), 0, nb - 1) with a correctly rounded fma; NaN -> 0 (float -> int conversion of NaN)"""
    if y != y:
        return 0
    if math.isinf(y):
        return nb - 1 if (y > 0) == (s > 0) else 0
    v = Fraction(y) * Fraction(s) + Fraction(o)
    if v < -2:
        return 0
    if v > nb + 2:
        return nb - 1
    return min(max(math.floor(float(v)), 0), nb - 1)     # float(Fraction): one correctly rounded division


def counted(xs, x):
    return sum(1 for b in xs[1:-1] if ((b <= x) if b < 0 else (b < x)))


class Plan:
    def __init__(self, xs, s, o, nb, tie, bkt):
        self.xs, self.s, self.o, self.nb, self.tie, self.bkt = xs, s, o, nb, tie, bkt

    def index(self, x):
        y = tie_up(x, self.tie)
        n0 = self.bkt[cell(y, self.s, self.o, self.nb)]
        return n0 + (1 if self.xs[n0 + 1] < y else 0)

    def name(self):
        import hashlib
        return 'B%d_%s' % (self.nb, hashlib.md5(bytes(self.bkt)).hexdigest()[:10])


def _first_at_least(k, s, o, nb, tie):
    """key of the smallest double x whose cell is >= k (cells are nondecreasing in x)"""
    lo, hi = _key(-_INF), _key(_INF)
    if cell(tie_up(_unkey(lo), tie), s, o, nb) >= k:
        return lo
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if cell(tie_up(_unkey(mid), tie), s, o, nb) >= k:
            hi = mid
        else:
            lo = mid
    return hi


def _build(xs, s, o, nb, tie):
    m = len(xs) - 2
    starts = [_first_at_least(k, s, o, nb, tie) for k in range(1, nb)]
    firsts = [_key(-_INF)] + starts
    lasts = [k - 1 for k in starts] + [_key(_INF)]
    bkt = []
    for a, z in zip(firsts, lasts):
        na = counted(xs, _unkey(min(a, _key(_INF))))
        if a <= z and counted(xs, _unkey(z)) - na > 1:
            return None, None
        bkt.append(min(na, m - 1))
    return bkt, starts


def certify(plan, starts):
    """bucketed == counted at every critical double (module docstring) and at NaN"""
    xs = plan.xs
    pts = {0.0, -0.0, 5e-324, -5e-324, _INF, -_INF, 1.7976931348623157e308, -1.7976931348623157e308}
    for b in xs[1:-1]:
        pts.update((math.nextafter(b, -_INF), b, math.nextafter(b, _INF)))
    for k in starts:
        if _key(-_INF) < k <= _key(_INF):
            pts.update((_unkey(k - 1), _unkey(k)))
    if plan.index(float('nan')) != 0:
        return False
    return all(plan.index(x) == counted(xs, x) for x in pts)


def _quick_reject(inter, s, o):
    """two breakpoints in one cell (by a rounded float evaluation: a filter only, the certificate decides)"""
    cs = [math.floor(b * s + o) for b in inter]
    return any(a == b for a, b in zip(cs, cs[1:]))


_cache = {}


def plan(xs):
    """a certified Plan for the breakpoints xs (strictly increasing), or None when the counted form stays"""
    xs = tuple(xs)
    if xs in _cache:
        return _cache[xs]
    inter = xs[1:-1]
    result = None
    if len(inter) >= MIN_TERMS and all(a < b for a, b in zip(xs, xs[1:])) and all(math.isfinite(b) for b in xs):
        tie = any(b < 0 for b in inter)
        span = inter[-1] - inter[0]
        for nb in range(2, MAX_NB + 1):
            s = (nb - 1) / span
            for phase in (0.5, 0.25, 0.75, 0.125, 0.375, 0.625, 0.875):
                o = phase - inter[0] * s
                if _quick_reject(inter, s, o):
                    continue
                bkt, starts = _build(xs, s, o, nb, tie)
                if bkt is None:
                    continue
                p = Plan(xs, s, o, nb, tie, bkt)
                if certify(p, starts):
                    result = p
                    break
            if result is not None:
                break
    _cache[xs] = result
    return result
