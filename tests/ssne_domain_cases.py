"""Shared by tests/golden/make_golden_ea_domain.py and the K2-K5 domain tests: the seeded genome rule of the fixture
tests/golden/ssne_domain_kat.npz, the numpy model of K3/K4/K5 (csrc/evo.cu), and the comparison rule.

Comparison rule: fp32 bits are equal everywhere, except at an element the point mutations wrote whose reference value
is NaN; there both values must be NaN. x86 keeps an input NaN's payload through arithmetic, the GPU returns its
canonical NaN. Copied NaNs (clones, crossover rows, untouched elements) keep their exact bits.
"""
import hashlib

import numpy as np

from oracle.ssne import param_table

f32 = np.float32
_MAX = np.float32(1e6)
# planted edge values: signed zeros, NaNs with distinct payloads (copies must keep them), infinities, the clamp bound
# and the floats one ulp inside it, values super mutation pushes across the clamp, subnormals
EDGE = np.concatenate([
    np.array([0.0, -0.0, np.inf, -np.inf, 1e6, -1e6, 9.9e5, -9.9e5, 1e-40, -1e-40], np.float32),
    np.array([np.nextafter(_MAX, f32(0)), np.nextafter(-_MAX, f32(0)),
              np.finfo(np.float32).smallest_subnormal, -np.finfo(np.float32).smallest_subnormal], np.float32),
    np.array([0x7fc00000, 0xffc12345], np.uint32).view(np.float32)])
CANONICAL_NAN = np.uint32(0x7fc00000)
N_SAMPLE_COLS = 64


def host_select(fit, num_elitists):
    """K2's model: the tournament draws of selection_tournament (np.random) and the stable-reversed rank"""
    pop = len(fit)
    draws = np.stack([np.random.randint(pop, size=3) for _ in range(pop - num_elitists)])
    rank = np.argsort(fit, kind='stable')[::-1]
    return rank, rank[draws.min(1)]


def genomes(seed, pop, shape, planted):
    """[pop, P] fp32: N(0, 0.2), and with `planted` a quarter of the elements (2-D and 1-D parameters alike) replaced by
    EDGE values at seeded positions."""
    P = param_table(*shape)[1]
    rng = np.random.RandomState(seed)
    W = rng.normal(0, 0.2, (pop, P)).astype(np.float32)
    if planted:
        n = (pop * P + 3) // 4
        W.reshape(-1)[rng.randint(pop * P, size=n)] = EDGE[rng.randint(len(EDGE), size=n)]
    return W


def sample_cols(seed, P):
    return np.unique(np.random.RandomState(seed + 12345).randint(P, size=N_SAMPLE_COLS))


def canonical_bits(W, written):
    """W's bits with every NaN at a written element replaced by one canonical NaN."""
    bits = W.view(np.uint32).copy()
    bits[written & np.isnan(W)] = CANONICAL_NAN
    return bits


def row_digests(W, written):
    bits = canonical_bits(W, written)
    return np.stack([np.frombuffer(hashlib.sha256(r.tobytes()).digest(), np.uint8) for r in bits])


def written_mask(plan, pop, P):
    """the elements K5 writes under `plan`"""
    m = np.zeros((pop, P), bool)
    for a, b, n in plan.mut_seg:
        m[a, plan.mut_off[b:b + n]] = True
    return m


def assert_same(W, ref, written, what=''):
    """W equals ref under the comparison rule (both [rows, cols] fp32, written a bool mask of the same shape)."""
    bad = (W.view(np.uint32) != ref.view(np.uint32)) & ~(written & np.isnan(W) & np.isnan(ref))
    if bad.any():
        r, c = np.argwhere(bad)[0]
        raise AssertionError('%s: %d elements differ, first [%d, %d]: got %r (0x%08x), want %r (0x%08x), written %s'
                             % (what, bad.sum(), r, c, W[r, c], W.view(np.uint32)[r, c], ref[r, c],
                                ref.view(np.uint32)[r, c], written[r, c]))


def load_cases(kat):
    """{name: dict of the case's arrays} from the loaded fixture"""
    out = {}
    for k in kat.files:
        name, field = k.split('_', 1)
        out.setdefault(name, {})[field] = kat[k]
    return out


def case_params(c):
    shape = tuple(int(x) for x in c['shape'])
    return (int(c['seed']), int(c['pop']), shape, bool(c['planted']), float(c['elite_fraction']), float(c['mutation_prob']),
            float(c['mutation_mag']))


def assert_case(W, c, written, what=''):
    """W (the genomes after one epoch) against a fixture case under the comparison rule"""
    assert written.sum(1).tolist() == c['written'].tolist(), what + ': K5 wrote other elements than the reference mutated'
    if 'after' in c:
        assert_same(W, c['after'], written, what)
        return
    cols = c['cols']
    assert_same(np.ascontiguousarray(W[:, cols]), c['sample'], written[:, cols], what + ' (sampled columns)')
    dig = row_digests(W, written)
    bad = [i for i in range(W.shape[0]) if not np.array_equal(dig[i], c['digest'][i])]
    assert not bad, '%s: rows %s differ from the reference (per-row SHA-256)' % (what, bad[:10])


def interpret(W, plan, mag):
    """numpy model of K3/K4/K5 (csrc/evo.cu) applying `plan` to W [pop, P] in place"""
    for wave in plan.clone_waves:
        src = W[wave[:, 0]].copy()
        W[wave[:, 1]] = src                       # all ops of a launch are independent by construction
    for desc, ops in plan.cross_waves:
        snap = W.copy()
        for g1, g2, s1, s2, b, n in desc:
            W[g1] = snap[s1]
            W[g2] = snap[s2]
            for off, ln, d in ops[b:b + n]:
                if d == 0:
                    W[g1, off:off + ln] = W[g2, off:off + ln]
                else:
                    W[g2, off:off + ln] = W[g1, off:off + ln]
    mutate(W, plan.mut_seg, plan.mut_off, plan.mut_kind, plan.mut_z, mag)


def mutate(W, seg, off, kind, z, mag):
    """K5: the reference adds random.gauss(0, s*w) = 0 + z*(s*w), so a zero increment is +0.0; min / max keep NaN"""
    with np.errstate(invalid='ignore', over='ignore'):
        _mutate(W, seg, off, kind, z, mag)


def _mutate(W, seg, off, kind, z, mag):
    for a, b, n in seg:
        for k in range(b, b + n):
            w = W[a, off[k]]
            if kind[k] == 2:
                w = f32(z[k])
            else:
                s = f32(10 * mag) if kind[k] == 1 else f32(mag)
                w = f32(w + f32(f32(0) + f32(f32(z[k]) * f32(s * w))))
            W[a, off[k]] = min(max(w, f32(-1e6)), f32(1e6))
