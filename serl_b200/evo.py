"""Host side of K2-K5: one SSNE generation on the flat [pop, P] device genome matrix.

Control flow and random-number consumption follow base/core/mod_neuro_evo.py SSNE.epoch (:447-543, classic
operators) draw for draw — stdlib `random` and legacy `np.random` global streams, so a run seeded like
base/train.py:88-91 selects, crosses and mutates exactly the individuals the reference would.  The host only
*plans*: it emits compact op lists; every genome byte is moved / changed on the GPU (csrc/evo.cu).

Documented deviations (SURVEY.md F3): index draws use an exclusive upper bound (the reference's inclusive
`random.randint(0, n)` indexes one past the end); ranking ties resolve to the larger index first.
"""
import math
import random

import numpy as np
import torch

from . import _native


def param_table(state_dim, action_dim, hidden, num_layers):
    """[(offset, rows, cols)] in nn.Module.parameters() order (genetic_agent.py:78-101); cols == 0: 1-D of length rows."""
    t, off = [], 0
    for r, c in [(hidden, state_dim), (hidden, 0)] + [(hidden, hidden), (hidden, 0), (hidden, 0), (hidden, 0)] * num_layers + \
            [(action_dim, hidden), (action_dim, 0)]:
        t.append((off, r, c))
        off += r * max(c, 1)
    return t, off


def _waves(items, reads, writes):
    """split an ordered op list into launches with no RAW / WAW / WAR hazard inside a launch."""
    waves, cur, rset, wset = [], [], set(), set()
    for it in items:
        r, w = set(reads(it)), set(writes(it))
        if (w & wset) or (w & rset) or (r & wset):
            waves.append(cur)
            cur, rset, wset = [], set(), set()
        cur.append(it)
        rset |= r
        wset |= w
    if cur:
        waves.append(cur)
    return waves


class EvoPlan:
    __slots__ = ('clone_waves', 'cross_waves', 'mut_seg', 'mut_off', 'mut_kind', 'mut_z', 'elite', 'new_elitists',
                 'offsprings', 'unselects', 'n_cross_ops', 'timing', 'elitist_index', 'mut_candidates', 'distil_unselects')


def plan_epoch(index_rank, offsprings_raw, table, population_size, num_elitists, mutation_prob, selection=None, native=False,
               classic_crossover=True):
    """Everything of SSNE.epoch after the tournaments, as op lists. `selection` (dict) receives rl-selection bookkeeping."""
    index_rank = [int(x) for x in index_rank]
    elitist_index = index_rank[:num_elitists]
    # :49-51
    offsprings = list(set(int(x) for x in offsprings_raw))
    if len(offsprings) % 2 != 0:
        offsprings.append(offsprings[random.randrange(len(offsprings))])
    # :471-476
    new_elitists, unselects = [], []
    sel_set, elite_set = set(offsprings), set(elitist_index)
    for i in range(population_size):
        if i not in sel_set and i not in elite_set:
            unselects.append(i)
    random.shuffle(unselects)
    if selection is not None:
        selection(elitist_index, offsprings, unselects)
    plan = EvoPlan()
    # :489-493 elitism
    clones = []
    for i in elitist_index:
        try:
            replacee = unselects.pop(0)
        except Exception:
            replacee = offsprings.pop(0)
        new_elitists.append(replacee)
        clones.append((i, replacee))
    plan.clone_waves = [np.asarray(w, dtype=np.int32).reshape(-1, 2)
                        for w in _waves(clones, lambda c: (c[0],), lambda c: (c[1],))]
    # :516-523 classic crossover (the distillation branch :497-513 neither pads the list nor draws anything here)
    plan.distil_unselects = list(unselects)
    if not classic_crossover:
        unselects = []
    if len(unselects) % 2 != 0:
        unselects.append(unselects[random.randrange(len(unselects))])
    plan.elite = new_elitists[0]
    plan.new_elitists, plan.offsprings, plan.unselects = new_elitists, offsprings, unselects
    plan.elitist_index = [int(i) for i in elitist_index]       # the ranked elites; new_elitists[k] is the protected clone of [k]
    plan.timing = None
    if native:
        return _plan_tail_native(plan, table, index_rank[num_elitists:] if mutation_prob >= 0 else [], max(mutation_prob, 0.0))
    pairs, ops = [], []
    rnd, rrange, rint = random.random, random.randrange, random.randint
    for i, j in zip(unselects[0::2], unselects[1::2]):
        off_i = random.choice(new_elitists)
        off_j = random.choice(offsprings)
        begin = len(ops)
        for off, rows, cols in table:          # crossover_inplace :61-93
            if cols > 0:
                for _ in range(rint(0, rows * 2)):
                    d = 0 if rnd() < 0.5 else 1
                    ops.append((off + rrange(rows) * cols, cols, d))
            else:
                for _ in range(rint(0, rows)):
                    d = 0 if rnd() < 0.5 else 1
                    ops.append((off + rrange(rows), 1, d))
        pairs.append((i, j, off_i, off_j, begin, len(ops) - begin))
    plan.n_cross_ops = len(ops)
    ops_arr = np.asarray(ops, dtype=np.int32).reshape(-1, 3)
    plan.cross_waves = [(np.asarray(w, dtype=np.int32).reshape(-1, 6), ops_arr)
                        for w in _waves(pairs, lambda p: (p[2], p[3]), lambda p: (p[0], p[1]))]
    # :537-539 mutation of every non-elite rank (mutate_inplace :329-369)
    seg, m_off, m_kind, m_z = [], [], [], []
    for i in (index_rank[num_elitists:] if mutation_prob >= 0 else []):
        if rnd() < mutation_prob:
            plan_mutate_inplace(table, i, np.random.uniform(0, 1, len(table)) * 2, seg, m_off, m_kind, m_z)
    plan.mut_seg, plan.mut_off, plan.mut_kind, plan.mut_z = mutation_arrays(seg, m_off, m_kind, m_z)
    plan.elite = new_elitists[0]
    plan.new_elitists, plan.offsprings, plan.unselects = new_elitists, offsprings, unselects
    return plan


def plan_mutate_inplace(table, actor, ssne_probabilities, seg, m_off, m_kind, m_z):
    """the stdlib `random` draws of one mutate_inplace (:329-369) of genome row `actor`, given its
    ssne_probabilities = np.random.uniform(0, 1, len(table)) * 2: appends K5's ops to the four lists."""
    rnd, rrange, rint, gauss = random.random, random.randrange, random.randint, random.gauss
    for k, (off, rows, cols) in enumerate(table):
        if cols == 0:
            continue
        if rnd() < ssne_probabilities[k]:
            n = rint(0, int(math.ceil(0.1 * rows * cols)))
            begin = len(m_off)
            for _ in range(n):
                e = off + rrange(rows) * cols + rrange(cols)
                r = rnd()
                m_off.append(e)
                m_kind.append(1 if r < 0.05 else (2 if r < 0.1 else 0))
                m_z.append(gauss(0, 1))
            if n:
                seg.append((actor, begin, n))


def mutation_arrays(seg, m_off, m_kind, m_z):
    """K5's op arrays (mut_seg, mut_off, mut_kind, mut_z) from the lists plan_mutate_inplace fills"""
    return (np.asarray(seg, dtype=np.int32).reshape(-1, 3), np.asarray(m_off, dtype=np.int32), np.asarray(m_kind, dtype=np.int32),
            np.asarray(m_z, dtype=np.float64).astype(np.float32))       # fl32(z): torch casts the python scalar first


def _plan_tail_native(plan, table, mut_order, mutation_prob):
    """the two heavy loops (crossover op generation, mutation op generation) in C (csrc/evo_plan.cpp), continuing the
    stdlib `random` and legacy `np.random` streams from their current state and handing the advanced state back."""
    L = _native.lib()
    ver, st, gnext = random.getstate()
    py_state = np.asarray(st, dtype=np.uint32).copy()
    py_gauss = np.array([0.0 if gnext is None else 1.0, 0.0 if gnext is None else gnext], dtype=np.float64)
    name, keys, pos, has_gauss, cached = np.random.get_state()
    np_state = np.concatenate([np.asarray(keys, dtype=np.uint32), np.array([pos], dtype=np.uint32)])
    tab = np.asarray(table, dtype=np.int32).reshape(-1, 3).copy()
    i32 = lambda a: np.ascontiguousarray(np.asarray(a, dtype=np.int32))
    uns, ne, offs, mo = i32(plan.unselects), i32(plan.new_elitists), i32(plan.offsprings), i32(mut_order)
    # ndarray.ctypes keeps its array alive while ctypes converts it to the pointer argument
    h = L.serl_plan_create(py_state.ctypes, py_gauss.ctypes, np_state.ctypes, tab.ctypes, tab.shape[0], uns.ctypes, uns.shape[0],
                           ne.ctypes, ne.shape[0], offs.ctypes, offs.shape[0], mo.ctypes, mo.shape[0], mutation_prob)
    if not h:
        raise IndexError('SSNE.epoch: empty choice pool (no new elitists / offsprings) with crossover pairs pending, as '
                         'random.choice([]) in base/core/mod_neuro_evo.py:519-520')
    sizes = np.zeros(5, dtype=np.int64)
    L.serl_plan_sizes(h, sizes.ctypes)
    n_pairs, n_ops, n_seg, n_mut = (int(x) for x in sizes[:4])
    pairs = np.zeros((n_pairs, 6), np.int32); ops = np.zeros((max(n_ops, 1), 3), np.int32)
    seg = np.zeros((n_seg, 3), np.int32); m_off = np.zeros(n_mut, np.int32); m_kind = np.zeros(n_mut, np.int32)
    m_z = np.zeros(n_mut, np.float32)
    L.serl_plan_copy(h, *(a.ctypes for a in (pairs, ops, seg, m_off, m_kind, m_z)))
    L.serl_plan_destroy(h)
    random.setstate((ver, tuple(int(x) for x in py_state), (py_gauss[1] if py_gauss[0] else None)))
    np.random.set_state((name, np_state[:624], int(np_state[624]), has_gauss, cached))
    plan.n_cross_ops = n_ops
    ops = ops[:n_ops]
    plan.cross_waves = [(np.asarray(w, dtype=np.int32).reshape(-1, 6), ops)
                        for w in _waves([tuple(r) for r in pairs.tolist()], lambda p: (p[2], p[3]), lambda p: (p[0], p[1]))]
    plan.mut_seg, plan.mut_off, plan.mut_kind, plan.mut_z = seg, m_off, m_kind, m_z
    return plan


def _dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device, non_blocking=False)


def select_device(fitness, num_elitists):
    """K2 on the device: tournament draws are made on the host first (np.random.randint(pop, size=3) per slot, :46)."""
    dev = fitness.device
    pop = fitness.shape[0]
    n_off = pop - num_elitists
    draws = np.stack([np.random.randint(pop, size=3) for _ in range(n_off)]).astype(np.int32) if n_off > 0 else np.zeros((0, 3), np.int32)
    d_draws = _dev(draws, dev)
    rank = torch.empty(pop, dtype=torch.int32, device=dev)
    offs = torch.empty(max(n_off, 1), dtype=torch.int32, device=dev)
    _native.call('serl_ssne_select', fitness, pop, d_draws, n_off, rank, offs)
    both = torch.cat([rank, offs[:n_off]]).cpu().numpy()
    return both[:pop], both[pop:]


def apply_plan(weights, plan, mutation_mag, phase='all'):
    """phase 'all', or 'pre' (elitism clones + crossover) / 'mut' (point mutations) when something runs in between
    (distillation crossover writes the unselected genomes before they are mutated)."""
    dev = weights.device
    pop, P = weights.shape
    keep = []
    for w in (plan.clone_waves if phase in ('all', 'pre') else []):
        t = _dev(w, dev); keep.append(t)
        _native.call('serl_ssne_clone', weights, pop, P, t, w.shape[0])
    d_ops = None
    for desc, ops in (plan.cross_waves if phase in ('all', 'pre') else []):
        if d_ops is None:
            d_ops = _dev(ops if ops.size else np.zeros((1, 3), np.int32), dev); keep.append(d_ops)
        t = _dev(desc, dev); keep.append(t)
        _native.call('serl_ssne_crossover', weights, pop, P, t, desc.shape[0], d_ops)
    if plan.mut_seg.shape[0] and phase in ('all', 'mut'):
        seg, off, kind, z = (_dev(a, dev) for a in (plan.mut_seg, plan.mut_off, plan.mut_kind, plan.mut_z))
        keep += [seg, off, kind, z]
        _native.call('serl_ssne_mutate', weights, pop, P, seg, plan.mut_seg.shape[0], off, kind, z,
                     float(np.float32(mutation_mag)), float(np.float32(10 * mutation_mag)))
    torch.cuda.current_stream(dev).synchronize()      # op buffers must outlive the kernels


def epoch_flat(weights, fitness, shape, elite_fraction=0.2, mutation_prob=0.9, mutation_mag=0.0247682869654, selection=None,
               classic_mutation=True, classic_crossover=True, between=None):
    """One generation on device genomes. weights [pop,P] fp32 cuda (modified in place); fitness: cuda f64 tensor or array-like.
    shape = (state_dim, action_dim, hidden, num_layers). Returns (new elite index, plan)."""
    if not weights.is_cuda:
        raise _native.NativeError('epoch_flat needs CUDA genomes (no CPU fallback)')
    pop = weights.shape[0]
    table, P = param_table(*shape)
    assert P == weights.shape[1]
    if not torch.is_tensor(fitness):
        fitness = torch.as_tensor(np.asarray(fitness, dtype=np.float64))
    fitness = fitness.to(device=weights.device, dtype=torch.float64).contiguous()
    import time
    num_elitists = max(int(elite_fraction * pop), 1)
    torch.cuda.current_stream(weights.device).synchronize()     # the fitness may still be in flight: keep its wait out of select_ms
    t0 = time.perf_counter()
    index_rank, offs_raw = select_device(fitness, num_elitists)
    t1 = time.perf_counter()
    # classic_mutation=False (proximal / safe mutation, core/mod_neuro_evo.py): the planner emits no Gaussian point
    # mutations and consumes no draws for them; the caller draws the per-actor decisions itself, in the reference's order
    plan = plan_epoch(index_rank, offs_raw, table, pop, num_elitists, mutation_prob if classic_mutation else -1.0, selection, native=True,
                      classic_crossover=classic_crossover)
    plan.mut_candidates = [int(i) for i in index_rank[num_elitists:]]
    t2 = time.perf_counter()
    if between is None:
        apply_plan(weights, plan, mutation_mag)
    else:          # e.g. distillation crossover: after the elitism clones, before the mutations
        apply_plan(weights, plan, mutation_mag, phase='pre')
        between(plan)
        apply_plan(weights, plan, mutation_mag, phase='mut')
    t3 = time.perf_counter()
    plan.timing = {'select_ms': 1e3 * (t1 - t0), 'plan_ms': 1e3 * (t2 - t1), 'apply_ms': 1e3 * (t3 - t2),
                   'mutations': int(plan.mut_off.shape[0]), 'crossover_copies': int(plan.n_cross_ops)}
    return plan.elite, plan
