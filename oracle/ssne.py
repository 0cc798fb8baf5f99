"""Oracle restatement of the reference's classic neuro-evolution operators on flat fp32 genomes (checker only).

base/core/mod_neuro_evo.py: SSNE.epoch :447-543, selection_tournament :40-52, crossover_inplace :61-93,
mutate_inplace :329-369, clone :371-376, with the documented patches (SURVEY.md F3 / 8(c)):
  * every *index* draw (`random.randint(0, n)` at :51,76,79,89,92,357,358,517) uses an exclusive upper bound
    (random.randrange(n)); the *count* draws (:72,85,355) stay inclusive;
  * ranking is `np.argsort(fitness, kind='stable')[::-1]` — the reference calls the default (unstable) quicksort,
    whose order among exactly equal fitness values is platform dependent; stable-reversed is the documented rule.
Random numbers are consumed from the stdlib `random` and legacy `np.random` global streams in the reference's order.
Arithmetic follows torch's fp32 semantics for 0-d tensor (x) python-scalar expressions. A point mutation adds
random.gauss(0, s*w) = 0 + z*(s*w), so a zero increment is +0.0 and a -0.0 weight comes out +0.0; NaN stays NaN through
the clamp. Validated against the reference module itself: tests/golden/ssne_kat.npz (tests/test_oracle_ssne.py) and,
over the engine's actor shapes with planted signed zeros, NaNs, infinities and subnormals,
tests/golden/ssne_domain_kat.npz (tests/test_evo_domain.py).
"""
import math
import random

import numpy as np


def param_table(state_dim, action_dim, hidden, num_layers):
    """[(offset, rows, cols)] in nn.Module.parameters() order; cols == 0 marks a 1-D parameter of length rows."""
    t, off = [], 0

    def add(r, c):
        nonlocal off
        t.append((off, r, c))
        off += r * max(c, 1)
    add(hidden, state_dim); add(hidden, 0)
    for _ in range(num_layers):
        add(hidden, hidden); add(hidden, 0); add(hidden, 0); add(hidden, 0)
    add(action_dim, hidden); add(action_dim, 0)
    return t, off


class SSNE:
    def __init__(self, pop_size, shape, elite_fraction=0.2, mutation_prob=0.9, mutation_mag=0.0247682869654):
        self.population_size = pop_size
        self.num_elitists = max(int(elite_fraction * pop_size), 1)
        self.mutation_prob = mutation_prob
        self.mutation_mag = mutation_mag
        self.table, self.P = param_table(*shape)
        self.rl_policy = None
        self.selection_stats = {'elite': 0, 'selected': 0, 'discarded': 0, 'total': 0.0000001}

    # :40-52
    def selection_tournament(self, index_rank, num_offsprings, tournament_size):
        total_choices = len(index_rank)
        offsprings = []
        for _ in range(num_offsprings):
            winner = np.min(np.random.randint(total_choices, size=tournament_size))
            offsprings.append(int(index_rank[winner]))
        offsprings = list(set(offsprings))
        if len(offsprings) % 2 != 0:
            offsprings.append(offsprings[random.randrange(len(offsprings))])
        return offsprings

    # :371-376
    @staticmethod
    def clone(W, master, replacee):
        W[replacee] = W[master]

    # :61-93
    def crossover_inplace(self, W, g1, g2):
        for off, rows, cols in self.table:
            if cols > 0:
                n = random.randint(0, rows * 2)
                for _ in range(n):
                    if random.random() < 0.5:
                        r = random.randrange(rows)
                        W[g1, off + r * cols: off + (r + 1) * cols] = W[g2, off + r * cols: off + (r + 1) * cols]
                    else:
                        r = random.randrange(rows)
                        W[g2, off + r * cols: off + (r + 1) * cols] = W[g1, off + r * cols: off + (r + 1) * cols]
            else:
                n = random.randint(0, rows)
                for _ in range(n):
                    if random.random() < 0.5:
                        r = random.randrange(rows)
                        W[g1, off + r] = W[g2, off + r]
                    else:
                        r = random.randrange(rows)
                        W[g2, off + r] = W[g1, off + r]

    # :329-369
    def mutate_inplace(self, W, g, mag):
        f32 = np.float32
        super_mut_strength = 10 * mag
        ssne_probabilities = np.random.uniform(0, 1, len(self.table)) * 2
        for i, (off, rows, cols) in enumerate(self.table):
            if cols == 0:
                continue
            num_weights = rows * cols
            if random.random() < ssne_probabilities[i]:
                num_mutations = random.randint(0, int(math.ceil(0.1 * num_weights)))
                for _ in range(num_mutations):
                    k = off + random.randrange(rows) * cols + random.randrange(cols)
                    random_num = random.random()
                    w = W[g, k]
                    if random_num < 0.05:
                        z = random.gauss(0, 1)
                        w = f32(w + f32(f32(0) + f32(f32(z) * f32(f32(super_mut_strength) * w))))
                    elif random_num < 0.1:
                        w = f32(random.gauss(0, 1))
                    else:
                        z = random.gauss(0, 1)
                        w = f32(w + f32(f32(0) + f32(f32(z) * f32(f32(mag) * w))))
                    W[g, k] = min(max(w, f32(-1000000)), f32(1000000))

    # :447-543 (classic branch)
    def epoch(self, W, fitness_evals):
        index_rank = np.argsort(np.asarray(fitness_evals), kind='stable')[::-1]
        elitist_index = index_rank[:self.num_elitists]
        offsprings = self.selection_tournament(index_rank, len(index_rank) - self.num_elitists, 3)
        new_elitists, unselects = [], []
        for i in range(self.population_size):
            if i not in offsprings and i not in elitist_index:
                unselects.append(i)
        random.shuffle(unselects)
        if self.rl_policy is not None:
            self.selection_stats['total'] += 1.0
            if self.rl_policy in elitist_index:
                self.selection_stats['elite'] += 1.0
            elif self.rl_policy in offsprings:
                self.selection_stats['selected'] += 1.0
            elif self.rl_policy in unselects:
                self.selection_stats['discarded'] += 1.0
            self.rl_policy = None
        for i in elitist_index:
            try:
                replacee = unselects.pop(0)
            except Exception:
                replacee = offsprings.pop(0)
            new_elitists.append(replacee)
            self.clone(W, int(i), replacee)
        if len(unselects) % 2 != 0:
            unselects.append(unselects[random.randrange(len(unselects))])
        for i, j in zip(unselects[0::2], unselects[1::2]):
            off_i = random.choice(new_elitists)
            off_j = random.choice(offsprings)
            self.clone(W, off_i, i)
            self.clone(W, off_j, j)
            self.crossover_inplace(W, i, j)
        for i in index_rank[self.num_elitists:]:
            if random.random() < self.mutation_prob:
                self.mutate_inplace(W, int(i), self.mutation_mag)
        return new_elitists[0]
