"""K1's two schedules of a CTA's genome slots: lockstep (the default) and slot 1 half a step behind slot 0
(SERL_ROLLOUT_STAGGER) must give the same bits: returns, steps, per-step traces and replay rows, including the time-split
hand-over, idle slots, ragged env counts with early terminations, mixed fault modes and the gust instantiation."""
import os

import numpy as np
import pytest
import torch

from oracle import actor as A, refsig

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), 'golden')
ACT = np.load(os.path.join(G, 'actors.npz'))


def genomes(n, hidden, seed):
    torch.manual_seed(seed)
    return np.stack([A.flatten(A.Actor(hidden=hidden, num_layers=3, activation='tanh')) for _ in range(n)])


def both(weights, hidden, n_envs, modes, horizon, seed, **kw):
    from serl_b200 import rollout
    dev = torch.device('cuda:0')
    sh = rollout.actor_shape(hidden, 3, 'tanh')
    w = torch.as_tensor(np.ascontiguousarray(weights, dtype=np.float32), device=dev)
    lv, st = (torch.as_tensor(x, device=dev) for x in refsig.make_ref_params(n_envs, seed_base=seed))
    md = torch.as_tensor(np.array([rollout.mode_code(modes[i % len(modes)]) for i in range(n_envs)], dtype=np.int32), device=dev)
    out = []
    for stagger in (False, True):
        r = rollout.population_rollout(w, sh, lv, st, md, horizon=horizon, env_order=rollout.variant_sorted_order(md),
                                       stagger=stagger, **kw)
        torch.cuda.synchronize()
        r.check()
        out.append(r)
    return out


def assert_same(a, b, replay_env=None):
    assert torch.equal(a.returns, b.returns) and torch.equal(a.steps, b.steps)
    if a.trace is not None:
        assert torch.equal(torch.nan_to_num(a.trace, nan=-7.0), torch.nan_to_num(b.trace, nan=-7.0))
    if replay_env is not None:          # the rows of the episode (the rest of the buffer is not written)
        for k, n in enumerate(a.steps[:, replay_env].tolist()):
            assert n > 0 and torch.equal(a.replay[k, :n], b.replay[k, :n]), k


@pytest.mark.parametrize('hidden', [32, 72, 96])
@pytest.mark.parametrize('pop', [1, 263, 311, 700])
def test_stagger_equals_lockstep_with_hand_over_and_idle_slots(hidden, pop):
    """pop 1 and 263: fewer tasks than slots (idle slots; at 263 one slot of a two-slot CTA on 132 SMs); 311 and 700: more tasks than slots,
    so slots fly head / tail segments and hand trajectories over through HBM"""
    g = ACT['serl10_pop_h72_tanh'][:5] if hidden == 72 else genomes(5, hidden, 11)
    w = np.tile(g, (pop // 5 + 1, 1))[:pop]
    lock, stag = both(w, hidden, 128, ['nominal', 'ice', 'be', 'jr', 'sa', 'se', 'cg'], 300, 31)
    assert_same(lock, stag)


def test_stagger_equals_lockstep_ragged_early_terminations_traces_replay():
    """70 envs (a ragged last warp), random-init actors that crash early, across a hand-over; traces and replay rows too"""
    w = np.tile(genomes(9, 72, 3), (40, 1))
    lock, stag = both(w, 72, 70, ['nominal'], 2001, 77)
    assert (lock.steps.cpu().numpy() < 2001).any()
    assert_same(lock, stag)
    lock, stag = both(w[:12], 72, 70, ['nominal', 'be', 'ice'], 400, 77, trace=True, replay_env=5)
    assert_same(lock, stag, replay_env=5)


def test_stagger_equals_lockstep_gust():
    """the gust instantiation, across the pulse (20 s to 23 s), with traces"""
    w = np.tile(ACT['serl10_pop_h72_tanh'][:4], (100, 1))
    lock, stag = both(w, 72, 64, ['gust', 'test', 'nominal'], 2001, 5, gust=True)
    assert_same(lock, stag)
    lock, stag = both(w[:6], 72, 64, ['gust', 'test', 'nominal'], 2001, 5, gust=True, trace=True)
    assert_same(lock, stag)
